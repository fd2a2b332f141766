"""Every GroupNorm statistics route of the launcher (rs_op_groupnorm_ex), and each GroupNorm the shipped plans run,
against a float64 GroupNorm32 (F.group_norm on the fp16-stored input, on the CPU; FiLM and SiLU in float64 too).

Routes (include/resshift_b200.h RS_GN_*): the caller's gstat; producer pairs in 128-pixel conv-tile slots or in 8x8
windows, combined by every apply CTA; producer pairs reduced by the finalisation kernel; the statistics kernel's pairs
combined by the apply CTAs; the statistics kernel with the last-CTA reduction into gstat.  Producer pairs are built
here in float64 from the fp16 input, the way a conv epilogue or the fused Swin attention delivers them (their own
correctness is tested with those kernels).

Bounds, with U = 2^-24 (one fp32 rounding) and a, b the float64 per-channel affine y = a x + b:
  * statistics: |mean - mean64| <= K_MU U (|mean64| + std64), |rstd / rstd64 - 1| <= K_R U, for the gstat a route
    writes; for the (mean, M2) pairs of the statistics kernel, the same for the mean (std64 -> max|x - mean|) and
    |M2 - M2_64| <= K_Q U (M2_64 + rows max|x - mean|^2), the magnitude of the pivot-shifted sum of squares;
  * output, per element: |y - y64| <= ulp16(y64) + K_FOLD U (|x a| + |b|) + |a| K_MU U (|mean| + std)
    + |a (x - mean)| K_R U (x 1.1 behind SiLU, its steepest slope): one fp16 rounding, the fp32 fold of mean, rstd,
    gamma, beta and FiLM into a, b, and the statistics error the first bullet allows;
  * without SiLU, the group mean and rstd implied by the output (least squares of (y - B) / A against x, with
    A = gamma (1 + scale), B = beta (1 + scale) + shift) must agree with float64 within the worst case of the fp16
    rounding and fold errors of y propagated through the fit, plus the statistics allowance.
Worst cases observed over this module on an H100 80GB HBM3 (700 W power limit), in U: group mean 3.9, group rstd 129
(the statistics kernel's last-CTA reduction; 2.7 behind the finalisation kernel), pair mean 5.2, pair M2 931; outputs
within 0.50 of their bound (the fp16 rounding dominates), implied statistics within 0.82.  test_every_route_ran prints
the worst ratio of each check to its bound, per route."""
import ctypes as C
import re

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from tests import gpu_util as G
    from resshift_b200 import _lib

U = 2.0 ** -24
K_MU, K_R, K_Q, K_FOLD = 16.0, 512.0, 3072.0, 4.0
ROUTES = {"gstat": 0, "conv_pairs": 1, "window_pairs": 2, "finalize": 3, "stats_pairs": 4, "stats_gstat": 5}
INFO_KEYS = ("route", "slots", "rows_per_slot", "stats_ctas", "finalize", "apply_ctas", "apply_rows", "csplit")
RAN = set()           # (route, eps, film form, csplit unit or 0) of every launch of this module
OBS = {}              # route -> worst observed ratio of each check to its allowance
PLAN_UNITS = set()    # csplit units (lcm(8, C / 32)) of plan GroupNorms that split channels


def _note(route, key, v):
    OBS.setdefault(route, {})
    OBS[route][key] = max(OBS[route].get(key, 0.0), float(v))


def _unit(C):
    cpg = C // 32
    u = cpg
    while u % 8:
        u += cpg
    return u


def _box(H, W):
    """The conv epilogue's 128-pixel box (bw, bh, images per box) and its tile slots per image."""
    def p2(x, cap):
        p = 1
        while p * 2 <= cap and x % (p * 2) == 0:
            p *= 2
        return p
    bw = p2(W, 128)
    bh = p2(H, 128 // bw)
    return bw, bh, 128 // (bw * bh), (W // bw) * (H // bh)


def _pairs(t):
    """(mean, M2) over dim 2 of float64 [N, slots, values, C] -> fp32 [N, slots, C, 2]."""
    m = t.mean(2)
    return torch.stack([m, ((t - m[:, :, None]) ** 2).sum(2)], -1).float()


def _boxes(x, bh, bw):
    N, H, W, Cc = x.shape
    return x.reshape(N, H // bh, bh, W // bw, bw, Cc).permute(0, 1, 3, 2, 4, 5).reshape(N, -1, bh * bw, Cc)


def _data(kind, N, H, W, Cc, g):
    """float64 [N, H, W, C] of fp16-representable values, on the generator's device."""
    x = torch.randn(N, H, W, Cc, generator=g, dtype=torch.float64, device=g.device)
    grp = torch.arange(Cc, device=g.device) // (Cc // 32)
    if kind == "randn":
        x = x * 2 + 0.5
    elif kind == "large_mean":            # per-group mean +-30, std 0.5
        x = x * 0.5 + torch.where(grp % 2 == 0, 30.0, -30.0).double()
    elif kind == "constant":              # groups exactly constant (rstd set by eps), near-constant, and ordinary
        base = torch.where(grp % 2 == 0, 30.0, -0.75).double().expand(N, H, W, Cc).clone()
        near = base + torch.randint(-1, 2, (N, H, W, Cc), generator=g, device=g.device).double() * 2.0 ** -6
        x = torch.where((grp % 3 == 0), base, torch.where(grp % 3 == 1, near, x))
    elif kind == "outlier":               # one value 300 in every group of every image
        x = x.clone()
        for n in range(N):
            for gi in range(32):
                c = gi * (Cc // 32) + (gi + n) % (Cc // 32)
                x[n, (gi * 7 + n) % H, (gi * 3) % W, c] = 300.0
    elif kind == "near_max":              # fp16 values near +-6e4
        x = torch.where(grp % 2 == 0, 6.0e4, -6.0e4).double() + x * 2000
        x = x.clamp(-65504, 65504)
    else:
        raise ValueError(kind)
    return x.half().double()


class Case:
    """One GroupNorm launch: fp16 input view (channel slice of a wider row when padded), gamma, beta, optional FiLM
    rows inside a wider embedding row (per image, or one shared row), and the float64 reference.  The data and the
    reference live on `device` (the CPU unless given; "cuda" for maps whose float64 reference is too slow there)."""

    def __init__(self, N, H, W, Cc, eps=1e-5, silu=0, film=None, pad=False, kind="randn", seed=0, device="cpu"):
        g = torch.Generator(device=device).manual_seed(seed)
        self.dev = g.device
        self.N, self.H, self.W, self.C, self.eps, self.silu, self.film_kind = N, H, W, Cc, eps, silu, film
        self.x64 = _data(kind, N, H, W, Cc, g)
        self.xc0, self.x_ld = (8, Cc + 24) if pad else (0, Cc)
        self.yc0, self.y_ld = (16, Cc + 40) if pad else (0, Cc)
        xbuf = (torch.randn(N, H, W, self.x_ld, generator=g, device=g.device) * 1e4).half()   # what lies outside the view
        xbuf[..., self.xc0:self.xc0 + Cc] = self.x64.half()
        self.xbuf = xbuf.cuda()
        self.gamma = (1 + 0.2 * torch.randn(Cc, generator=g, device=g.device)).float()
        self.beta = (0.2 * torch.randn(Cc, generator=g, device=g.device)).float()
        self.film_off, self.film_sN, self.fbuf = 0, 0, None
        if film is not None:              # this layer's [2C] slice at offset film_off of rows film_sN apart
            self.film_off = 24
            self.film_sN = self.film_off + 2 * Cc + 40 if film == "image" else 0
            rows = N if film == "image" else 1
            self.fbuf = (0.3 * torch.randn(rows * max(self.film_sN, self.film_off + 2 * Cc), generator=g,
                                           device=g.device)).float()
        self._ref = self._stats = None

    def film_rows(self):
        """float64 (scale, shift) [N, C] or None."""
        if self.fbuf is None:
            return None
        f = self.fbuf.double()
        idx = self.film_off + torch.arange(self.N, device=self.dev)[:, None] * self.film_sN + torch.arange(self.C, device=self.dev)[None]
        return f[idx], f[idx + self.C]

    def group_stats(self):
        """float64 group mean, biased variance, std [N, 32]."""
        if self._stats is None:
            t = self.x64.reshape(self.N, -1, 32, self.C // 32)          # (a view: no copy of a large map)
            mu = t.mean((1, 3))
            var = ((t - mu[:, None, :, None]) ** 2).mean((1, 3))
            self._stats = (mu, var, var.sqrt())
        return self._stats

    def ref(self, rows=None):
        """float64 (y, y before SiLU, a, b) as [N, H, W, C], [N, C], [N, C]; with rows (a 1-D index tensor), y of those
        rows of every image only, [N, R, W, C]."""
        if self._ref is None or rows is not None:
            mu, var, _ = self.group_stats()
            r = 1.0 / (var + self.eps).sqrt()
            cpg = self.C // 32
            mu_c, r_c = mu.repeat_interleave(cpg, 1), r.repeat_interleave(cpg, 1)
            gm, bt = self.gamma.double()[None], self.beta.double()[None]
            a = r_c * gm
            b = bt - mu_c * a
            fr = self.film_rows()
            if fr is not None:
                a, b = a * (1 + fr[0]), b * (1 + fr[0]) + fr[1]
            x = self.x64 if rows is None else self.x64[:, rows.to(self.dev)]
            lin = x * a[:, None, None] + b[:, None, None]
            if rows is None:
                # the module's own reference op on the same values, as a cross-check of the affine form above
                yg = F.group_norm(x.permute(0, 3, 1, 2), 32, gm[0], bt[0], eps=self.eps).permute(0, 2, 3, 1)
                if fr is not None:
                    yg = yg * (1 + fr[0][:, None, None]) + fr[1][:, None, None]
                assert (yg - lin).abs().max().item() <= 1e-9 * (1 + lin.abs().max().item())
            y = F.silu(lin) if self.silu else lin
            if rows is not None:
                return (y, lin, a, b)
            self._ref = (y, lin, a, b)
        return self._ref

    def row_pairs(self, slots):
        return _pairs(self.x64.reshape(self.N, slots, -1, self.C))

    def conv_pairs(self):
        bw, bh, box_n, slots = _box(self.H, self.W)
        assert box_n <= 2, "conv epilogues deliver statistics for boxes of at most two images"
        return _pairs(_boxes(self.x64, bh, bw)), slots

    def window_pairs(self, shift):
        x = torch.roll(self.x64, (-shift, -shift), (1, 2))
        return _pairs(_boxes(x, 8, 8)), (self.H // 8) * (self.W // 8)

    def exact_gstat(self):
        mu, var, _ = self.group_stats()
        return torch.stack([mu, 1.0 / (var + self.eps).sqrt()], -1).float()

    def run(self, route, slots=None, shift=0, counter=None):
        """One rs_op_groupnorm_ex launch.  Returns (y view, info, gstat or None, part or None)."""
        N, Cc = self.N, self.C
        a = _lib.GnArgsC()
        a.x, a.x_ld = self.xbuf.data_ptr() + 2 * self.xc0, self.x_ld
        ybuf = torch.full((N, self.H, self.W, self.y_ld), float("nan"), dtype=torch.float16, device="cuda")
        a.y, a.y_ld = ybuf.data_ptr() + 2 * self.yc0, self.y_ld
        a.N, a.H, a.W, a.C = N, self.H, self.W, Cc
        gamma, beta = self.gamma.cuda(), self.beta.cuda()
        a.gamma, a.beta = gamma.data_ptr(), beta.data_ptr()
        fbuf = None if self.fbuf is None else self.fbuf.cuda()
        a.film = None if fbuf is None else fbuf.data_ptr() + 4 * self.film_off
        a.film_sN = self.film_sN
        a.silu, a.eps, a.route = self.silu, self.eps, ROUTES[route]
        part = gstat = None
        if route == "gstat":
            gstat = self.exact_gstat().cuda()
        elif route in ("conv_pairs", "finalize"):
            p, s = self.conv_pairs() if slots is None else (self.row_pairs(slots), slots)
            part, a.slots = p.cuda(), s
        elif route == "window_pairs":
            p, a.slots = self.window_pairs(shift)
            part = p.cuda()
        else:                              # the statistics kernel writes the pairs: NaN until it does
            a.slots = slots or 0
            size = N * slots * Cc * 2 if slots else _lib.lib.rs_op_groupnorm_scratch_floats(N, self.H, self.W, Cc)
            part = torch.full((size,), float("nan"), device="cuda")
        if route in ("finalize", "stats_gstat"):
            gstat = torch.full((N, 32, 2), float("nan"), device="cuda")
        if route == "stats_gstat":
            if counter is None:
                counter = torch.full((N,), 12345, dtype=torch.int32, device="cuda")    # the entry zeroes them
            a.counter = counter.data_ptr()
        a.part = _lib.ptr(part)
        a.gstat = _lib.ptr(gstat)
        info = (C.c_int32 * 8)()
        _lib.check(_lib.lib.rs_op_groupnorm_ex(C.byref(a), info, G.stream()))
        torch.cuda.synchronize()
        info = dict(zip(INFO_KEYS, list(info)))
        assert info["route"] == ROUTES[route]
        if a.slots:
            assert info["slots"] == a.slots, info
        film = self.film_kind or "none"
        RAN.add((route, self.eps, film, _unit(Cc) if info["csplit"] > 1 else 0))
        rest = torch.cat([ybuf[..., :self.yc0], ybuf[..., self.yc0 + Cc:]], -1)
        assert torch.isnan(rest.float()).all(), "channels outside the output view were written"
        y = ybuf[..., self.yc0:self.yc0 + Cc]
        if route in ("stats_pairs", "stats_gstat"):
            part = part[:N * info["slots"] * Cc * 2].view(N, info["slots"], Cc, 2)
        return y, info, (None if route == "gstat" else gstat), part

    # ------------------------------------------------------------------------------------------ checks
    def check_gstat(self, tag, route, gs):
        mu, var, sd = self.group_stats()
        r = 1.0 / (var + self.eps).sqrt()
        gs = gs.double().to(self.dev)
        assert torch.isfinite(gs).all(), f"{tag}: gstat not written"
        e_mu = ((gs[..., 0] - mu).abs() / (U * (mu.abs() + sd)).clamp(min=1e-300)).max().item()
        e_r = ((gs[..., 1] / r - 1).abs() / U).max().item()
        _note(route, "gstat_mean", e_mu / K_MU)
        _note(route, "gstat_rstd", e_r / K_R)
        assert e_mu <= K_MU and e_r <= K_R, f"{tag}: gstat mean error {e_mu:.1f} U, rstd error {e_r:.1f} U"

    def check_stats_pairs(self, tag, route, part, info):
        t = self.x64.reshape(self.N, info["slots"], -1, self.C)
        m = t.mean(2)
        dev = t - m[:, :, None]
        m2 = (dev ** 2).sum(2)
        maxdev = dev.abs().amax(2)
        p = part.double().to(self.dev)
        assert torch.isfinite(p).all(), f"{tag}: pairs not written"
        e_m = ((p[..., 0] - m).abs() / (U * (m.abs() + maxdev)).clamp(min=1e-300)).max().item()
        e_q = ((p[..., 1] - m2).abs() / (U * (m2 + t.shape[2] * maxdev ** 2)).clamp(min=1e-300)).max().item()
        _note(route, "pair_mean", e_m / K_MU)
        _note(route, "pair_m2", e_q / K_Q)
        assert e_m <= K_MU and e_q <= K_Q, f"{tag}: pair mean error {e_m:.1f} U, M2 error {e_q:.1f} U"

    def check_y(self, tag, route, y, rows=None):
        """y against the float64 bound, on every element or on the rows `rows` of every image (the apply is local)."""
        ref, lin, a, b = self.ref(rows)
        mu, _, sd = self.group_stats()
        cpg = self.C // 32
        mu_c, sd_c = mu.repeat_interleave(cpg, 1)[:, None, None], sd.repeat_interleave(cpg, 1)[:, None, None]
        x = self.x64
        if rows is not None:
            x, y = x[:, rows.to(self.dev)], y[:, rows.to(y.device)]
        A, B = a[:, None, None], b[:, None, None]
        gain = 1.1 if self.silu else 1.0
        allow = gain * (K_FOLD * U * ((x * A).abs() + B.abs()) + A.abs() * K_MU * U * (mu_c.abs() + sd_c)
                        + (A * (x - mu_c)).abs() * K_R * U)
        tol = G.ulp16(ref.abs() + allow) + allow
        err = (y.double().to(self.dev) - ref).abs()
        ratio = (err / tol).max().item()
        _note(route, "y", ratio)
        bad = ~(err <= tol)
        assert not bad.any(), f"{tag}: {int(bad.sum())} of {bad.numel()} outside the bound (worst {ratio:.2f} of it)"
        if not self.silu:
            self.check_implied(tag, route, y, (K_FOLD * U * ((x * A).abs() + B.abs())), x)

    def check_implied(self, tag, route, y, fold, x=None):
        """Group mean and rstd implied by the output: with A = gamma (1 + scale), B = beta (1 + scale) + shift,
        y' = (y - B) / A = rstd (x - mean); least squares per group, over the elements of x (all of them unless given)
        and y."""
        N, cpg = self.N, self.C // 32
        A, B = self.gamma.double()[None].expand(N, -1), self.beta.double()[None].expand(N, -1)
        fr = self.film_rows()
        if fr is not None:
            A, B = A * (1 + fr[0]), B * (1 + fr[0]) + fr[1]
        A, B = A[:, None, None], B[:, None, None]
        yd = y.double().to(self.dev)
        u = (0.5 * G.ulp16(yd) + fold) / A.abs()
        yp = (yd - B) / A

        def grp(t):
            return t.reshape(N, -1, 32, cpg).permute(0, 2, 1, 3).reshape(N, 32, -1)
        x, yp, u = grp(self.x64 if x is None else x), grp(yp), grp(u)
        n = x.shape[-1]
        xm = x.mean(-1, keepdim=True)
        dx = x - xm
        sxx = (dx ** 2).sum(-1)
        ok = sxx > 0
        k = (dx * yp).sum(-1) / sxx.clamp(min=1e-300)
        mu_imp = xm[..., 0] - yp.mean(-1) / k.where(ok, torch.ones_like(k))
        mu, var, sd = self.group_stats()
        r = 1.0 / (var + self.eps).sqrt()
        sig_k = (dx.abs() * u).sum(-1) / sxx.clamp(min=1e-300)     # worst case: equal x values round alike
        sig_mu = u.sum(-1) / n / r
        e_r = ((k - r).abs() / (sig_k + K_R * U * r))[ok]
        e_mu = ((mu_imp - mu).abs() / (sig_mu + K_MU * U * (mu.abs() + sd)))[ok]
        if e_r.numel():
            _note(route, "implied_rstd", e_r.max().item())
            _note(route, "implied_mean", e_mu.max().item())
            assert e_r.max().item() <= 1 and e_mu.max().item() <= 1, \
                f"{tag}: implied statistics off (rstd {e_r.max().item():.2f}, mean {e_mu.max().item():.2f} of the bound)"

    def check(self, tag, route, out, rows=None):
        y, info, gs, part = out
        if gs is not None:
            self.check_gstat(tag, route, gs)
        if route.startswith("stats"):
            self.check_stats_pairs(tag, route, part, info)
        self.check_y(tag, route, y, rows)


# ---------------------------------------------------------------------------------------------- a. route matrix

CS = [32, 64, 96, 128, 160, 192, 256, 320, 480, 512, 640, 960, 1280, 2048]
# maps each route admits (H, W): conv pairs need boxes of at most two images, windows whole 8x8 windows
MAPS = {
    "gstat": [(256, 256), (5, 3), (40, 24), (16, 16), (64, 64), (8, 8), (7, 9)],
    "conv_pairs": [(128, 128), (256, 256), (8, 8), (40, 24), (16, 16), (64, 64), (32, 48)],
    "window_pairs": [(128, 128), (8, 8), (40, 24), (16, 16), (64, 64), (32, 64), (24, 40)],
    "finalize": [(256, 256), (128, 128), (40, 24), (64, 64), (16, 16), (128, 64), (8, 8)],
    "stats_pairs": [(5, 3), (256, 256), (40, 24), (16, 16), (64, 64), (7, 9), (8, 8)],
    "stats_gstat": [(256, 256), (5, 3), (40, 24), (16, 16), (64, 64), (7, 9), (128, 128)],
}
MAX_ELEMS = 1 << 22       # float64 reference size per case


def _matrix():
    cases = []
    for route in ROUTES:
        maps = MAPS[route]
        for i, Cc in enumerate(CS):
            # the route's next map (from the i-th) whose reference stays small, at the preferred batch or a smaller one
            H, W = next(m for j in range(len(maps)) for m in [maps[(i + j) % len(maps)]] if m[0] * m[1] * Cc <= MAX_ELEMS)
            N = (1, 3, 16)[i % 3]
            while N > 1 and N * H * W * Cc > MAX_ELEMS:
                N = {16: 3, 3: 1}[N]
            cases.append((route, Cc, N, H, W, (1e-5, 1e-6)[i % 2], (i // 2) % 2, (None, "image", "shared")[i % 3],
                          i % 4 != 0, i))
    return cases


MATRIX = _matrix()


@pytest.mark.parametrize("case", MATRIX, ids=[f"{c[0]}-C{c[1]}-n{c[2]}-{c[3]}x{c[4]}" for c in MATRIX])
def test_route_matrix(case):
    """Each route at every channel count (cpg 1 ... 64), maps from 5x3 to 256x256, both eps, SiLU on and off, FiLM per
    image (row wider than 2C, non-zero offset) and shared, and views with ld > C."""
    route, Cc, N, H, W, eps, silu, film, pad, i = case
    L = Case(N, H, W, Cc, eps=eps, silu=silu, film=film, pad=pad, seed=1000 + i * 7 + ROUTES[route])
    out = L.run(route, shift=4 * (i % 2))
    L.check(f"{route} C={Cc} N={N} {H}x{W} eps={eps} silu={silu} film={film} {out[1]}", route, out)


# explicit statistics slots: more than 64 (the finaliser's share of work per image), and fewer rows per slot than the
# statistics kernel has row lanes (256 / (C / 8): 64 lanes at C = 32)
STATS_SLOTS = [("stats_gstat", 32, 1, 64, 64, 256), ("stats_gstat", 96, 3, 32, 32, 128), ("stats_pairs", 32, 3, 16, 16, 32),
               ("stats_pairs", 64, 16, 8, 8, 4), ("stats_gstat", 160, 1, 40, 24, 96), ("stats_pairs", 2048, 1, 16, 16, 256)]


@pytest.mark.parametrize("case", STATS_SLOTS, ids=[f"{c[0]}-C{c[1]}-n{c[2]}-{c[3]}x{c[4]}-s{c[5]}" for c in STATS_SLOTS])
def test_stats_slots(case):
    route, Cc, N, H, W, slots = case
    L = Case(N, H, W, Cc, eps=1e-6, film="image", seed=slots + Cc)
    out = L.run(route, slots=slots)
    assert out[1]["stats_ctas"] == slots and out[1]["rows_per_slot"] == H * W // slots, out[1]
    L.check(f"{route} C={Cc} N={N} {H}x{W} slots={slots}", route, out)


# ---------------------------------------------------------------------------------------------- b. numerics edges

EDGES = ["large_mean", "constant", "outlier", "near_max"]


@pytest.mark.parametrize("eps", [1e-5, 1e-6])
@pytest.mark.parametrize("kind", EDGES)
@pytest.mark.parametrize("route", list(ROUTES))
def test_numerics_edges(route, kind, eps):
    """Group means far above the spread, constant and near-constant groups (rstd set by eps), a single outlier per
    group, and values near the fp16 limit: what a one-pass E[x^2] - mean^2 or a dropped eps gets wrong."""
    for Cc, N, H, W in ((96, 3, 64, 64), (640, 2, 16, 16)):
        L = Case(N, H, W, Cc, eps=eps, film="shared" if Cc == 640 else None, kind=kind, seed=Cc + len(kind))
        out = L.run(route)
        L.check(f"{route} {kind} eps={eps} C={Cc} {out[1]}", route, out)


# ---------------------------------------------------------------------------------------------- c. cross-route agreement

def test_cross_route_agreement():
    """One input through every route: each route's gstat (or the statistics implied by its output) agrees with float64;
    each route run twice is bit-identical; the statistics route run twice on the same counters too (the entry zeroes
    them itself)."""
    L = Case(3, 32, 32, 320, eps=1e-6, seed=77)
    counter = torch.zeros(3, dtype=torch.int32, device="cuda")
    for route in ROUTES:
        a = L.run(route, counter=counter)
        b = L.run(route, counter=counter)
        assert torch.equal(G.bits(a[0]), G.bits(b[0])), f"{route}: two runs differ"
        if a[2] is not None:
            assert torch.equal(G.bits(a[2]), G.bits(b[2])), f"{route}: gstat of two runs differ"
        L.check(f"cross-route {route} {a[1]}", route, a)


# ---------------------------------------------------------------------------------------------- d. plan replay

_GN = re.compile(r"gn (\d+)x(\d+) C=(\d+) N=(\d+) route=(\w+) slots=(\d+) eps=(\S+) silu=(\d) film=(\w+)@(-?\d+) "
                 r"apply=(\d+) rows=(\d+) csplit=(\d+) ")


def _gn_rows(rows):
    """Distinct GroupNorms of an op list, as dicts of the description's fields."""
    keys = ("H", "W", "C", "N", "route", "slots", "eps", "silu", "film", "film_off", "apply", "rows", "csplit")
    seen = {}
    for r in rows:
        if r.startswith("gn "):
            m = _GN.match(r)
            assert m, r
            d = dict(zip(keys, m.groups()))
            for k in keys:
                if k not in ("route", "eps", "film"):
                    d[k] = int(d[k])
            d["eps"] = float(d["eps"])
            seen.setdefault(tuple(d.values()), d)
    return list(seen.values())


def _unetmodel_rows():
    from oracle.make_golden_unetmodel import case_config, case_inputs
    from resshift_b200.models.unet import UNetModel
    from resshift_b200.weights import random_state_dict
    from tests.test_gpu_conv_instances import _desc_rows
    ucfg, _, _ = case_config("nonsquare")
    m = UNetModel(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 0), strict=True)
    m = m.cuda().eval()
    x, lq = (t.cuda() for t in case_inputs(ucfg, 3, 40, 24, 5))
    t = torch.tensor([3.0, 1.0, 0.0], device="cuda")
    m(x, t, lq=lq)
    return _desc_rows(_lib.lib.rs_plan_profile_ops, m.plan(3, 40, 24).handle, x.data_ptr(), t.data_ptr(), lq.data_ptr(), None)


def _swin_variant_rows():
    from oracle.make_golden_variants import variant_config, variant_inputs
    from resshift_b200.models.unet import UNetModelSwin
    from resshift_b200.weights import random_state_dict
    from tests.test_gpu_conv_instances import _desc_rows
    ucfg, _ = variant_config("updown")
    assert ucfg.use_scale_shift_norm
    m = UNetModelSwin(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 0), strict=True)
    m = m.cuda().eval()
    x, lq, _ = (None if t is None else t.cuda() for t in variant_inputs(ucfg, 3, 64, 64, 6))
    t = torch.tensor([3.0, 1.0, 0.0], device="cuda")
    m(x, t, lq=lq)
    return _desc_rows(_lib.lib.rs_plan_profile_ops, m.plan(3, 64, 64).handle, x.data_ptr(), t.data_ptr(), lq.data_ptr(), None)


def _plans():
    from tests import test_gpu_conv_instances as T
    return dict(T.PLANS, unetmodel_nonsquare_b3_40x24=_unetmodel_rows, swin_updown_b3_64x64=_swin_variant_rows)


PLAN_NAMES = ["realsr_denoiser_b16_64x64", "vq_f4_encode_256", "vq_f4_decode_256", "vq_f8_face_decode_512", "kl_tiny_encode",
              "kl_tiny_decode", "unetmodel_nonsquare_b3_40x24", "swin_updown_b3_64x64"]


@pytest.mark.parametrize("plan", PLAN_NAMES)
def test_plan_groupnorms(plan):
    """Each distinct GroupNorm of a shipped plan (random weights), replayed through rs_op_groupnorm_ex with the plan's
    route, slots, eps, SiLU and FiLM form (FiLM rows replayed once per image and once shared), random gamma, beta and
    input: the entry reports the plan's apply grid and channel slices, and the result is within the float64 bound."""
    from tests.test_gpu_conv_instances import conv_env
    with conv_env():
        rows = _gn_rows(_plans()[plan]())
    assert rows
    print(f"[plan] {plan}: {len(rows)} distinct GroupNorms: " + ", ".join(sorted({d['route'] for d in rows})))
    for i, d in enumerate(rows):
        if d["csplit"] > 1:
            PLAN_UNITS.add(_unit(d["C"]))
        films = [None] if d["film"] == "none" else ["image", "shared"]
        for film in films:
            L = Case(d["N"], d["H"], d["W"], d["C"], eps=d["eps"], silu=d["silu"], film=film, seed=i)
            route = d["route"]
            slots = d["slots"] if route.startswith("stats") else None
            out = L.run(route, slots=slots)
            info = out[1]
            assert (info["slots"], info["apply_ctas"], info["apply_rows"], info["csplit"]) == \
                (d["slots"], d["apply"], d["rows"], d["csplit"]), f"{plan} {d}: launched {info}"
            L.check(f"{plan} {d} film={film}", route, out)


# ---------------------------------------------------------------------------------------------- e. refusals, coverage

def test_refusals():
    """Arguments outside the launcher's domain are refused by name, never launched some other way."""
    x = torch.zeros(16 * 16 * 2080, dtype=torch.float16, device="cuda")
    y = torch.empty_like(x)
    gamma, beta = torch.ones(2080, device="cuda"), torch.zeros(2080, device="cuda")
    part = torch.zeros(1 << 16, device="cuda")
    gstat = torch.zeros(64, device="cuda")

    def refused(match, route="conv_pairs", Cc=64, **fields):
        a = _lib.GnArgsC()
        a.x, a.x_ld, a.y, a.y_ld = x.data_ptr(), Cc, y.data_ptr(), Cc
        a.N, a.H, a.W, a.C = 1, 16, 16, Cc
        a.gamma, a.beta, a.eps, a.route = gamma.data_ptr(), beta.data_ptr(), 1e-5, ROUTES.get(route, route)
        a.part, a.slots, a.gstat = part.data_ptr(), 2, gstat.data_ptr()
        for k, v in fields.items():
            setattr(a, k, v)
        with pytest.raises(_lib.RsError, match=match):
            _lib.check(_lib.lib.rs_op_groupnorm_ex(C.byref(a), None, G.stream()))
    refused("C must be a multiple of 32", Cc=48)
    refused("C must be at most 2048", Cc=2080)
    refused("misaligned ld", x_ld=68)
    refused("misaligned ld", y_ld=60)
    refused("misaligned ld", x=x.data_ptr() + 8)
    refused("slots must divide", slots=3)
    refused("slots must divide", route="finalize", slots=7)
    refused("window pairs", route="window_pairs", slots=2)
    refused("gstat requested without counters", route="stats_gstat")
    refused("eps must be positive", eps=0.0)
    refused("unknown GroupNorm route", route=9)


def test_every_route_ran():
    """Across the module (run it whole): every route, both eps values, both FiLM forms and every channel-slice unit the
    plans use have run.  Prints the worst observed ratio of each check to its allowance, per route."""
    if not RAN:
        pytest.skip("run with the rest of the module")
    for route, d in sorted(OBS.items()):
        print(f"[observed] {route}: " + " ".join(f"{k}={v:.3g}" for k, v in sorted(d.items())))
    assert {r[0] for r in RAN} == set(ROUTES), sorted(set(ROUTES) - {r[0] for r in RAN})
    assert {r[1] for r in RAN} == {1e-5, 1e-6}
    assert {"image", "shared", "none"} <= {r[2] for r in RAN}
    assert PLAN_UNITS <= {r[3] for r in RAN}, sorted(PLAN_UNITS - {r[3] for r in RAN})
