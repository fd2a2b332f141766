"""GroupNorm (rs_op_groupnorm_ex) as the GPU tests drive it: one launch on any statistics route, and its float64
reference with the bounds of test_gpu_groupnorm.py's module docstring.  Each check returns the worst ratio of its error
to its allowance, per check."""
import ctypes as C

import torch
import torch.nn.functional as F

from resshift_b200 import _lib
from tests import gpu_util as G

U = 2.0 ** -24
K_MU, K_R, K_Q, K_FOLD = 16.0, 512.0, 3072.0, 4.0
ROUTES = {"gstat": 0, "conv_pairs": 1, "window_pairs": 2, "finalize": 3, "stats_pairs": 4, "stats_gstat": 5}
INFO_KEYS = ("route", "slots", "rows_per_slot", "stats_ctas", "finalize", "apply_ctas", "apply_rows", "csplit")


def pairs(t):
    """(mean, M2) over dim 2 of float64 [N, slots, values, C] -> fp32 [N, slots, C, 2]."""
    m = t.mean(2)
    return torch.stack([m, ((t - m[:, :, None]) ** 2).sum(2)], -1).float()


def boxes(x, bh, bw):
    N, H, W, Cc = x.shape
    return x.reshape(N, H // bh, bh, W // bw, bw, Cc).permute(0, 1, 3, 2, 4, 5).reshape(N, -1, bh * bw, Cc)


def conv_pairs(x64):
    """The (mean, M2) pairs a conv epilogue delivers for the float64 map x64 [N, H, W, C], and its tile slots."""
    bw, bh, box_n, slots = G.box128(x64.shape[1], x64.shape[2])
    assert box_n <= 2, "conv epilogues deliver statistics for boxes of at most two images"
    return pairs(boxes(x64, bh, bw)), slots


def group_stats(x64):
    """float64 group mean, biased variance, std [N, 32] of x64 [N, H, W, C]."""
    t = x64.reshape(x64.shape[0], -1, 32, x64.shape[-1] // 32)          # (a view: no copy of a large map)
    mu = t.mean((1, 3))
    var = ((t - mu[:, None, :, None]) ** 2).mean((1, 3))
    return mu, var, var.sqrt()


def data(kind, N, H, W, Cc, g):
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
        self.x64 = data(kind, N, H, W, Cc, g)
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
            self._stats = group_stats(self.x64)
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
        return pairs(self.x64.reshape(self.N, slots, -1, self.C))

    def window_pairs(self, shift):
        x = torch.roll(self.x64, (-shift, -shift), (1, 2))
        return pairs(boxes(x, 8, 8)), (self.H // 8) * (self.W // 8)

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
            p, s = conv_pairs(self.x64) if slots is None else (self.row_pairs(slots), slots)
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
        rest = torch.cat([ybuf[..., :self.yc0], ybuf[..., self.yc0 + Cc:]], -1)
        assert torch.isnan(rest.float()).all(), "channels outside the output view were written"
        y = ybuf[..., self.yc0:self.yc0 + Cc]
        if route in ("stats_pairs", "stats_gstat"):
            part = part[:N * info["slots"] * Cc * 2].view(N, info["slots"], Cc, 2)
        return y, info, (None if route == "gstat" else gstat), part

    # ------------------------------------------------------------------------------------------ checks
    def check_gstat(self, tag, gs):
        mu, var, sd = self.group_stats()
        r = 1.0 / (var + self.eps).sqrt()
        gs = gs.double().to(self.dev)
        assert torch.isfinite(gs).all(), f"{tag}: gstat not written"
        e_mu = ((gs[..., 0] - mu).abs() / (U * (mu.abs() + sd)).clamp(min=1e-300)).max().item()
        e_r = ((gs[..., 1] / r - 1).abs() / U).max().item()
        assert e_mu <= K_MU and e_r <= K_R, f"{tag}: gstat mean error {e_mu:.1f} U, rstd error {e_r:.1f} U"
        return {"gstat_mean": e_mu / K_MU, "gstat_rstd": e_r / K_R}

    def check_stats_pairs(self, tag, part, info):
        t = self.x64.reshape(self.N, info["slots"], -1, self.C)
        m = t.mean(2)
        dev = t - m[:, :, None]
        m2 = (dev ** 2).sum(2)
        maxdev = dev.abs().amax(2)
        p = part.double().to(self.dev)
        assert torch.isfinite(p).all(), f"{tag}: pairs not written"
        e_m = ((p[..., 0] - m).abs() / (U * (m.abs() + maxdev)).clamp(min=1e-300)).max().item()
        e_q = ((p[..., 1] - m2).abs() / (U * (m2 + t.shape[2] * maxdev ** 2)).clamp(min=1e-300)).max().item()
        assert e_m <= K_MU and e_q <= K_Q, f"{tag}: pair mean error {e_m:.1f} U, M2 error {e_q:.1f} U"
        return {"pair_mean": e_m / K_MU, "pair_m2": e_q / K_Q}

    def check_y(self, tag, y, rows=None):
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
        bad = ~(err <= tol)
        assert not bad.any(), f"{tag}: {int(bad.sum())} of {bad.numel()} outside the bound (worst {ratio:.2f} of it)"
        obs = {"y": ratio}
        if not self.silu:
            obs.update(self.check_implied(tag, y, (K_FOLD * U * ((x * A).abs() + B.abs())), x))
        return obs

    def check_implied(self, tag, y, fold, x=None):
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
        if not e_r.numel():
            return {}
        assert e_r.max().item() <= 1 and e_mu.max().item() <= 1, \
            f"{tag}: implied statistics off (rstd {e_r.max().item():.2f}, mean {e_mu.max().item():.2f} of the bound)"
        return {"implied_rstd": e_r.max().item(), "implied_mean": e_mu.max().item()}

    def check(self, tag, route, out, rows=None):
        """Every check the route's outputs take; returns {check: worst ratio to its allowance}."""
        y, info, gs, part = out
        obs = {}
        if gs is not None:
            obs.update(self.check_gstat(tag, gs))
        if route.startswith("stats"):
            obs.update(self.check_stats_pairs(tag, part, info))
        obs.update(self.check_y(tag, y, rows))
        return obs


def check_finalize_gstat(tag, x64, eps, gs, slots):
    """gstat of gn_finalize_kernel, fed the conv pairs of the float64 map x64 [N, H, W, C] in `slots` tile slots per
    image, against float64.  Besides the fixed K_MU / K_R allowances, each of the K = slots * cpg items passes through
    at most n + 16 fp32 roundings (n = K / 256 in one thread's sequential sum, 5 shuffle levels, 8 warp partials, the
    pivot subtraction and the scaling), so with d_i = mean_i - pivot:
        |mean - mean64| <= K_MU U (|mean64| + std64) + (n + 16) U mean|d_i|
        |rstd / rstd64 - 1| <= K_R U + (n + 16) U (1/2 (var + dm^2) + |dm| mean|d_i|) / (var + eps),  dm = mean(d_i),
    the first-order bound of a recursive fp32 sum (relative to the sum of |terms|) pushed through the mean and through
    rsqrt(m2 / (ns K) + eps).  At K = 262144 the count-dependent term is what the rstd needs (n = 1024).  Returns the
    worst ratios (mean, rstd) to the bound."""
    N, Cc = x64.shape[0], x64.shape[-1]
    cpg = Cc // 32
    items = conv_pairs(x64)[0].double()[..., 0].reshape(N, slots, 32, cpg).permute(0, 2, 1, 3).reshape(N, 32, -1)
    n = items.shape[-1] // 256
    dd = items - items[..., :1]
    md, dm = dd.abs().mean(-1), dd.mean(-1)
    mu, var, sd = group_stats(x64)
    gs = gs.double()
    assert torch.isfinite(gs).all(), f"{tag}: gstat not written"
    a_mu = K_MU * U * (mu.abs() + sd) + (n + 16) * U * md
    a_r = K_R * U + (n + 16) * U * (0.5 * (var + dm * dm) + dm.abs() * md) / (var + eps)
    e_mu = ((gs[..., 0] - mu).abs() / a_mu).max().item()
    e_r = ((gs[..., 1] * (var + eps).sqrt() - 1).abs() / a_r).max().item()
    print(f"[gn outlier] {tag}: mean {e_mu:.3g}, rstd {e_r:.3g} of the bound (n = {n})")
    assert e_mu <= 1 and e_r <= 1, f"{tag}: gstat mean {e_mu:.2f}, rstd {e_r:.2f} of the bound"
    return e_mu, e_r
