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

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from tests import gpu_util as G
    from tests import plan_ops
    from tests.conv_ref import conv_env
    from resshift_b200 import _lib

from tests.gn_ref import ROUTES, Case

RAN = set()           # (route, eps, film form, csplit unit or 0) of every launch of this module
OBS = {}              # route -> worst observed ratio of each check to its allowance
PLAN_UNITS = set()    # csplit units (lcm(8, C / 32)) of plan GroupNorms that split channels


def _unit(C):
    cpg = C // 32
    u = cpg
    while u % 8:
        u += cpg
    return u


def _run(L, route, **kw):
    """L.run, its launch recorded."""
    out = L.run(route, **kw)
    RAN.add((route, L.eps, L.film_kind or "none", _unit(L.C) if out[1]["csplit"] > 1 else 0))
    return out


def _check(L, tag, route, out):
    """L.check, its worst ratios recorded per route."""
    for k, v in L.check(tag, route, out).items():
        G.note(OBS.setdefault(route, {}), k, v)


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
    out = _run(L, route, shift=4 * (i % 2))
    _check(L, f"{route} C={Cc} N={N} {H}x{W} eps={eps} silu={silu} film={film} {out[1]}", route, out)


# explicit statistics slots: more than 64 (the finaliser's share of work per image), and fewer rows per slot than the
# statistics kernel has row lanes (256 / (C / 8): 64 lanes at C = 32)
STATS_SLOTS = [("stats_gstat", 32, 1, 64, 64, 256), ("stats_gstat", 96, 3, 32, 32, 128), ("stats_pairs", 32, 3, 16, 16, 32),
               ("stats_pairs", 64, 16, 8, 8, 4), ("stats_gstat", 160, 1, 40, 24, 96), ("stats_pairs", 2048, 1, 16, 16, 256)]


@pytest.mark.parametrize("case", STATS_SLOTS, ids=[f"{c[0]}-C{c[1]}-n{c[2]}-{c[3]}x{c[4]}-s{c[5]}" for c in STATS_SLOTS])
def test_stats_slots(case):
    route, Cc, N, H, W, slots = case
    L = Case(N, H, W, Cc, eps=1e-6, film="image", seed=slots + Cc)
    out = _run(L, route, slots=slots)
    assert out[1]["stats_ctas"] == slots and out[1]["rows_per_slot"] == H * W // slots, out[1]
    _check(L, f"{route} C={Cc} N={N} {H}x{W} slots={slots}", route, out)


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
        out = _run(L, route)
        _check(L, f"{route} {kind} eps={eps} C={Cc} {out[1]}", route, out)


# ---------------------------------------------------------------------------------------------- c. cross-route agreement

def test_cross_route_agreement():
    """One input through every route: each route's gstat (or the statistics implied by its output) agrees with float64;
    each route run twice is bit-identical; the statistics route run twice on the same counters too (the entry zeroes
    them itself)."""
    L = Case(3, 32, 32, 320, eps=1e-6, seed=77)
    counter = torch.zeros(3, dtype=torch.int32, device="cuda")
    for route in ROUTES:
        a = _run(L, route, counter=counter)
        b = _run(L, route, counter=counter)
        assert torch.equal(G.bits(a[0]), G.bits(b[0])), f"{route}: two runs differ"
        if a[2] is not None:
            assert torch.equal(G.bits(a[2]), G.bits(b[2])), f"{route}: gstat of two runs differ"
        _check(L, f"cross-route {route} {a[1]}", route, a)


# ---------------------------------------------------------------------------------------------- d. plan replay

def _plans():
    from oracle.make_golden_variants import variant_config
    ucfg = variant_config("updown")[0]
    assert ucfg.use_scale_shift_norm
    return dict(plan_ops.SHIPPED, unetmodel_nonsquare_b3_40x24=lambda: plan_ops.unetmodel_rows("nonsquare", 40, 24),
                swin_updown_b3_64x64=lambda: plan_ops.swin_rows(ucfg, 3, 64, 64))


PLAN_NAMES = ["realsr_denoiser_b16_64x64", "vq_f4_encode_256", "vq_f4_decode_256", "vq_f8_face_decode_512", "kl_tiny_encode",
              "kl_tiny_decode", "unetmodel_nonsquare_b3_40x24", "swin_updown_b3_64x64"]


@pytest.mark.parametrize("plan", PLAN_NAMES)
def test_plan_groupnorms(plan):
    """Each distinct GroupNorm of a shipped plan (random weights), replayed through rs_op_groupnorm_ex with the plan's
    route, slots, eps, SiLU and FiLM form (FiLM rows replayed once per image and once shared), random gamma, beta and
    input: the entry reports the plan's apply grid and channel slices, and the result is within the float64 bound."""
    with conv_env():
        rows = plan_ops.gn_rows(_plans()[plan]())
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
            out = _run(L, route, slots=slots)
            info = out[1]
            assert (info["slots"], info["apply_ctas"], info["apply_rows"], info["csplit"]) == \
                (d["slots"], d["apply"], d["rows"], d["csplit"]), f"{plan} {d}: launched {info}"
            _check(L, f"{plan} {d} film={film}", route, out)


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
