"""Every attention kernel instance, and each attention the shipped plans run on one of them, against float64 references
on the fp16 operands, with a bound per output element.

Kernels: window_attn_kernel<WS, HD> (WS 8 / 16, HD 32 / 64) and the SIMT cross-check (rs_op_window_attention_cfg, with
forced heads per CTA), swin_attn_fused_kernel<E> (rs_op_swin_attn_ex, with forced persistent grids), unet_attn_sm90_kernel
<D> (rs_op_unet_attention) and vq_attn_sm90_kernel<C> (rs_op_vq_attention / _rows).  The first stage's attention over
8192 positions or fewer runs in GEMM form instead (three GEMMs on the conv kernel with softmax_rows_kernel between them,
csrc/vq.inc attn_block); test_gpu_first_stage_kernels.py holds every such block of the first-stage plans and the row
softmax to float64.  test_gpu_cli_tile.py holds vq_attn_sm90_kernel<512> at T = 262144 (the default CLI tile), where
the bound below is too loose to see a lost key block in these classes and a "needle" class is added.

Bound.  For query row i and output channel c, with p_ij the exact (float64) softmax weights, o_ic the exact output and
u16 = 2^-11, u32 = 2^-23 (one fp32 operation; tensor-core accumulation may truncate, so a full ulp):

    |o~ - o| <= 1/2 ulp16 + kP * sum_j p_ij |v_jc| + kS * L_i * dev_ic + s16 * sum_j |v_jc| / l_i

  * The kernels round the unnormalised weights P = exp(s - max) to fp16 for the PV MMA (relative error u16, or an
    absolute 2^-25 below the fp16 normal range: the s16 term, with l_i = sum_j exp(s_ij - max_i) >= 1) while the row sum
    stays fp32.  O and the row sum accumulate in fp32: n_O additions into O (one per k16 MMA step, plus one rescale per
    64-key block for the online kernels) and n_l into the row sum, each relative to the magnitudes summed; the
    normalisation costs two more roundings, ex2.approx a relative 2^-22.  So kP = u16 + (n_O + n_l + 4) u32 + 2^-22:
      - window / fused Swin cores: n_O = T/16, n_l = T/4 + 2 (a lane's 16 or 64 keys, then two shuffles);
      - unet / VQ online softmax: n_O = ceil(T/16) + ceil(T/64), n_l = 18 + 2 ceil(T/64).
    The SIMT cross-check keeps P in fp32 and accumulates with fmaf in round-to-nearest: kP = (2T + 6) 2^-24 + 2^-22, and
    no s16 term.
  * A logit error d_j changes o by sum_j p_ij d_j (v_jc - o_ic), at most max|d| * sum_j p_ij |v_jc - o_ic|; dev_ic =
    sqrt(sum_j p_ij (v_jc - o_ic)^2) bounds that sum from above (Jensen).  The logits accumulate D products in fp32, then
    take the scale, the bias, the mask, the max subtraction and the log2(e) factor of __expf / exp2 (the last two on
    values up to 2 L_i): |d| <= kS L_i with kS = (D + 7) u32 (D + 8 for VQ, which adds two channel halves), where
    L_i = max_j (scale sum_d |q_id| |k_jd| + |bias_ij|) (bias includes the -100 of the shift mask).
  * Equal logits (q = 0, no bias): every P is exactly 1, so only the accumulation part of kP applies.

The fused Swin reference reproduces the unfused path's fp16 stores (norm1 output, qkv, attention output) on float64
values and carries an allowance forward through each stage: the fp16 ulp of the stored intermediate (kernel and
reference may round neighbouring values apart), the stage's own term, and the previous allowance pushed through the
stage in absolute values (|W| * allow for the GEMMs; for attention sum_j p_ij allow(v_jc) plus the logit perturbation
e_i = scale max_j sum_d (a(q) |k| + |q| a(k) + a(q) a(k)) times e^(2 e_i) dev_ic).  norm1 allows a group-mean error of
64 * 2^-24 (|mean| + std) and a relative rstd error of 1024 * 2^-24 on top of the fp32 affine fold.

The worst ratio of each check to its allowance is printed per kernel and input class by test_coverage.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from tests import gpu_util as G
    from tests import plan_ops
    from tests.attn_ref import SwinCase, WindowCase, sms, unet_case, vq_case
    from resshift_b200 import _lib

INSTANCES = [(8, 32), (8, 64), (16, 32), (16, 64)]
CLASSES = ("randn", "peaked", "probe", "equal", "large")
SLOTS = (1, 4, 15, 16, 17, 32, 128, 512)

RAN = set()          # what ran: (kind, feature)
OBS = {}             # worst ratio per (kernel, input class)


def _note(kernel, cls, ratio):
    G.note(OBS, (kernel, cls), ratio)
    RAN.add(("class", kernel, cls))
    RAN.add(("instance", kernel))


def _window(L, tag, hpc=0, simt=False):
    """L.check, recorded: the kernel, its input class and the heads per CTA it ran."""
    out, info, ratio = L.check(tag, hpc=hpc, simt=simt)
    kernel = "window_simt" if simt else f"window<{L.ws},{L.hd}>"
    _note(kernel, L.cls, ratio)
    if not simt:
        RAN.add(("hpc", kernel, "1" if info["hpc"] == 1 else "all" if info["hpc"] == L.heads else "divisor"))
    return out, info


def _swin(L, tag, grid=0):
    """L.check, recorded: the instance, its input class, the norm1 slot count and how pairs fell on the CTAs."""
    y, pout, info, ratio = L.check(tag, grid)
    _note(f"swin<{L.E}>", L.cls, ratio)
    RAN.add(("slots", L.slots))
    if info["pairs_per_cta"] >= 2:
        RAN.add(("swin", "several pairs per CTA"))
    pairs = (L.N * L.nW + 1) // 2
    if any((2 * p + 1) % L.nW == 0 for p in range(pairs) if 2 * p + 1 < L.N * L.nW):
        RAN.add(("swin", "pair straddles images"))
    return y, pout


def _unet(cls, N, T, heads, D, new_order, seed, tag=None):
    _note(f"unet<{D}>", cls, unet_case(cls, N, T, heads, D, new_order, seed, tag)[1])


def _vq(cls, N, T, Cc, seed, rows=None):
    _note(f"vq<{Cc}>", cls, vq_case(cls, N, T, Cc, seed, rows))


# ------------------------------------------------------------------------------------------------ window core

def default_hpc(heads, windows):
    """The launcher's rule (launch.cuh attn_default_hpc)."""
    hpc = heads
    while hpc > 1 and windows * (heads // hpc) < 4 * sms() and hpc % 2 == 0:
        hpc //= 2
    if hpc > 1 and windows * (heads // hpc) < 4 * sms():
        hpc = 1
    return hpc


WINDOW_SHAPES = [(1, 1, 1, False), (3, 3, 5, False), (3, 3, 5, True), (1, 2, 3, True)]


def _divisors(n):
    return [d for d in range(1, n + 1) if n % d == 0]


@pytest.mark.parametrize("shape", WINDOW_SHAPES, ids=lambda s: f"N{s[0]}-{s[1]}x{s[2]}-shift{int(s[3])}")
@pytest.mark.parametrize("ws,hd,heads", [(8, 32, 6), (8, 64, 4), (16, 32, 6), (16, 64, 4), (8, 32, 3), (16, 64, 1)])
def test_window_core_every_hpc(ws, hd, heads, shape):
    """randn operands: every heads-per-CTA count (1, each proper divisor, all heads) and the SIMT kernel agree with
    float64, and the entry reports the launch it was asked for."""
    N, nwy, nwx, shifted = shape
    L = WindowCase("randn", N, nwy, nwx, heads, ws, hd, ws // 2 if shifted else 0, seed=ws * 131 + hd + heads + nwx + shifted)
    outs = []
    for hpc in _divisors(heads):
        out, info = _window(L, f"window<{ws},{hd}> heads={heads} {shape} hpc={hpc}", hpc=hpc)
        assert info["hpc"] == hpc and info["grid"] == (N * nwy * nwx, heads // hpc) and info["simt"] == 0, info
        outs.append(out)
    assert all(torch.equal(outs[0], o) for o in outs[1:]), "results depend on the heads per CTA"
    _, info = _window(L, f"window simt ws={ws} hd={hd} {shape}", simt=True)
    assert info["simt"] == 1 and info["grid"] == (N * nwy * nwx, heads)


@pytest.mark.parametrize("cls", ["peaked", "probe", "equal", "large"])
@pytest.mark.parametrize("ws,hd,heads", [(8, 32, 6), (8, 64, 4), (16, 32, 6), (16, 64, 4)])
def test_window_core_input_classes(ws, hd, heads, cls):
    """Peaked logits with the maximum at a window's first / last token and on both sides of the mask boundary, the
    bias / mask probe (q = 0, S = bias + mask exactly) on every window position of a shifted map, equal logits and
    large magnitudes, through the instance with all heads per CTA and one, and the SIMT kernel."""
    shift = 0 if cls == "equal" else ws // 2
    L = WindowCase(cls, 3, 3, 5, heads, ws, hd, shift, seed=ws + hd + len(cls))
    a, _ = _window(L, f"window<{ws},{hd}> {cls} hpc=all", hpc=heads)
    b, _ = _window(L, f"window<{ws},{hd}> {cls} hpc=1", hpc=1)
    assert torch.equal(a, b)
    _window(L, f"window simt ws={ws} hd={hd} {cls}", simt=True)


@pytest.mark.parametrize("ws,hd,heads", [(8, 32, 6), (16, 64, 4)])
def test_window_core_launcher_rule_picks_several_heads(ws, hd, heads):
    """At a window count of at least 4 * SMs per head group the launcher itself puts all heads in one CTA."""
    per = math.ceil(4 * sms() / 12)
    L = WindowCase("peaked", 4, 3, per, heads, ws, hd, ws // 2, seed=3)
    windows = 12 * per
    want = default_hpc(heads, windows)
    assert want > 1
    _, info = _window(L, f"window<{ws},{hd}> launcher rule, {windows} windows", hpc=0)
    assert info["hpc"] == want and info["grid"] == (windows, heads // want), info
    RAN.add(("rule_hpc", f"window<{ws},{hd}>"))


def test_window_core_refusals():
    qkv = torch.zeros(1, 16, 16, 3 * 128, dtype=torch.float16, device="cuda")
    dense = torch.zeros(4 * 64 * 64, device="cuda")
    for hpc, simt, match in ((3, 0, "hpc must divide heads"), (-1, 0, "hpc must divide heads"), (2, 1, "SIMT")):
        rc = _lib.lib.rs_op_window_attention_cfg(qkv.data_ptr(), 1, 16, 16, 4, 8, 32, 0, dense.data_ptr(), qkv.data_ptr(),
                                                 hpc, simt, None, G.stream())
        assert rc != 0 and match.encode() in _lib.lib.rs_last_error(), (hpc, simt)


# ------------------------------------------------------------------------------------------------ fused Swin attention half

@pytest.mark.parametrize("E", [64, 192])
@pytest.mark.parametrize("shift", [0, 4])
@pytest.mark.parametrize("grid", [1, 2, 3, 7, 0])
def test_swin_forced_grids_odd_windows(grid, shift, E):
    """24x40 maps (15 windows per image) at N = 3: 23 pairs, so pairs straddle images and the last pair has one window;
    grids of 1, 2, 3 and 7 CTAs walk many pairs each.  In place equals out of place bit for bit, and runs repeat."""
    L = SwinCase("randn", 3, 24, 40, E, shift, 16, seed=E + shift + grid)
    y, pout = _swin(L, f"swin<{E}> shift={shift} grid={grid}", grid=grid)
    y2, pout2, _ = L.run(grid, inplace=True)
    assert torch.equal(G.bits(y), G.bits(y2)) and torch.equal(G.bits(pout), G.bits(pout2)), "in place differs"
    y3, pout3, _ = L.run(grid)
    assert torch.equal(G.bits(y), G.bits(y3)) and torch.equal(G.bits(pout), G.bits(pout3)), "two runs differ"


@pytest.mark.parametrize("E", [64, 192])
@pytest.mark.parametrize("cls", ["peaked", "probe", "equal", "large", "largemean"])
def test_swin_input_classes(cls, E):
    shift = 0 if cls == "equal" else 4
    L = SwinCase(cls, 3, 24, 40, E, shift, 15, seed=len(cls) * 7 + E)
    _swin(L, f"swin<{E}> {cls}", grid=3)
    _swin(L, f"swin<{E}> {cls} default grid")


# (slots, H, W): equal boxes of H*W / slots pixels
SLOT_MAPS = {1: (8, 8), 4: (16, 16), 15: (24, 40), 16: (24, 40), 17: (136, 8), 32: (24, 40), 128: (64, 64), 512: (64, 64)}


@pytest.mark.parametrize("cls", ["randn", "largemean"])
@pytest.mark.parametrize("slots", SLOTS)
def test_swin_norm1_slot_counts(slots, cls):
    H, W = SLOT_MAPS[slots]
    E = 192 if slots % 2 == 0 else 64
    L = SwinCase(cls, 3, H, W, E, 4 if H > 8 and W > 8 else 0, slots, seed=slots + len(cls))
    _swin(L, f"swin<{E}> {cls} slots={slots} {H}x{W}", grid=7 if 3 * L.nW >= 14 else 0)


def test_swin_refusals():
    L = SwinCase("randn", 1, 16, 16, 64, 0, 4, seed=1)
    for grid, match in ((3, "grid must be in"), (-1, "grid must be in")):
        with pytest.raises(_lib.RsError, match=match):
            L.run(grid)
    L.slots = 3
    with pytest.raises(_lib.RsError, match="slots must divide"):
        L.run(0)
    gst = torch.zeros(64, device="cuda")
    with pytest.raises(_lib.RsError, match="gstat_out and counters must be NULL"):
        _lib.check(G.L.rs_op_swin_attn(L.x.data_ptr(), 1, 16, 16, 64, 2, 0, L.part.data_ptr(), 4, L.gamma.data_ptr(),
                                       L.beta.data_ptr(), L.wq_p.data_ptr(), L.bqkv.data_ptr(), L.dense.data_ptr(),
                                       L.wp_p.data_ptr(), L.bproj.data_ptr(), L.x.data_ptr(), None, gst.data_ptr(), None,
                                       G.stream()))


# ------------------------------------------------------------------------------------------------ unet_attn

UNET_T = [2, 127, 128, 129, 191, 193, 4095, 4097]


@pytest.mark.parametrize("T", UNET_T)
@pytest.mark.parametrize("D", [32, 64, 128])
def test_unet_attention_lengths(D, T):
    """The T on either side of the 64-key blocks and the 128-query CTAs that test_gpu_unetmodel.py's head-count matrix
    (T = 1, 15, 63, 64, 65, 1000, 4096, 16384) does not take; three heads, the head order alternating with T, N = 2."""
    _unet("randn", 2, T, 3, D, UNET_T.index(T) % 2 == 1, seed=D * 1000 + T)


@pytest.mark.parametrize("cls", ["peaked", "equal", "large"])
@pytest.mark.parametrize("T", [63, 129, 4097])
@pytest.mark.parametrize("D", [32, 64, 128])
def test_unet_attention_input_classes(D, T, cls):
    _unet(cls, 2, T, 3, D, T % 2 == 1, seed=D + T + len(cls))


# ------------------------------------------------------------------------------------------------ vq_attn

# randn at T = 64, 384, 4096, 16384 and 65536 is held by test_gpu_vq_attention.py::test_op_vs_fp32; equal and large
# logits at T <= 4096
VQ_CASES = [(c, t, cls) for c in (128, 256, 512) for t in (64, 128, 4096, 16384) for cls in ("randn", "peaked", "equal", "large")
            if (cls != "randn" or t == 128) and (t < 16384 or cls == "peaked")]


@pytest.mark.parametrize("Cc,T,cls", VQ_CASES, ids=[f"C{c}-T{t}-{cls}" for c, t, cls in VQ_CASES])
def test_vq_attention(Cc, T, cls):
    _vq(cls, 2, T, Cc, seed=Cc + T + len(cls))


def test_vq_attention_row_range():
    _vq("peaked", 2, 4096, 256, seed=5, rows=(64, 1216))
    RAN.add(("vq", "rows"))


# ------------------------------------------------------------------------------------------------ plan replay

def _plans():
    from oracle.make_golden_unetmodel import CASES
    from oracle.make_golden_windows import windows_config
    plans = {"realsr_denoiser_b16_64x64": plan_ops.SHIPPED["realsr_denoiser_b16_64x64"]}
    for name in ("w16_h32", "w8_h64", "w16_h64"):
        for hw in (64, 128):
            plans[f"{name}_b16_{hw}x{hw}"] = (lambda n=name, s=hw: plan_ops.swin_rows(windows_config(n)[0], 16, s, s))
    plans["w16_h64_variant_b16_64x64"] = lambda: plan_ops.swin_rows(windows_config("w16_h64_variant")[0], 16, 64, 64)
    for name in CASES:
        plans[f"unetmodel_{name}_b3"] = (lambda n=name: plan_ops.unetmodel_rows(n, *CASES[n][1:]))
    plans["unetmodel_legacy_b3_64x128"] = lambda: plan_ops.unetmodel_rows("legacy", 64, 128)
    plans["vq_f4_encode_1024"] = lambda: plan_ops.first_stage_rows("vq", "f4", 0, 1, 1024, 1024)
    return plans


def _plan_names():
    from oracle.make_golden_unetmodel import CASES
    return (["realsr_denoiser_b16_64x64"] + [f"{n}_b16_{s}x{s}" for n in ("w16_h32", "w8_h64", "w16_h64") for s in (64, 128)] +
            ["w16_h64_variant_b16_64x64"] + [f"unetmodel_{n}_b3" for n in CASES] +
            ["unetmodel_legacy_b3_64x128", "vq_f4_encode_1024"])


@pytest.mark.parametrize("plan", _plan_names() if torch.cuda.is_available() else [])
def test_plan_attention(plan):
    """Each distinct attention of a shipped plan (random weights) replayed through the entries with the plan's
    configuration, on randn and peaked operands: the entry reports the plan's heads per CTA or persistent grid, and the
    result is within the float64 bound."""
    rows = _plans()[plan]()
    attn, swin = plan_ops.distinct(rows, "attn"), plan_ops.distinct(rows, "swin_attn")
    unet, vq = plan_ops.distinct(rows, "unet_attn"), plan_ops.distinct(rows, "vq_attn")
    print(f"[plan] {plan}: {len(attn)} window, {len(swin)} fused Swin, {len(unet)} unet, {len(vq)} vq attentions")
    assert attn or swin or unet or vq
    for i, d in enumerate(attn):
        H, W, ws, shift, N, heads, hd, hpc, simt = map(int, d)
        assert not simt
        for cls in ("randn", "peaked"):
            L = WindowCase(cls, N, H // ws, W // ws, heads, ws, hd, shift, seed=i)
            _, info = _window(L, f"{plan} attn {d} {cls}", hpc=0)
            assert info["hpc"] == hpc, (d, info)
    for i, d in enumerate(swin):
        H, W, shift, grid, N, E, heads, slots = map(int, d)
        for cls in ("randn", "peaked"):
            L = SwinCase(cls, N, H, W, E, shift, slots, seed=i)
            y, pout, info = L.run(0)
            assert info["grid"] == grid, (d, info)
            _swin(L, f"{plan} swin_attn {d} {cls}")
    for i, d in enumerate(unet):
        T, heads, D, N = map(int, d[:4])
        for cls in ("randn", "peaked"):
            _unet(cls, N, T, heads, D, d[4] == "new", seed=i, tag=f"{plan} unet_attn {d} {cls}")
    for i, d in enumerate(vq):
        T, Cc, N = map(int, d)
        for cls in ("randn", "peaked"):
            _vq(cls, N, T, Cc, seed=i)
    RAN.add(("plan", plan))


# ------------------------------------------------------------------------------------------------ coverage

def test_coverage():
    """Across the module (run it whole): every instance ran, each with every input class it takes; heads per CTA of 1,
    a proper divisor and all heads; a CTA with several window pairs and a pair straddling images; every norm1 slot
    count.  Prints the worst observed ratio of error to allowance per kernel and input class."""
    if not RAN:
        pytest.skip("run with the rest of the module")
    for (kernel, cls), r in sorted(OBS.items()):
        print(f"[observed] {kernel:14s} {cls:10s} worst ratio {r:.3g}")
    kernels = [f"window<{ws},{hd}>" for ws, hd in INSTANCES] + ["window_simt", "swin<64>", "swin<192>", "unet<32>", "unet<64>",
                                                                 "unet<128>", "vq<128>", "vq<256>", "vq<512>"]
    missing = [k for k in kernels if ("instance", k) not in RAN]
    assert not missing, missing
    want = {k: (CLASSES if k.startswith("window") else ("randn", "peaked", "equal", "large")) for k in kernels}
    for k in ("swin<64>", "swin<192>"):
        want[k] = CLASSES + ("largemean",)
    gaps = [(k, c) for k, cs in want.items() for c in cs if ("class", k, c) not in RAN]
    assert not gaps, gaps
    gaps = [(ws, hd, h) for ws, hd in INSTANCES for h in ("1", "divisor", "all") if ("hpc", f"window<{ws},{hd}>", h) not in RAN]
    assert not gaps, gaps
    assert ("swin", "several pairs per CTA") in RAN and ("swin", "pair straddles images") in RAN
    assert {("slots", s) for s in SLOTS} <= RAN
