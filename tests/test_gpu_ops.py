"""GPU parity tests of the single operators, through the C ABI, against plain PyTorch fp32 on the same
fp16-rounded operands.  Tolerances: the kernels keep fp32 accumulators and round once to fp16 on store,
so the bound is one fp16 ulp of the result plus accumulation-order noise: |d| <= 2e-3 * max|ref| + 2e-3."""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from tests import gpu_util as G
    from resshift_b200 import _lib


def _tol(ref):
    return 2e-3 * ref.abs().max().item() + 2e-3


CONV_CASES = [
    # N, H, W, Cin, Cout, k, stride, bn
    (1, 8, 8, 64, 64, 1, 1, 0),          # one tile, one k-block
    (2, 16, 16, 64, 32, 1, 1, 0),
    (1, 16, 16, 128, 160, 1, 1, 0),      # N = 160 single UMMA
    (2, 16, 16, 160, 192, 1, 1, 0),      # Cin not a multiple of 64 (zero-filled tail)
    (1, 64, 64, 32, 32, 3, 1, 0),        # 3x3, bw=64
    (2, 32, 32, 64, 96, 3, 1, 0),        # 3x3, bw=32
    (3, 16, 16, 160, 320, 3, 1, 160),    # 2 channel tiles
    (3, 8, 8, 320, 640, 3, 1, 0),        # box spans 2 images, odd batch (masked rows)
    (2, 64, 64, 8, 160, 3, 1, 0),        # head conv: 8 (6 + pad) input channels
    (2, 64, 64, 160, 3, 3, 1, 0),        # out conv: 3 output channels
    (2, 32, 32, 64, 64, 3, 2, 0),        # stride 2 via parity views
    (1, 64, 64, 160, 160, 3, 2, 0),
    (16, 8, 8, 192, 576, 1, 1, 0),
]


# (parameter ids kept from the first GPU generation: "tcgen05_*" names the tensor-core kernel, today the wgmma one)
@pytest.mark.parametrize("impl", ["tcgen05_cg1", "tcgen05_cg2", "tcgen05_msub2", "tcgen05_persist_cg1", "tcgen05_persist_cg2", "simt"])
@pytest.mark.parametrize("case", CONV_CASES)
def test_conv2d(case, impl):
    N, H, W, Ci, Co, k, s, bn = case
    os.environ["RS_CONV_IMPL"] = impl.split("_")[0]
    if impl.endswith("msub2"):
        os.environ["RS_CONV_MSUB"] = "2"       # two 128-pixel sub-tiles per CTA (falls back to 1 for odd tile counts)
        os.environ["RS_CONV_CG"] = "1"
    elif impl.endswith("cg1"):
        os.environ["RS_CONV_CG"] = "1"         # one CTA per 128-pixel tile
    elif impl.endswith("cg2"):
        os.environ["RS_CONV_CG"] = "2"         # CTA pairs: two 128-pixel tiles, each CTA loads half of B and multicasts it
    # persistent mode (one CTA / pair per SM walking several tiles) forced on; off
    # otherwise so that both kernels are covered whatever the cost model would pick
    os.environ["RS_CONV_PERSIST"] = "1" if "persist" in impl else "0"
    try:
        g = torch.Generator(device="cuda").manual_seed(hash(case) % 1000)
        x = G.nhwc16(torch.randn(N, Ci, H, W, device="cuda", generator=g))
        w = torch.randn(Co, Ci, k, k, device="cuda", generator=g) / (Ci * k * k) ** 0.5
        b = torch.randn(Co, device="cuda", generator=g)
        if Co % 8:          # the 3-channel model head writes fp32 NCHW (fp16 views need 16-byte rows)
            got = G.conv2d(x, w, b, stride=s, bn=bn, out_f32=True)
        else:
            got = G.nchw32(G.conv2d(x, w, b, stride=s, bn=bn))
        ref = G.ref_conv(x, w, b, stride=s)
        st = G.err_stats(got, ref)
        assert st["nan"] == 0 and st["max_abs"] <= _tol(ref), st
    finally:
        os.environ.pop("RS_CONV_IMPL", None)
        os.environ.pop("RS_CONV_MSUB", None)
        os.environ.pop("RS_CONV_CG", None)


@pytest.mark.parametrize("act", [1, 2])
def test_conv2d_epilogue(act):
    g = torch.Generator(device="cuda").manual_seed(5)
    x = G.nhwc16(torch.randn(2, 192, 16, 16, device="cuda", generator=g))
    w = torch.randn(192, 192, 1, 1, device="cuda", generator=g) / 192 ** 0.5
    b = torch.randn(192, device="cuda", generator=g)
    res = G.nhwc16(torch.randn(2, 192, 16, 16, device="cuda", generator=g))
    got = G.nchw32(G.conv2d(x, w, b, residual=res, act=act))
    ref = G.ref_conv(x, w, b, residual=res, act=act)
    st = G.err_stats(got, ref)
    assert st["nan"] == 0 and st["max_abs"] <= _tol(ref), st
    # fp32 NCHW output mode (the model head)
    got32 = G.conv2d(x, w, b, act=0, out_f32=True)
    ref32 = G.ref_conv(x, w, b)
    assert (got32 - ref32).abs().max().item() <= 1e-3 * ref32.abs().max().item() + 1e-4


def test_conv2d_channel_slices():
    """Reads a channel slice of a wider buffer and writes into a slice of another (concat-free skips)."""
    g = torch.Generator(device="cuda").manual_seed(6)
    buf = G.nhwc16(torch.randn(2, 320, 16, 16, device="cuda", generator=g))
    w = torch.randn(160, 160, 3, 3, device="cuda", generator=g) / (160 * 9) ** 0.5
    b = torch.randn(160, device="cuda", generator=g)
    obuf = torch.zeros(2, 16, 16, 480, dtype=torch.float16, device="cuda")
    G.conv2d(None, w, b, in_view=(buf, 160, 160), out_view=(obuf, 320))
    ref = G.ref_conv(buf[..., 160:].contiguous(), w, b)
    got = G.nchw32(obuf[..., 320:].contiguous())
    assert (got - ref).abs().max().item() <= _tol(ref)
    assert obuf[..., :320].abs().max().item() == 0.0


@pytest.mark.parametrize("msub", ["cg1", "cg1_msub2", "cg2"])
@pytest.mark.parametrize("case", [(2, 64, 64, 64, 160, 3), (3, 16, 16, 160, 320, 3), (3, 8, 8, 320, 640, 1), (5, 8, 8, 64, 32, 3)])
def test_conv2d_fused_groupnorm_statistics(case, msub):
    """The conv epilogue's per-(image, tile slot, channel) partial sums must add up to the sums of the stored fp16
    output, written at a channel offset of a wider statistics buffer (concat consumers), and be bit-reproducible."""
    import ctypes as C
    N, H, W, Ci, Co, k = case
    g = torch.Generator(device="cuda").manual_seed(sum(case))
    x = G.nhwc16(torch.randn(N, Ci, H, W, device="cuda", generator=g))
    w = torch.randn(Co, Ci, k, k, device="cuda", generator=g) / (Ci * k * k) ** 0.5
    b = torch.randn(Co, device="cuda", generator=g)
    res = G.nhwc16(torch.randn(N, Co, H, W, device="cuda", generator=g))
    wp, ipad = G.pack_weight(w)
    cstride, coff = Co + 32, 32
    outs, parts = [], []
    os.environ["RS_CONV_MSUB"] = "2" if msub.endswith("msub2") else "1"
    os.environ["RS_CONV_CG"] = "2" if msub.endswith("cg2") else "1"
    os.environ["RS_CONV_PERSIST"] = "1" if msub.startswith("persist") else "0"
    for rep in range(2):
        out = torch.empty(N, H, W, Co, dtype=torch.float16, device="cuda")
        part = torch.full((N * 64 * cstride * 2,), float("nan"), dtype=torch.float32, device="cuda")
        slots = C.c_int32()
        _lib.check(G.L.rs_op_conv2d_stats(x.data_ptr(), N, H, W, Ci, Ci, wp.data_ptr(), ipad, b.data_ptr(), Co, k, 1,
                                          res.data_ptr(), Co, out.data_ptr(), Co, 0, 0, part.data_ptr(), cstride, coff,
                                          C.byref(slots), None, None, 0, G.stream()))
        torch.cuda.synchronize()
        outs.append(out)
        parts.append(part[:N * slots.value * cstride * 2].view(N, slots.value, cstride, 2)[:, :, coff:coff + Co].clone())
    os.environ.pop("RS_CONV_MSUB", None)
    os.environ.pop("RS_CONV_CG", None)
    os.environ.pop("RS_CONV_PERSIST", None)
    assert torch.equal(outs[0], outs[1]) and torch.equal(parts[0], parts[1])         # deterministic
    ref = G.ref_conv(x, w, b, residual=res)
    assert (G.nchw32(outs[0]) - ref).abs().max().item() <= _tol(ref)
    assert not torch.isnan(parts[0]).any()
    mean_c, var_c = _combine_pairs(parts[0], H * W)
    of = outs[0].float()
    assert (mean_c - of.mean(dim=(1, 2))).abs().max().item() <= 1e-5 * (1 + of.abs().max().item())
    v_ref = of.var(dim=(1, 2), unbiased=False)
    assert ((var_c - v_ref).abs() / (v_ref + 1e-6)).max().item() <= 1e-4


def _combine_pairs(pairs, hw):
    """(mean, M2) pairs [N, slots, C, 2] of equal-count slots -> per-(image, channel) mean and biased variance
    (Chan et al.), the same combine the kernels' finaliser does per group."""
    m, q = pairs[..., 0].double(), pairs[..., 1].double()
    ns = hw / pairs.shape[1]
    mean_c = m.mean(dim=1)
    m2 = q.sum(dim=1) + ns * ((m - mean_c[:, None]) ** 2).sum(dim=1)
    return mean_c.float(), (m2 / hw).float()


@pytest.mark.parametrize("variant", ["cg1", "cg2", "persist_cg2", "splitk_global", "splitk_cluster"])
@pytest.mark.parametrize("case", [(16, 64, 64, 64, 160, 3, 30.0), (3, 16, 16, 160, 320, 3, 0.5), (16, 8, 8, 320, 640, 3, -30.0),
                                  (5, 8, 8, 64, 192, 1, 30.0)])
def test_conv_statistics_finalised_by_last_cta(case, variant):
    """Producer -> consumer GroupNorm without a statistics pass: the conv epilogue delivers (mean, M2) pairs, the last CTA
    to finish an image writes gstat[N][32] = (mean, rstd), rs_op_groupnorm_apply consumes it.  Checked against
    F.group_norm (fp32) of the STORED fp16 conv output, including channels whose mean (conv bias +-30) dwarfs their
    spread — the case a single-pass E[x^2] - mean^2 loses.  reference: GroupNorm32, models/basic_ops.py:15-17."""
    import ctypes as C
    N, H, W, Ci, Co, k, bias_mean = case
    if variant.startswith("splitk") and H > 16:
        pytest.skip("split-K is for the few-tile layers")
    if variant == "persist_cg2" and N * H * W < 128 * 4:
        pytest.skip("too few tiles for a persistent pair")
    g = torch.Generator(device="cuda").manual_seed(sum(int(abs(v)) for v in case))
    x = G.nhwc16(torch.randn(N, Ci, H, W, device="cuda", generator=g))
    w = torch.randn(Co, Ci, k, k, device="cuda", generator=g) / (Ci * k * k) ** 0.5 * 0.5
    b = torch.randn(Co, device="cuda", generator=g) * 0.2 + bias_mean
    wp, ipad = G.pack_weight(w)
    gamma = 1 + 0.2 * torch.randn(Co, device="cuda", generator=g)
    beta = 0.2 * torch.randn(Co, device="cuda", generator=g)
    env = {"cg1": {"RS_CONV_CG": "1", "RS_CONV_PERSIST": "0"}, "cg2": {"RS_CONV_CG": "2", "RS_CONV_PERSIST": "0"},
           "persist_cg2": {"RS_CONV_CG": "2", "RS_CONV_PERSIST": "1"},
           "splitk_global": {"RS_CONV_SPLITK": "2", "RS_CONV_SPLITK_MODE": "global"},
           "splitk_cluster": {"RS_CONV_SPLITK": "2", "RS_CONV_SPLITK_MODE": "cluster"}}[variant]
    os.environ.update(env)
    try:
        results = []
        for rep in range(2):
            out = torch.full((N, H, W, Co), float("nan"), dtype=torch.float16, device="cuda")
            part = torch.full((N * 64 * Co * 2,), float("nan"), dtype=torch.float32, device="cuda")
            gstat = torch.full((N, 32, 2), float("nan"), dtype=torch.float32, device="cuda")
            counter = torch.zeros(N, dtype=torch.int32, device="cuda")
            if variant.startswith("splitk"):
                scratch = torch.empty(8 * N * H * W * Co, dtype=torch.float32, device="cuda")
                S = C.c_int32()
                _lib.check(G.L.rs_op_conv2d_splitk(x.data_ptr(), N, H, W, Ci, Ci, wp.data_ptr(), ipad, b.data_ptr(), Co, k, 1,
                                                   None, 0, out.data_ptr(), Co, 0, part.data_ptr(), Co, 0, scratch.data_ptr(),
                                                   C.byref(S), gstat.data_ptr(), counter.data_ptr(), G.stream()))
            else:
                slots = C.c_int32()
                _lib.check(G.L.rs_op_conv2d_stats(x.data_ptr(), N, H, W, Ci, Ci, wp.data_ptr(), ipad, b.data_ptr(), Co, k, 1,
                                                  None, 0, out.data_ptr(), Co, 0, 0, part.data_ptr(), Co, 0, C.byref(slots),
                                                  gstat.data_ptr(), counter.data_ptr(), 0, G.stream()))
            y = torch.empty_like(out)
            _lib.check(G.L.rs_op_groupnorm_apply(out.data_ptr(), N, H, W, Co, Co, gamma.data_ptr(), beta.data_ptr(), None, 0, 0,
                                                 y.data_ptr(), Co, gstat.data_ptr(), G.stream()))
            # the consumer-side combine of the same pairs (what the denoiser's small maps use) must agree with it
            y2 = torch.empty_like(out)
            _lib.check(G.L.rs_op_groupnorm_apply_pairs(out.data_ptr(), N, H, W, Co, Co, gamma.data_ptr(), beta.data_ptr(), None, 0, 0,
                                                       y2.data_ptr(), Co, part.data_ptr(), max(1, H * W // 128), G.stream()))
            # ... and so must the stand-alone finalisation kernel (what the first-stage plans run for many-slot tensors)
            gstat3 = torch.full((N, 32, 2), float("nan"), dtype=torch.float32, device="cuda")
            nsl = max(1, H * W // 128)
            _lib.check(G.L.rs_op_groupnorm_finalize(part.data_ptr(), N, nsl, Co, H * W // nsl, 0.0, gstat3.data_ptr(), G.stream()))
            torch.cuda.synchronize()
            assert (y2.float() - y.float()).abs().max().item() <= 2e-3 * (1 + y.float().abs().max().item())
            assert not torch.isnan(gstat3).any()
            assert ((gstat3 - gstat).abs() <= 1e-4 * (1 + gstat.abs())).all(), (gstat3 - gstat).abs().max().item()
            results.append((out, gstat.clone(), y))
    finally:
        for kk in env:
            os.environ.pop(kk, None)
    out, gstat, y = results[0]
    assert torch.equal(gstat, results[1][1]) and torch.equal(y, results[1][2])           # deterministic whoever arrives last
    assert not torch.isnan(gstat).any()
    of = G.nchw32(out)                                                                  # [N, Co, H, W] fp32 of the stored values
    grp = of.reshape(N, 32, -1).double()
    mean_ref, var_ref = grp.mean(dim=2), grp.var(dim=2, unbiased=False)
    rstd_ref = 1.0 / torch.sqrt(var_ref + 1e-5)
    assert (gstat[..., 0].double() - mean_ref).abs().max().item() <= 1e-5 * (1 + mean_ref.abs().max().item())
    assert ((gstat[..., 1].double() - rstd_ref).abs() / rstd_ref).max().item() <= 2e-4
    ref = F.group_norm(of, 32, gamma, beta, eps=1e-5)
    st = G.err_stats(G.nchw32(y), ref)
    print(f"[gn fused] {variant} {case}: {st}")
    assert st["nan"] == 0 and st["max_abs"] <= _tol(ref), st


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("case", [(16, 64, 64, 160, 160, 3), (16, 64, 64, 192, 576, 1), (5, 64, 64, 96, 320, 3), (16, 32, 32, 64, 64, 3)])
def test_conv2d_persistent_matches_one_tile_per_cta(case, cg):
    """Many tiles per SM: the persistent kernel (tiles strided over one CTA / CTA pair per SM, TMEM double buffering,
    epilogue overlapped with the next tile's main loop) must give bit-identical outputs and GroupNorm partials to the
    one-tile-per-CTA kernel (same accumulation order), with a residual input and fused statistics."""
    import ctypes as C
    N, H, W, Ci, Co, k = case
    g = torch.Generator(device="cuda").manual_seed(sum(case))
    x = G.nhwc16(torch.randn(N, Ci, H, W, device="cuda", generator=g))
    w = torch.randn(Co, Ci, k, k, device="cuda", generator=g) / (Ci * k * k) ** 0.5
    b = torch.randn(Co, device="cuda", generator=g)
    res = G.nhwc16(torch.randn(N, Co, H, W, device="cuda", generator=g))
    wp, ipad = G.pack_weight(w)
    outs, parts = [], []
    os.environ["RS_CONV_CG"] = str(cg)
    try:
        for persist in (0, 1, 1):
            os.environ["RS_CONV_PERSIST"] = str(persist)
            out = torch.full((N, H, W, Co), float("nan"), dtype=torch.float16, device="cuda")
            part = torch.full((N * 64 * Co * 2,), float("nan"), dtype=torch.float32, device="cuda")
            slots = C.c_int32()
            _lib.check(G.L.rs_op_conv2d_stats(x.data_ptr(), N, H, W, Ci, Ci, wp.data_ptr(), ipad, b.data_ptr(), Co, k, 1,
                                              res.data_ptr(), Co, out.data_ptr(), Co, 0, 0, part.data_ptr(), Co, 0,
                                              C.byref(slots), None, None, 0, G.stream()))
            torch.cuda.synchronize()
            outs.append(out)
            parts.append(part[:N * slots.value * Co * 2].clone())
    finally:
        os.environ.pop("RS_CONV_CG", None)
        os.environ.pop("RS_CONV_PERSIST", None)
    assert not torch.isnan(outs[1].float()).any() and not torch.isnan(parts[1]).any()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2])
    assert torch.equal(parts[0], parts[1]) and torch.equal(parts[1], parts[2])
    ref = G.ref_conv(x, w, b, residual=res)
    assert (G.nchw32(outs[1]) - ref).abs().max().item() <= _tol(ref)


@pytest.mark.parametrize("mode", ["global", "cluster"])
@pytest.mark.parametrize("force", [0, 2, 4])
@pytest.mark.parametrize("case", [(16, 8, 8, 640, 640, 3), (3, 16, 16, 320, 320, 3), (5, 8, 8, 192, 192, 1), (2, 16, 16, 960, 320, 3)])
def test_conv2d_split_k(case, force, mode):
    """Layers with few output tiles split their K loop over several CTAs (pairs).  `global`: fp32 partial sums go to a
    scratch buffer and the reduce kernel combines them in a fixed order, applies bias / residual and emits the GroupNorm
    partial statistics.  `cluster`: the K ranges of a tile form one thread-block cluster, keep their partial tiles in
    shared memory and finish the layer themselves through distributed shared memory (no scratch, no second kernel)."""
    import ctypes as C
    if mode == "cluster" and force == 4:
        pytest.skip("cluster split-K is limited to two K ranges (clusters of 4 CTAs)")
    N, H, W, Ci, Co, k = case
    g = torch.Generator(device="cuda").manual_seed(sum(case))
    x = G.nhwc16(torch.randn(N, Ci, H, W, device="cuda", generator=g))
    w = torch.randn(Co, Ci, k, k, device="cuda", generator=g) / (Ci * k * k) ** 0.5
    b = torch.randn(Co, device="cuda", generator=g)
    res = G.nhwc16(torch.randn(N, Co, H, W, device="cuda", generator=g))
    wp, ipad = G.pack_weight(w)
    scratch = torch.empty(8 * N * H * W * Co, dtype=torch.float32, device="cuda")
    if force:
        os.environ["RS_CONV_SPLITK"] = str(force)
    os.environ["RS_CONV_SPLITK_MODE"] = mode
    try:
        outs, parts, used = [], [], []
        for rep in range(2):
            out = torch.full((N, H, W, Co), float("nan"), dtype=torch.float16, device="cuda")
            part = torch.full((N * 64 * Co * 2,), float("nan"), dtype=torch.float32, device="cuda")
            S = C.c_int32()
            _lib.check(G.L.rs_op_conv2d_splitk(x.data_ptr(), N, H, W, Ci, Ci, wp.data_ptr(), ipad, b.data_ptr(), Co, k, 1,
                                               res.data_ptr(), Co, out.data_ptr(), Co, 0, part.data_ptr(), Co, 0,
                                               scratch.data_ptr(), C.byref(S), None, None, G.stream()))
            torch.cuda.synchronize()
            outs.append(out); parts.append(part.clone()); used.append(S.value)
    finally:
        os.environ.pop("RS_CONV_SPLITK", None)
        os.environ.pop("RS_CONV_SPLITK_MODE", None)
    print(f"[split-k] case {case} forced {force} mode {mode}: S = {used[0]}")
    assert torch.equal(outs[0], outs[1]) and torch.equal(parts[0][~torch.isnan(parts[0])], parts[1][~torch.isnan(parts[1])])
    ref = G.ref_conv(x, w, b, residual=res)
    st = G.err_stats(G.nchw32(outs[0]), ref)
    assert st["nan"] == 0 and st["max_abs"] <= _tol(ref), st
    slots = max(1, H * W // 128)
    pv = parts[0][:N * slots * Co * 2].view(N, slots, Co, 2)
    of = outs[0].float()
    mean_c, var_c = _combine_pairs(pv, H * W)
    assert (mean_c - of.mean(dim=(1, 2))).abs().max().item() <= 1e-5 * (1 + of.abs().max().item())
    v_ref = of.var(dim=(1, 2), unbiased=False)
    assert ((var_c - v_ref).abs() / (v_ref + 1e-6)).max().item() <= 1e-4


@pytest.mark.parametrize("hsplit", [1, 2])
@pytest.mark.parametrize("case", [(2, 16, 16, 192, 768), (1, 64, 64, 64, 256), (3, 8, 8, 192, 768), (4, 32, 32, 192, 768)])
def test_fused_mlp(case, hsplit, monkeypatch):
    """out = residual + fc2(GELU(fc1(x))) in one kernel (hidden activations stay on chip, rounded to fp16 like the
    unfused path rounds its stored intermediate).  RS_MLP_HSPLIT is set both ways: the kernel has no hidden-dimension
    split, so the results must not depend on it."""
    monkeypatch.setenv("RS_MLP_HSPLIT", str(hsplit))
    N, H, W, E, Hd = case
    g = torch.Generator(device="cuda").manual_seed(sum(case))
    x = G.nhwc16(torch.randn(N, E, H, W, device="cuda", generator=g))
    res = G.nhwc16(torch.randn(N, E, H, W, device="cuda", generator=g))
    w1 = torch.randn(Hd, E, device="cuda", generator=g) / E ** 0.5
    b1 = torch.randn(Hd, device="cuda", generator=g) * 0.5
    w2 = torch.randn(E, Hd, device="cuda", generator=g) / Hd ** 0.5
    b2 = torch.randn(E, device="cuda", generator=g) * 0.5
    w1p, _ = G.pack_weight(w1)
    w2p, _ = G.pack_weight(w2)
    outs = []
    for _ in range(2):
        out = torch.full((N, H, W, E), float("nan"), dtype=torch.float16, device="cuda")
        _lib.check(G.L.rs_op_mlp(x.data_ptr(), N, H, W, E, Hd, w1p.data_ptr(), b1.data_ptr(), w2p.data_ptr(), b2.data_ptr(),
                                 res.data_ptr(), out.data_ptr(), None, G.stream()))
        torch.cuda.synchronize()
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    xf = x.float().reshape(-1, E)
    h = F.gelu(xf @ w1.half().float().T + b1).half().float()
    ref = (h @ w2.half().float().T + b2 + res.float().reshape(-1, E)).reshape(N, H, W, E)
    st = G.err_stats(outs[0], ref)
    assert st["nan"] == 0 and st["max_abs"] <= _tol(ref), st


@pytest.mark.parametrize("C,cfg", [(32, "plain"), (160, "silu"), (192, "plain"), (480, "film"), (1280, "film")])
def test_groupnorm(C, cfg):
    g = torch.Generator(device="cuda").manual_seed(C)
    N, H, W = 3, 16, 16
    x = G.nhwc16(torch.randn(N, C, H, W, device="cuda", generator=g) * 2 + 0.5)
    gamma = 1 + 0.2 * torch.randn(C, device="cuda", generator=g)
    beta = 0.2 * torch.randn(C, device="cuda", generator=g)
    film = torch.randn(N, 2 * C, device="cuda", generator=g) * 0.3 if cfg == "film" else None
    silu = int(cfg != "plain")
    y = torch.empty_like(x)
    scratch = torch.empty(G.L.rs_op_groupnorm_scratch_floats(N, H, W, C), dtype=torch.float32, device="cuda")
    _lib.check(G.L.rs_op_groupnorm(x.data_ptr(), N, H, W, C, C, gamma.data_ptr(), beta.data_ptr(), _lib.ptr(film),
                                   0 if film is None else 2 * C, silu, y.data_ptr(), C, scratch.data_ptr(), G.stream()))
    torch.cuda.synchronize()
    ref = F.group_norm(G.nchw32(x), 32, gamma, beta, eps=1e-5)
    if film is not None:
        ref = ref * (1 + film[:, :C, None, None]) + film[:, C:, None, None]
    if silu:
        ref = F.silu(ref)
    st = G.err_stats(G.nchw32(y), ref)
    assert st["nan"] == 0 and st["max_abs"] <= _tol(ref), st


@pytest.mark.parametrize("C,H", [(160, 64), (192, 16), (640, 8)])
def test_groupnorm_large_mean(C, H):
    """Stress case for the variance: per-group mean >> std (mean 30, std 0.5; fp16 storage of the input is part of the
    operand, so the fp32 reference sees the same rounded values).  A single-pass E[x^2] - mean^2 in fp32 loses the
    variance to cancellation here; the statistics are kept as (mean, M2) around local means instead.
    reference: GroupNorm32 = F.group_norm in fp32 (models/basic_ops.py:15-17)."""
    g = torch.Generator(device="cuda").manual_seed(C + H)
    N = 2
    x = G.nhwc16(torch.randn(N, C, H, H, device="cuda", generator=g) * 0.5 + 30.0)
    gamma = 1 + 0.2 * torch.randn(C, device="cuda", generator=g)
    beta = 0.2 * torch.randn(C, device="cuda", generator=g)
    y = torch.empty_like(x)
    scratch = torch.empty(G.L.rs_op_groupnorm_scratch_floats(N, H, H, C), dtype=torch.float32, device="cuda")
    _lib.check(G.L.rs_op_groupnorm(x.data_ptr(), N, H, H, C, C, gamma.data_ptr(), beta.data_ptr(), None, 0, 0,
                                   y.data_ptr(), C, scratch.data_ptr(), G.stream()))
    torch.cuda.synchronize()
    ref = F.group_norm(G.nchw32(x), 32, gamma, beta, eps=1e-5)
    st = G.err_stats(G.nchw32(y), ref)
    print(f"[groupnorm stress] C={C} H={H}: {st}")
    assert st["nan"] == 0 and st["max_abs"] <= _tol(ref), st


@pytest.mark.parametrize("impl", ["mma", "simt"])
@pytest.mark.parametrize("shift", [0, 4])
@pytest.mark.parametrize("hw", [(8, 8), (16, 32), (64, 64)])
def test_window_attention(hw, shift, impl):
    import sys
    from oracle import unet_oracle as uo
    from resshift_b200.arch import relative_position_index, shifted_window_mask
    H, W = hw
    if H == 8 and shift:
        pytest.skip("no shifted windows at a single-window resolution")
    heads, N = 6, 2
    E = heads * 32
    g = torch.Generator(device="cuda").manual_seed(H * 7 + shift)
    qkv = (torch.randn(N, H, W, 3 * E, device="cuda", generator=g)).half()
    table = torch.randn(225, heads, device="cuda", generator=g) * 0.5
    dense = torch.empty(heads * 64 * 64, dtype=torch.float32, device="cuda")
    _lib.check(G.L.rs_op_expand_relpos(table.data_ptr(), dense.data_ptr(), heads, G.stream()))
    out = torch.empty(N, H, W, E, dtype=torch.float16, device="cuda")
    os.environ["RS_ATTN_IMPL"] = impl
    try:
        _lib.check(G.L.rs_op_window_attention(qkv.data_ptr(), N, H, W, heads, shift, dense.data_ptr(), out.data_ptr(), G.stream()))
        torch.cuda.synchronize()
    finally:
        os.environ.pop("RS_ATTN_IMPL", None)
    # reference: roll / partition / attention core / reverse / roll, fp32 on CPU (oracle pieces)
    q = qkv.float().cpu()                                   # [N,H,W,3E]
    y = q.permute(0, 3, 1, 2)
    if shift:
        y = torch.roll(y, (-shift, -shift), (2, 3))
    yw = y.reshape(N, 3 * E, H // 8, 8, W // 8, 8).permute(0, 2, 4, 3, 5, 1).reshape(-1, 64, 3, heads, 32)
    qq, kk, vv = (yw[:, :, i].transpose(1, 2) for i in range(3))
    attn = (qq * 32 ** -0.5) @ kk.transpose(-2, -1)
    idx = relative_position_index(8).reshape(-1)
    attn = attn + table.cpu()[idx].view(64, 64, heads).permute(2, 0, 1)[None]
    if shift:
        m = shifted_window_mask(H, W, 8, shift)
        nw = m.shape[0]
        attn = (attn.view(-1, nw, heads, 64, 64) + m[None, :, None]).view(-1, heads, 64, 64)
    o = (attn.softmax(-1) @ vv).transpose(1, 2).reshape(-1, 64, E)
    o = o.view(N, H // 8, W // 8, 8, 8, E).permute(0, 5, 1, 3, 2, 4).reshape(N, E, H, W)
    if shift:
        o = torch.roll(o, (shift, shift), (2, 3))
    ref = o.permute(0, 2, 3, 1)
    st = G.err_stats(out.cpu(), ref)
    assert st["nan"] == 0 and st["max_abs"] <= 4e-3 * ref.abs().max().item() + 2e-3, st


# impl "tc": the kernel also delivers the group statistics of y; "mma": window pairs only (ids kept from the first GPU
# generation, where they named two kernels; both run the mma.sync fused kernel now)
@pytest.mark.parametrize("impl", ["tc", "mma"])
@pytest.mark.parametrize("E", [192, 64])
@pytest.mark.parametrize("case", [(2, 16, 32, 0), (2, 16, 32, 4), (3, 8, 8, 0), (1, 64, 64, 4), (5, 16, 16, 4), (16, 64, 64, 4)])
def test_swin_attention_half_fused(case, E, impl):
    """norm1 + qkv + (shifted-)window attention + proj + residual as ONE kernel against plain torch on the same fp16
    operands, with the intermediate roundings of the unfused path (fp16 n1 / qkv / attention output); also the
    (mean, M2) pairs of the result per 8x8 window.  reference: models/swin_transformer.py:246-275,114-145.
    The last case is the benchmark shape: 512 window pairs on 132 persistent CTAs, i.e. several tiles per CTA with the
    image changing inside a CTA's range (state carried from tile to tile: norm1 affine, weight ring, barrier phases)."""
    from resshift_b200.arch import relative_position_index, shifted_window_mask
    if case[0] == 16 and E == 64:
        pytest.skip("the multi-tile case is covered at the model's width")
    N, H, W, shift = case
    heads = E // 32
    g = torch.Generator(device="cuda").manual_seed(E + H * 3 + shift + N)
    x = (torch.randn(N, H, W, E, device="cuda", generator=g) * 1.5 + 0.3).half()
    gamma = 1 + 0.2 * torch.randn(E, device="cuda", generator=g)
    beta = 0.2 * torch.randn(E, device="cuda", generator=g)
    wqkv = torch.randn(3 * E, E, device="cuda", generator=g) / E ** 0.5
    bqkv = torch.randn(3 * E, device="cuda", generator=g) * 0.1
    wproj = torch.randn(E, E, device="cuda", generator=g) / E ** 0.5 * 0.5
    bproj = torch.randn(E, device="cuda", generator=g) * 0.1
    table = torch.randn(225, heads, device="cuda", generator=g) * 0.5
    dense = torch.empty(heads * 64 * 64, dtype=torch.float32, device="cuda")
    _lib.check(G.L.rs_op_expand_relpos(table.data_ptr(), dense.data_ptr(), heads, G.stream()))
    # norm1 statistics as a producer would deliver them: (mean, M2) per (image, 128-pixel slot, channel); 8x8 maps have
    # one 64-pixel slot per image
    rows = 128 if H * W >= 128 else 64
    slots = H * W // rows
    xs = x.float().reshape(N, slots, rows, E)
    mean_s = xs.mean(dim=2)
    part = torch.stack([mean_s, ((xs - mean_s[:, :, None]) ** 2).sum(dim=2)], dim=-1).contiguous()
    wq_p, _ = G.pack_weight(wqkv)
    wp_p, _ = G.pack_weight(wproj)
    nW = (H // 8) * (W // 8)
    outs = []
    for rep in range(2):
        y = torch.full_like(x, float("nan"))
        pout = torch.full((N, nW, E, 2), float("nan"), dtype=torch.float32, device="cuda")
        # tc: the image's 32 group (mean, rstd) of y are also reduced from the window pairs
        gst = torch.full((N, 32, 2), float("nan"), dtype=torch.float32, device="cuda") if impl == "tc" else None
        cnt = torch.zeros(N, dtype=torch.int32, device="cuda") if impl == "tc" else None
        _lib.check(G.L.rs_op_swin_attn(x.data_ptr(), N, H, W, E, heads, shift, part.data_ptr(), slots, gamma.data_ptr(), beta.data_ptr(),
                                       wq_p.data_ptr(), bqkv.data_ptr(), dense.data_ptr(), wp_p.data_ptr(), bproj.data_ptr(),
                                       y.data_ptr(), pout.data_ptr(), gst.data_ptr() if gst is not None else None,
                                       cnt.data_ptr() if cnt is not None else None, G.stream()))
        torch.cuda.synchronize()
        outs.append((y, pout, gst))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert impl != "tc" or torch.equal(outs[0][2], outs[1][2])
    y, pout, gst = outs[0]
    # ---- reference (fp32 math on fp16-rounded operands, fp16 rounding where the unfused path stores) ----
    xc = x.float().cpu()
    xn = F.group_norm(xc.permute(0, 3, 1, 2), 32, gamma.cpu(), beta.cpu(), eps=1e-5).half().float()           # [N,E,H,W]
    qkv = F.conv2d(xn, wqkv.half().float().cpu()[:, :, None, None], bqkv.cpu()).half().float()               # [N,3E,H,W]
    if shift:
        qkv = torch.roll(qkv, (-shift, -shift), (2, 3))
    yw = qkv.reshape(N, 3 * E, H // 8, 8, W // 8, 8).permute(0, 2, 4, 3, 5, 1).reshape(-1, 64, 3, heads, 32)
    qq, kk, vv = (yw[:, :, i].transpose(1, 2) for i in range(3))
    attn = (qq * 32 ** -0.5) @ kk.transpose(-2, -1)
    idx = relative_position_index(8).reshape(-1)
    attn = attn + table.cpu()[idx].view(64, 64, heads).permute(2, 0, 1)[None]
    if shift:
        m = shifted_window_mask(H, W, 8, shift)
        attn = (attn.view(-1, m.shape[0], heads, 64, 64) + m[None, :, None]).view(-1, heads, 64, 64)
    o = (attn.softmax(-1) @ vv).transpose(1, 2).reshape(-1, 64, E)
    o = o.view(N, H // 8, W // 8, 8, 8, E).permute(0, 5, 1, 3, 2, 4).reshape(N, E, H, W)
    if shift:
        o = torch.roll(o, (shift, shift), (2, 3))
    o = o.half().float()
    ref = (F.conv2d(o, wproj.half().float().cpu()[:, :, None, None], bproj.cpu()) + xc.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    st = G.err_stats(y.cpu(), ref)
    print(f"[swin attn fused {impl}] E={E} {case}: {st}")
    assert st["nan"] == 0 and st["max_abs"] <= 4e-3 * ref.abs().max().item() + 4e-3, st
    # pairs of y per window (windows of the SHIFTED partition: statistics are over the same pixels the kernel owns)
    yy = y.float().cpu().permute(0, 3, 1, 2)
    if shift:
        yy = torch.roll(yy, (-shift, -shift), (2, 3))
    ywin = yy.reshape(N, E, H // 8, 8, W // 8, 8).permute(0, 2, 4, 1, 3, 5).reshape(N, nW, E, 64)
    m_ref = ywin.mean(dim=3)
    q_ref = ((ywin - m_ref[..., None]) ** 2).sum(dim=3)
    assert not torch.isnan(pout).any()
    assert (pout[..., 0].cpu() - m_ref).abs().max().item() <= 1e-4 * (1 + m_ref.abs().max().item())
    assert ((pout[..., 1].cpu() - q_ref).abs() / (q_ref + 1e-3)).max().item() <= 2e-3
    if gst is not None:
        # group statistics of the stored y per image: 32 groups of E / 32 channels over all pixels (biased variance, eps 1e-5)
        yg = y.float().cpu().permute(0, 3, 1, 2).reshape(N, 32, -1)
        m_g = yg.mean(dim=2)
        r_g = (yg.var(dim=2, unbiased=False) + 1e-5).rsqrt()
        assert not torch.isnan(gst).any()
        assert (gst[..., 0].cpu() - m_g).abs().max().item() <= 1e-4 * (1 + m_g.abs().max().item())
        assert ((gst[..., 1].cpu() - r_g).abs() / r_g).max().item() <= 2e-3


def test_upsample_and_p_sample():
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn(2, 8, 8, 64, device="cuda", generator=g).half()
    y = torch.empty(2, 16, 16, 64, dtype=torch.float16, device="cuda")
    _lib.check(G.L.rs_op_upsample2x(x.data_ptr(), 2, 8, 8, 64, y.data_ptr(), G.stream()))
    ref = F.interpolate(x.permute(0, 3, 1, 2).float(), scale_factor=2, mode="nearest").permute(0, 2, 3, 1).half()
    torch.cuda.synchronize()
    assert torch.equal(y, ref)
    a, b, n = (torch.randn(2, 3, 64, 64, device="cuda", generator=g) for _ in range(3))
    out = torch.empty_like(a)
    _lib.check(G.L.rs_p_sample(a.data_ptr(), b.data_ptr(), n.data_ptr(), out.data_ptr(), 0.8, 0.2, 0.5, 0, a.numel(), G.stream()))
    torch.cuda.synchronize()
    assert (out - (0.8 * a + 0.2 * b + 0.5 * n)).abs().max().item() < 1e-6
    _lib.check(G.L.rs_p_sample(a.data_ptr(), b.data_ptr(), n.data_ptr(), out.data_ptr(), 0.8, 0.2, 0.5, 1, a.numel(), G.stream()))
    torch.cuda.synchronize()
    assert (out - (0.8 * a + 0.2 * b)).abs().max().item() < 1e-6
