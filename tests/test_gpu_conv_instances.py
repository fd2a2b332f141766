"""Every compiled instance of the implicit-GEMM conv (conv_gemm_sm90_kernel<BN, MS>), each epilogue form and geometry, and
every distinct conv the shipped plans run, through rs_op_conv2d_ex against a float64 reference on the fp16-rounded
operands.

Per element  |got - ref| <= 1/2 ulp16(ref) + KAPPA * mag,  mag = (|x| (*) |w|) (x 1.13 behind GELU / SiLU, their
steepest slope) + |bias| + |residual|: the first term is the one rounding of the stored fp16 value, the second the
tensor core's fp32 accumulation (and the fp32 epilogue) relative to the magnitudes that entered the output.  Each case
runs twice and must be bit-identical; the configuration the entry reports (info) must be the one requested, so a forced
instance cannot be replaced silently; GroupNorm statistics sinks are checked per (image, tile slot, channel)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from tests import gpu_util as G
    from tests import plan_ops
    from tests.conv_ref import MODES, Conv, conv_env, epi_bc, run_conv
    from resshift_b200 import _lib

# channel-tile widths with a compiled kernel (conv_gemm.cuh kConvBNs); msub = 2 instances exist for BN <= 128
BNS = [16, 32, 48, 64, 80, 96, 128, 160, 192, 256]
COMBOS = set()      # (BN, msub, cg, persist, splitk, epilogue) launched by this module


def _ran(info, out_f32=False):
    COMBOS.add((info["BN"], info["msub"], info["cg"], info["persist"], info["splitk"],
                "f32" if out_f32 else ("direct" if info["epi_bc"] == 0 and info["splitk"] == 1 else
                                       ("reduce" if info["splitk"] > 1 else "staged"))))
    return info


def _run(tag, L, **kw):
    """conv_ref.run_conv, its launch recorded; returns (output, sink buffers, info)."""
    out, parts, info, _ = run_conv(tag, L, **kw)
    return out, parts, _ran(info, kw.get("out_f32"))


# ---------------------------------------------------------------------------------------------- a. instance matrix

# (N, H, W, Cin, k): a 3x3 layer whose Cin = 72 leaves a partial second k-chunk (6 tiles), and a 1x1 layer with more
# 128-pixel tiles (160) than the H100's 132 SMs, so that persistent CTAs (pairs) walk several tiles
LAYERS = {"3x3_n3_16x16_cin72": (3, 16, 16, 72, 3), "1x1_n5_64x64_cin136": (5, 64, 64, 136, 1)}


@pytest.mark.parametrize("cout_kind", ["cout_bn", "cout_2bn_plus_8"])
@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("layer", list(LAYERS))
def test_instance_matrix(layer, bn, cout_kind):
    """Forced channel tile x {one tile per CTA, CTA pair, two sub-tiles, persistent, persistent pair}, with bias, residual,
    GELU or SiLU and two statistics sinks.  Within one BN the modes share the accumulation order: bit-identical."""
    N, H, W, Cin, k = LAYERS[layer]
    Cout = bn if cout_kind == "cout_bn" else 2 * bn + 8        # the second form ends on a partial channel tile
    L = Conv(N, H, W, Cin, Cout, k, act=1 + BNS.index(bn) % 2, seed=bn + Cout + k)
    results = {}
    for mode, (env, (cg, msub, persist)) in MODES.items():
        if msub == 2 and bn > 128:
            continue                                           # not compiled: test_refusals
        with conv_env(**env):
            out, parts, info = _run(f"{layer} BN={bn} Cout={Cout} {mode}", L, bn=bn, msub=msub,
                                    want={"BN": bn, "cg": cg, "msub": msub, "persist": persist, "splitk": 1,
                                          "epi_bc": epi_bc(bn)})
        if persist:             # one CTA (pair) per SM (pair of SMs) at most, each walking units u, u + grid / cg, ...
            n_tiles = -(-((Cout + 15) // 16 * 16) // bn)
            units = -(-(N * H * W // 128) // cg) * n_tiles
            workers = torch.cuda.get_device_properties(0).multi_processor_count // cg
            assert info["grid"] == cg * min(units, workers), info
        results[mode] = (out, parts)
    base_out, base_parts = results["one_tile"]
    for mode, (out, parts) in results.items():
        assert torch.equal(G.bits(out), G.bits(base_out)), f"{mode} differs from one tile per CTA"
        assert all(torch.equal(G.bits(a), G.bits(b)) for a, b in zip(parts, base_parts)), f"{mode} statistics differ"


# ---------------------------------------------------------------------------------------------- b. epilogue forms

@pytest.mark.parametrize("mode", ["one_tile", "pair", "msub2"])
@pytest.mark.parametrize("bn", BNS)
def test_direct_epilogue(bn, mode):
    """RS_CONV_EPI=direct: per-thread stores instead of the staged TMA epilogue; the same arithmetic in the same order,
    so bit-identical to the staged epilogue."""
    env, (cg, msub, _) = MODES[mode]
    if msub == 2 and bn > 128:
        pytest.skip("no two-sub-tile instance")
    L = Conv(3, 16, 16, 72, 2 * bn + 8, 3, act=2, seed=bn)
    with conv_env(**env, RS_CONV_EPI="direct"):
        out, _, info = _run(f"direct BN={bn} {mode}", L, stats=False, bn=bn, msub=msub,
                            want={"BN": bn, "cg": cg, "msub": msub, "persist": 0, "epi_bc": 0})
    with conv_env(**env):
        staged, info = L.run(bn=bn, msub=msub)
    _ran(info)
    assert torch.equal(G.bits(out), G.bits(staged))


@pytest.mark.parametrize("cout", [3, 4, 8])
def test_fp32_nchw_head(cout):
    """The model head: fp32 NCHW output written by the direct epilogue (no fp16 rounding)."""
    L = Conv(2, 32, 32, 160, cout, 3, res=False, seed=cout)
    with conv_env():
        _run(f"f32 head Cout={cout}", L, out_f32=True, want={"epi_bc": 0, "persist": 0, "splitk": 1})


# images per 128-pixel box: 1 (16x16), 2 (8x8), 4 (8 rows x 4 columns) and 8 (4x4), odd batches
BIAS_BOXES = {1: (3, 16, 16), 2: (3, 8, 8), 4: (5, 8, 4), 8: (9, 4, 4)}


@pytest.mark.parametrize("mode", ["one_tile", "pair", "persistent"])
@pytest.mark.parametrize("box", list(BIAS_BOXES))
def test_per_image_bias(box, mode):
    """bias_sN > 0: every image of a box adds its own bias row (the scale-shift-off ResBlock folds emb_layers(emb) into
    the conv bias)."""
    N, H, W = BIAS_BOXES[box]
    env, (cg, msub, persist) = MODES[mode]
    L = Conv(N, H, W, 80, 48, 3, act=1, bias="image", seed=box)
    if cg == 2 and G.box128(H, W)[3] * -(-N // box) < 2:
        pytest.skip("a single tile cannot form a pair")
    with conv_env(**env):
        _run(f"per-image bias box={box} {mode}", L, want={"box_n": box, "cg": cg, "persist": persist, "msub": 1})


@pytest.mark.parametrize("S", [2, 3, 4, 6, 8])
def test_split_k(S):
    """Split-K (S CTAs per output tile, fp32 partials, the reduce kernel finishes) with per-image bias, SiLU, residual
    and two statistics sinks.  Cin = 392: 63 k-blocks, a partial last chunk."""
    L = Conv(3, 8, 8, 392, 104, 3, act=2, bias="image", seed=S)
    with conv_env(RS_CONV_SPLITK=S, RS_CONV_PERSIST=0):
        _run(f"split-K S={S}", L, splitk=True, want={"splitk": S, "epi_bc": 0, "persist": 0})


# ---------------------------------------------------------------------------------------------- c. geometry

GEOMETRIES = {"4x4": (9, 4, 4), "8x8": (3, 8, 8), "16x16": (2, 16, 16), "8x32": (3, 8, 32), "128x128": (1, 128, 128)}


@pytest.mark.parametrize("conv", ["s1", "s2_pad1", "s2_pad0"])
@pytest.mark.parametrize("geom", list(GEOMETRIES))
def test_geometry(geom, conv):
    """Output maps of 4x4 (eight images per box), 8x8 (two), 16x16, 8x32 and 128x128; stride 1, and stride 2 with
    padding 1 on every side (UNet Downsample) or pad (0, 1, 0, 1) (VQ-GAN Downsample)."""
    N, Ho, Wo = GEOMETRIES[geom]
    s = 1 if conv == "s1" else 2
    L = Conv(N, Ho * s, Wo * s, 72, 96, 3, stride=s, pad_lo=0 if conv == "s2_pad0" else 1, act=1, seed=Ho + Wo + s)
    with conv_env():
        _run(f"geometry {geom} {conv}", L)


def test_cin3_padded_to_8():
    """The denoiser's first conv: 3 input channels in an 8-channel zero-padded buffer, weights packed with Ipad = 8."""
    L = Conv(2, 32, 32, 3, 160, 3, cin_pad=8, seed=3)
    with conv_env():
        _run("Cin 3 padded to 8", L)


@pytest.mark.parametrize("mode", ["one_tile", "persistent"])
def test_channel_slices(mode):
    """Input, output and residual as channel slices of wider buffers at offsets that are multiples of 8 but not of 64;
    nothing outside the output slice is written."""
    env, _ = MODES[mode]
    L = Conv(5, 32, 32, 96, 160, 3, act=2, seed=11, x_ld=200, xc0=24, res_ld=176, rc0=8)
    obuf = G.nan16(5, 32, 32, 264)
    with conv_env(**env):
        _run(f"channel slices {mode}", L, out=obuf, oc0=40)
    assert torch.isnan(obuf[..., :40].float()).all() and torch.isnan(obuf[..., 200:].float()).all()


# ---------------------------------------------------------------------------------------------- d. the shipped plans

PLANS = ["realsr_denoiser_b16_64x64", "vq_f4_encode_256", "vq_f4_decode_256", "vq_f8_face_decode_512", "kl_tiny_encode",
         "kl_tiny_decode"]


@pytest.mark.parametrize("plan", PLANS)
def test_plan_convs(plan):
    """Each distinct conv of a shipped plan (random weights), replayed once through rs_op_conv2d_ex: unforced, the entry
    picks the plan's configuration, and the result is within the float64 bound."""
    with conv_env():
        convs = plan_ops.conv_rows(plan_ops.SHIPPED[plan]())
    assert convs
    print(f"[plan] {plan}: {len(convs)} distinct convs")
    for i, d in enumerate(convs):
        L = plan_ops.conv_of(d, seed=i)
        want = {k: d[k] for k in plan_ops.CONV_WANT}
        with conv_env():
            _run(f"{plan} {d}", L, stats=False, want=want, out_f32=bool(d["f32"]), splitk=d["splitk"] > 1)


# ---------------------------------------------------------------------------------------------- e. refusals

def test_refusals():
    """Instances that are not compiled, sub-tile counts a layer cannot take, and arguments outside the operator's domain
    are refused with a message; a required configuration is never replaced by another."""
    L = Conv(3, 16, 16, 72, 392, 3, seed=1)
    with conv_env(RS_CONV_CG=1, RS_CONV_PERSIST=0):
        for bn in (160, 192, 256):                             # no two-sub-tile instance of these widths
            with pytest.raises(_lib.RsError, match="2 sub-tiles per CTA"):
                L.run(bn=bn, msub=2)
        with pytest.raises(_lib.RsError, match="2 sub-tiles per CTA"):
            Conv(3, 16, 8, 72, 64, 3, seed=2).run(bn=64, msub=2)            # three 128-pixel tiles: an odd count
        with pytest.raises(_lib.RsError, match="2 sub-tiles per CTA"):
            Conv(2, 16, 16, 72, 64, 3, bias="image", seed=3).run(bn=64, msub=2)   # per-image bias rows
        with pytest.raises(_lib.RsError, match="msub must be"):
            L.run(msub=3)
    with conv_env():
        with pytest.raises(_lib.RsError, match="no valid tile configuration"):
            L.run(bn=112)                                      # not a compiled width
        L.pad_lo = 2
        with pytest.raises(_lib.RsError, match="pad_lo"):
            L.run()


def test_every_instance_ran():
    """The combinations launched by this module (printed for the record) include every instance conv_kernel_for can
    return, in each mode the launcher can give it."""
    if not COMBOS:
        pytest.skip("run with the rest of the module")
    for c in sorted(COMBOS):
        print("[combo] BN=%d msub=%d cg=%d persist=%d splitk=%d epilogue=%s" % c)
    ran = {(c[0], c[1]) for c in COMBOS}
    want = {(bn, 1) for bn in BNS} | {(bn, 2) for bn in BNS if bn <= 128}
    assert want <= ran, sorted(want - ran)
    for bn in BNS:
        for cg in (1, 2):
            for persist in (0, 1):
                assert (bn, 1, cg, persist, 1, "staged") in COMBOS, (bn, cg, persist)


