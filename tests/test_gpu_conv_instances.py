"""Every compiled instance of the implicit-GEMM conv (conv_gemm_sm90_kernel<BN, MS>), each epilogue form and geometry, and
every distinct conv the shipped plans run, through rs_op_conv2d_ex against a float64 reference on the fp16-rounded
operands.

Per element  |got - ref| <= 1/2 ulp16(ref) + KAPPA * mag,  mag = (|x| (*) |w|) (x 1.13 behind GELU / SiLU, their
steepest slope) + |bias| + |residual|: the first term is the one rounding of the stored fp16 value, the second the
tensor core's fp32 accumulation (and the fp32 epilogue) relative to the magnitudes that entered the output.  Each case
runs twice and must be bit-identical; the configuration the entry reports (info) must be the one requested, so a forced
instance cannot be replaced silently; GroupNorm statistics sinks are checked per (image, tile slot, channel)."""
import ctypes as C
import os
import re
from contextlib import contextmanager

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from tests import gpu_util as G
    from resshift_b200 import _lib

# channel-tile widths with a compiled kernel (conv_gemm.cuh kConvBNs); msub = 2 instances exist for BN <= 128
BNS = [16, 32, 48, 64, 80, 96, 128, 160, 192, 256]
# accumulation error allowance relative to mag: the largest (|got - ref| - 1/2 ulp16) / mag observed over every launch of
# this module on an H100 80GB HBM3 (700 W power limit) was 5.8e-7 (~2^-20.7, a 3x3 Cin = 640 conv of the denoiser plan);
# KAPPA is 6.6 times that
KAPPA = 2.0 ** -18
ACT_GAIN = 1.13
INFO_KEYS = ("grid", "BN", "msub", "stages", "cg", "splitk", "persist", "epi_bc", "bw", "bh", "box_n", "gn_slots")
_ENV = ("RS_CONV_CG", "RS_CONV_MSUB", "RS_CONV_PERSIST", "RS_CONV_SPLITK", "RS_CONV_EPI", "RS_CONV_IMPL", "RS_CONV_BN",
        "RS_CONV_OCC")
# forced modes: environment and the (cg, msub, persist) the entry must report; msub is required through rs_conv_args
MODES = {
    "one_tile": ({"RS_CONV_CG": 1, "RS_CONV_PERSIST": 0}, (1, 1, 0)),
    "pair": ({"RS_CONV_CG": 2, "RS_CONV_PERSIST": 0}, (2, 1, 0)),
    "msub2": ({"RS_CONV_CG": 1, "RS_CONV_PERSIST": 0}, (1, 2, 0)),
    "persistent": ({"RS_CONV_CG": 1, "RS_CONV_PERSIST": 1}, (1, 1, 1)),
    "persistent_pair": ({"RS_CONV_CG": 2, "RS_CONV_PERSIST": 1}, (2, 1, 1)),
}
COMBOS = set()      # (BN, msub, cg, persist, splitk, epilogue) launched by this module


@contextmanager
def conv_env(**kv):
    """Exactly the given conv overrides (other tests may leave some set)."""
    saved = {k: os.environ.pop(k, None) for k in _ENV}
    os.environ.update({k: str(v) for k, v in kv.items()})
    try:
        yield
    finally:
        for k in _ENV:
            os.environ.pop(k, None)
        os.environ.update({k: v for k, v in saved.items() if v is not None})


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _nan16(*shape):
    return torch.full(shape, float("nan"), dtype=torch.float16, device="cuda")


class Conv:
    """Random operands of one conv layer: fp16 NHWC input (optionally a channel slice of a wider buffer), fp32 OIHW
    weights and their packed fp16 form, bias (one row, or one row per image), residual."""

    def __init__(self, N, H, W, Cin, Cout, k, stride=1, pad_lo=1, act=0, bias="row", res=True, seed=0, x_ld=None, xc0=0,
                 res_ld=None, rc0=0, cin_pad=None):
        g = _gen(seed)
        self.N, self.H, self.W, self.Cin, self.Cout, self.k, self.stride, self.pad_lo, self.act = N, H, W, Cin, Cout, k, stride, pad_lo, act
        self.Ho, self.Wo = H // stride, W // stride
        cin_x = cin_pad or Cin                         # channels the kernel reads (zero padding beyond Cin)
        self.x_ld, self.xc0, self.cin_x = x_ld or (cin_x + 7) // 8 * 8, xc0, cin_x   # (rows of 16-byte multiples)
        self.xbuf = torch.randn(N, H, W, self.x_ld, device="cuda", generator=g).half()
        if cin_pad:
            self.xbuf[..., Cin:] = 0
        self.x = self.xbuf[..., xc0:xc0 + cin_x]
        self.w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5
        self.wp, self.ipad = G.pack_weight(self.w)
        self.bias_sN = 0
        if bias == "row":
            self.bbuf = torch.randn(Cout, device="cuda", generator=g) * 0.5
            self.brows = self.bbuf[None].expand(N, Cout)
        elif bias == "image":                          # one row per image, rows Cout + 8 apart
            self.bias_sN = Cout + 8
            self.bbuf = torch.randn(N, self.bias_sN, device="cuda", generator=g) * 0.5
            self.brows = self.bbuf[:, :Cout]
        else:
            self.bbuf, self.brows = None, None
        self.rbuf, self.rc0 = None, rc0
        if res:
            self.rbuf = torch.randn(N, self.Ho, self.Wo, res_ld or (Cout + 7) // 8 * 8, device="cuda", generator=g).half()
        self._ref = None

    @property
    def res(self):
        return None if self.rbuf is None else self.rbuf[..., self.rc0:self.rc0 + self.Cout]

    def run(self, bn=0, msub=0, out=None, oc0=0, out_f32=False, sinks=(), gstat=None, splitk=False):
        """One rs_op_conv2d_ex launch; returns (fp16 output slice or fp32 NCHW output, info dict)."""
        if out is None and not out_f32:
            out = _nan16(self.N, self.Ho, self.Wo, (self.Cout + 7) // 8 * 8)
        o32 = torch.full((self.N, self.Cout, self.Ho, self.Wo), float("nan"), device="cuda") if out_f32 else None
        a = _lib.ConvArgsC()
        a.x, a.N, a.H, a.W, a.C, a.ld = self.xbuf.data_ptr() + 2 * self.xc0, self.N, self.H, self.W, self.cin_x, self.x_ld
        a.w_packed, a.ipad = self.wp.data_ptr(), self.ipad
        a.bias, a.bias_sN = _lib.ptr(self.bbuf), self.bias_sN
        a.cout, a.ksize, a.stride, a.pad_lo = self.Cout, self.k, self.stride, self.pad_lo
        if self.rbuf is not None:
            a.residual, a.res_ld = self.rbuf.data_ptr() + 2 * self.rc0, self.rbuf.shape[-1]
        if out is not None:
            a.out, a.out_ld = out.data_ptr() + 2 * oc0, out.shape[-1]
        a.out_f32_nchw = _lib.ptr(o32)
        a.act, a.bn, a.msub = self.act, bn, msub
        for i, (part, cstride, coff) in enumerate(sinks):
            a.part[i], a.cstride[i], a.coff[i] = part.data_ptr(), cstride, coff
        a.gstat = _lib.ptr(gstat)
        scratch = torch.empty(8 * self.N * self.Ho * self.Wo * self.Cout, device="cuda") if splitk else None
        a.splitk_scratch = _lib.ptr(scratch)
        info = (C.c_int32 * 12)()
        _lib.check(_lib.lib.rs_op_conv2d_ex(C.byref(a), info, G.stream()))
        torch.cuda.synchronize()
        info = dict(zip(INFO_KEYS, list(info)))
        COMBOS.add((info["BN"], info["msub"], info["cg"], info["persist"], info["splitk"],
                    "f32" if out_f32 else ("direct" if info["epi_bc"] == 0 and info["splitk"] == 1 else
                                           ("reduce" if info["splitk"] > 1 else "staged"))))
        return (o32 if out_f32 else out[..., oc0:oc0 + self.Cout]), info

    def ref(self, rows=None):
        """float64 (output NHWC, mag NHWC) of the layer; with rows (a 1-D index tensor), of those output rows of every
        image only, each computed from the k input rows it reads (zero rows outside the map)."""
        if rows is None and self._ref is not None:
            return self._ref
        wq = self.w.half().double()
        pt = 0 if (self.stride == 2 and self.pad_lo == 0) else self.k // 2     # input rows / columns before the first
        if rows is None:
            x = self.x[..., :self.Cin].permute(0, 3, 1, 2).double()
        else:                                           # [N * R, Cin, k, W]: one k-row slab per output row
            idx = rows.to(self.x.device)[:, None] * self.stride - pt + torch.arange(self.k, device=self.x.device)
            keep = ((idx >= 0) & (idx < self.H)).double()
            x = self.x[:, idx.clamp(0, self.H - 1), :, :self.Cin].double() * keep[None, :, :, None, None]
            x = x.permute(0, 1, 4, 2, 3).reshape(-1, self.Cin, self.k, self.W)

        def conv(a, b):
            if self.stride == 2 and self.pad_lo == 0:          # the VQ-GAN Downsample: pad (0, 1, 0, 1), no conv padding
                return F.conv2d(F.pad(a, (0, 1, 0, 0 if rows is not None else 1)), b, stride=2)
            if rows is not None:
                return F.conv2d(F.pad(a, (pt, pt)), b, stride=self.stride)
            return F.conv2d(a, b, stride=self.stride, padding=self.k // 2)
        y, mag = conv(x, wq), conv(x.abs(), wq.abs())
        if rows is not None:                            # [N * R, Cout, 1, Wo] -> [N, Cout, R, Wo]
            y, mag = (t.reshape(self.N, -1, self.Cout, self.Wo).permute(0, 2, 1, 3) for t in (y, mag))
        if self.brows is not None:
            y = y + self.brows.double()[:, :, None, None]
            mag = mag + self.brows.double().abs()[:, :, None, None]
        if self.act == 1:
            y, mag = F.gelu(y), mag * ACT_GAIN
        elif self.act == 2:
            y, mag = F.silu(y), mag * ACT_GAIN
        if self.res is not None:
            r = (self.res if rows is None else self.res[:, rows.to(self.res.device)]).permute(0, 3, 1, 2).double()
            y, mag = y + r, mag + r.abs()
        out = (y.permute(0, 2, 3, 1), mag.permute(0, 2, 3, 1))
        if rows is None:
            self._ref = out
        return out

    def check(self, tag, got, f32=False, rows=None):
        """got against the float64 bound, on every element or on the output rows `rows` of every image."""
        ref, mag = self.ref(rows)
        if f32:
            got = got.permute(0, 2, 3, 1)
        if rows is not None:
            got = got[:, rows.to(got.device)]
        return G.assert_within(tag, got, ref, mag, KAPPA, fp16=not f32)


def _sinks(N, Cout, slots, spec=None):
    """Statistics sinks (cstride, coff) of NaN-filled buffers: by default two at different channel offsets of wider
    buffers."""
    spec = ((Cout + 16, 8), (Cout + 72, 40)) if spec is None else spec
    return [(torch.full((N * slots * cstride * 2 + 64,), float("nan"), device="cuda"), cstride, coff)
            for cstride, coff in spec]


def _box(Ho, Wo):
    """The 128-pixel box (bw, bh, images) of the launcher and the tile slots per image."""
    def p2(x, cap):
        p = 1
        while p * 2 <= cap and x % (p * 2) == 0:
            p *= 2
        return p
    bw = p2(Wo, 128)
    bh = p2(Ho, 128 // bw)
    return bw, bh, 128 // (bw * bh), (Wo // bw) * (Ho // bh)


def _run(tag, L, want=None, stats=True, rows=None, sink_spec=None, **kw):
    """Two launches of layer L: bit-identical outputs and statistics, info as wanted, output within the bound (on the
    output rows `rows` only, if given), the statistics of each sink against the stored output (in full).  Sinks: the
    (cstride, coff) of sink_spec, or two default ones where the launcher takes statistics (boxes of at most two images,
    fp16 output).  Returns (output, sink buffers, info)."""
    bw, bh, box_n, slots = _box(L.Ho, L.Wo)
    if sink_spec is None:
        sink_spec = None if stats and box_n <= 2 and not kw.get("out_f32") else ()
    runs = []
    for _ in range(2):
        sinks = _sinks(L.N, L.Cout, slots, sink_spec)
        out, info = L.run(sinks=sinks, **kw)
        runs.append((out.clone(), [(s[0].clone(), s[1], s[2]) for s in sinks], info))
    (out, sinks, info), (out2, sinks2, info2) = runs
    parts = [s[0] for s in sinks]
    assert info == info2
    assert torch.equal(G.bits(out), G.bits(out2)) and all(torch.equal(G.bits(a), G.bits(b[0])) for a, b in zip(parts, sinks2)), \
        f"{tag}: two launches differ"
    assert (info["bw"], info["bh"], info["box_n"], info["gn_slots"]) == (bw, bh, box_n, slots), info
    for k, v in (want or {}).items():
        assert info[k] == v, f"{tag}: launched {k} = {info[k]}, wanted {v} ({info})"
    L.check(f"{tag} {info}", out, f32=bool(kw.get("out_f32")), rows=rows)
    for i, (part, cstride, coff) in enumerate(sinks):
        G.check_slot_pairs(f"{tag} sink {i}", part, out, bw, bh, slots, cstride, coff)
    return out, parts, info


def _epi_bc(bn):
    return 64 if bn % 64 == 0 else (32 if bn % 32 == 0 else 16)


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
                                          "epi_bc": _epi_bc(bn)})
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
        staged, _ = L.run(bn=bn, msub=msub)
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
    if cg == 2 and _box(H, W)[3] * -(-N // box) < 2:
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
    obuf = _nan16(5, 32, 32, 264)
    with conv_env(**env):
        _run(f"channel slices {mode}", L, out=obuf, oc0=40)
    assert torch.isnan(obuf[..., :40].float()).all() and torch.isnan(obuf[..., 200:].float()).all()


# ---------------------------------------------------------------------------------------------- d. the shipped plans

_DESC = re.compile(r"conv(\d)x\d s(\d) (\d+)x(\d+) Cin=(\d+) Cout=(\d+) grid=(\d+) BN=(\d+) st=(\d+) \S* cg=(\d+) ms=(\d+) "
                   r"sk=(\d+) box=(\d+)x(\d+)x(\d+) N=(\d+) persist=(\d+) pad=(\d+) act=(\d+) res=(\d+) f32=(\d+)"
                   r"(?: silu=(\d) film=(\d) bsN=(\d+) sinks=(\d) cs=(\d+),(\d+) co=(\d+),(\d+) gstat=(\d)$)?")
_EPI_KEYS = ("silu", "film", "bsN", "sinks", "cs0", "cs1", "co0", "co1", "gstat")


def _conv_rows(rows, epilogue=False):
    """Distinct conv launches of an op list, as dicts of the description's fields; with epilogue, also of the fields
    that describe the epilogue (SiLU output, FiLM, per-image bias row stride, statistics sinks, gstat bits)."""
    keys = ("k", "s", "Ho", "Wo", "Cin", "Cout", "grid", "BN", "stages", "cg", "msub", "splitk", "bw", "bh", "box_n", "N",
            "persist", "pad", "act", "res", "f32") + _EPI_KEYS
    seen = {}
    for r in rows:
        if r.startswith("conv"):
            m = _DESC.match(r)
            assert m and (m.group(len(keys)) is not None or not epilogue), r
            d = dict(zip(keys, (None if v is None else int(v) for v in m.groups())))
            if not epilogue:
                d = {k: d[k] for k in keys if k not in _EPI_KEYS}
            seen.setdefault(tuple(d.values()), d)
    return list(seen.values())


def _desc_rows(fn, *args):
    cap, stride = 2048, 256
    ms = (C.c_double * cap)()
    desc = C.create_string_buffer(cap * stride)
    n = C.c_int32()
    _lib.check(fn(*args, ms, desc, stride, cap, C.byref(n), _lib.current_stream()))
    return [desc.raw[i * stride:(i + 1) * stride].split(b"\0")[0].decode() for i in range(n.value)]


def _denoiser_rows():
    from resshift_b200.config import preset
    from resshift_b200.models.unet import UNetModelSwin
    from resshift_b200.weights import random_state_dict
    ucfg, _ = preset("realsr")
    m = UNetModelSwin(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 0))
    m = m.cuda().eval()
    g = _gen(1)
    x = torch.randn(16, 3, 64, 64, device="cuda", generator=g)
    lq = torch.rand(16, 3, 64, 64, device="cuda", generator=g) * 2 - 1
    t = torch.full((16,), 7.0, device="cuda")
    m(x, t, lq=lq)
    plan = m.plan(16, 64, 64)
    return _desc_rows(_lib.lib.rs_plan_profile_ops, plan.handle, x.data_ptr(), t.data_ptr(), lq.data_ptr(), None)


def _first_stage_rows(kind, name, which, batch, h, w):
    from resshift_b200.models.autoencoder import AutoencoderKLTorch, VQModelTorch
    from resshift_b200.vq_arch import kl_preset, random_kl_state_dict, random_vq_state_dict, vq_preset
    cfg = (vq_preset if kind == "vq" else kl_preset)(name)
    sd = (random_vq_state_dict if kind == "vq" else random_kl_state_dict)(cfg, 0)
    m = (VQModelTorch if kind == "vq" else AutoencoderKLTorch)(**cfg.to_kwargs())
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    g = _gen(2)
    f = 2 ** (len(cfg.ch_mult) - 1)
    if which == 0:
        m.encode(torch.rand(batch, 3, h, w, device="cuda", generator=g) * 2 - 1)
    else:
        z = torch.randn(batch, cfg.embed_dim, h // f, w // f, device="cuda", generator=g) * 0.6
        m.decode(z, force_not_quantize=True) if kind == "vq" else m.decode(z)
    return _desc_rows(_lib.lib.rs_vq_profile_ops, m.plan(which, batch, h, w).handle)


PLANS = {
    "realsr_denoiser_b16_64x64": _denoiser_rows,
    "vq_f4_encode_256": lambda: _first_stage_rows("vq", "f4", 0, 1, 256, 256),
    "vq_f4_decode_256": lambda: _first_stage_rows("vq", "f4", 1, 1, 256, 256),
    "vq_f8_face_decode_512": lambda: _first_stage_rows("vq", "f8_face", 1, 1, 512, 512),
    "kl_tiny_encode": lambda: _first_stage_rows("kl", "tiny", 0, 2, 64, 96),
    "kl_tiny_decode": lambda: _first_stage_rows("kl", "tiny", 1, 2, 64, 96),
}


@pytest.mark.parametrize("plan", list(PLANS))
def test_plan_convs(plan):
    """Each distinct conv of a shipped plan (random weights), replayed once through rs_op_conv2d_ex: unforced, the entry
    picks the plan's configuration, and the result is within the float64 bound."""
    with conv_env():
        convs = _conv_rows(PLANS[plan]())
    assert convs
    print(f"[plan] {plan}: {len(convs)} distinct convs")
    for i, d in enumerate(convs):
        L = Conv(d["N"], d["Ho"] * d["s"], d["Wo"] * d["s"], d["Cin"], d["Cout"], d["k"], stride=d["s"], pad_lo=d["pad"],
                 act=d["act"], res=bool(d["res"]), seed=i)
        want = {k: d[k] for k in ("grid", "BN", "stages", "cg", "msub", "splitk", "persist", "bw", "bh", "box_n")}
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


