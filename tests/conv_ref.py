"""The implicit-GEMM conv (rs_op_conv2d_ex) as the GPU tests drive it: random layers, launches with every epilogue the
entry takes, and the float64 reference with its error model (test_gpu_conv_instances.py's module docstring)."""
import ctypes as C
import os
from contextlib import contextmanager

import torch
import torch.nn.functional as F

from resshift_b200 import _lib
from tests import gpu_util as G

# accumulation error allowance relative to mag: the largest (|got - ref| - 1/2 ulp16) / mag observed over every launch
# of test_gpu_conv_instances.py on an H100 80GB HBM3 (700 W power limit) was 5.8e-7 (~2^-20.7, a 3x3 Cin = 640 conv of
# the denoiser plan); KAPPA is 6.6 times that
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
SILU_C0 = 16            # the SiLU output is the channel slice [16, 16 + Cout) of a buffer 40 channels wider


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


def epi_bc(bn):
    return 64 if bn % 64 == 0 else (32 if bn % 32 == 0 else 16)


class Conv:
    """Random operands of one conv layer: fp16 NHWC input (optionally a channel slice of a wider buffer), fp32 OIHW
    weights and their packed fp16 form, bias (one row, or one row per image), residual."""

    def __init__(self, N, H, W, Cin, Cout, k, stride=1, pad_lo=1, act=0, bias="row", res=True, seed=0, x_ld=None, xc0=0,
                 res_ld=None, rc0=0, cin_pad=None):
        g = G.gen(seed)
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

    def run(self, bn=0, msub=0, out=None, oc0=0, out_f32=False, sinks=(), gstat=None, splitk=False, silu=None,
            film=None, film_sN=0):
        """One rs_op_conv2d_ex launch; returns (fp16 output slice or fp32 NCHW output, info dict).  silu: a buffer
        whose channels [SILU_C0, SILU_C0 + Cout) take the SiLU output; film: FiLM rows, film_sN apart (0: one shared
        row)."""
        if out is None and not out_f32:
            out = G.nan16(self.N, self.Ho, self.Wo, (self.Cout + 7) // 8 * 8)
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
        if silu is not None:
            a.silu_out, a.silu_ld = silu.data_ptr() + 2 * SILU_C0, silu.shape[-1]
        a.film, a.film_sN = _lib.ptr(film), film_sN
        info = (C.c_int32 * 12)()
        _lib.check(_lib.lib.rs_op_conv2d_ex(C.byref(a), info, G.stream()))
        torch.cuda.synchronize()
        return (o32 if out_f32 else out[..., oc0:oc0 + self.Cout]), dict(zip(INFO_KEYS, list(info)))

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
        """got against the float64 bound, on every element or on the output rows `rows` of every image; returns the
        ratio G.assert_within reports."""
        ref, mag = self.ref(rows)
        if f32:
            got = got.permute(0, 2, 3, 1)
        if rows is not None:
            got = got[:, rows.to(got.device)]
        return G.assert_within(tag, got, ref, mag, KAPPA, fp16=not f32)


def make_sinks(N, Cout, slots, spec=None):
    """Statistics sinks (cstride, coff) of NaN-filled buffers: by default two at different channel offsets of wider
    buffers."""
    spec = ((Cout + 16, 8), (Cout + 72, 40)) if spec is None else spec
    return [(torch.full((N * slots * cstride * 2 + 64,), float("nan"), device="cuda"), cstride, coff)
            for cstride, coff in spec]


def run_conv(tag, L, want=None, stats=True, rows=None, sink_spec=None, **kw):
    """Two launches of layer L: bit-identical outputs and statistics, info as wanted, output within the bound (on the
    output rows `rows` only, if given), the statistics of each sink against the stored output (in full).  Sinks: the
    (cstride, coff) of sink_spec, or two default ones where the launcher takes statistics (boxes of at most two images,
    fp16 output).  Returns (output, sink buffers, info, ratio of the bound check)."""
    bw, bh, box_n, slots = G.box128(L.Ho, L.Wo)
    if sink_spec is None:
        sink_spec = None if stats and box_n <= 2 and not kw.get("out_f32") else ()
    runs = []
    for _ in range(2):
        sinks = make_sinks(L.N, L.Cout, slots, sink_spec)
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
    ratio = L.check(f"{tag} {info}", out, f32=bool(kw.get("out_f32")), rows=rows)
    for i, (part, cstride, coff) in enumerate(sinks):
        G.check_slot_pairs(f"{tag} sink {i}", part, out, cstride, coff)
    return out, parts, info, ratio


# ---------------------------------------------------------------------------------------------- SiLU output and FiLM

def launch_silu(L, film, film_sN, **kw):
    """One launch of Conv L with the SiLU output (and FiLM rows); returns (out buffer, silu buffer, info)."""
    cw = (L.Cout + 7) // 8 * 8
    out, silu = G.nan16(L.N, L.Ho, L.Wo, cw + 8), G.nan16(L.N, L.Ho, L.Wo, cw + 40)
    _, info = L.run(out=out, silu=silu, film=film, film_sN=film_sN, **kw)
    return out, silu, info


def film_rows(L, form, seed):
    """None, one row per image ([N, 2 Cout + 8], rows 2 Cout + 8 apart) or one shared row (film_sN = 0)."""
    if form == "none":
        return None, 0, None
    g = G.gen(seed)
    sN = 2 * L.Cout + 8
    buf = torch.randn(L.N if form == "image" else 1, sN, device="cuda", generator=g) * 0.4
    rows = buf[:, :2 * L.Cout].expand(L.N, 2 * L.Cout).double()
    return buf, sN if form == "image" else 0, rows


def check_silu_film(tag, L, form, seed, want, **kw):
    """Two launches: bit-identical, the route wanted, out within the bound (FiLM: one more fp16 rounding before it), the
    SiLU output within one fp16 ulp of SiLU(out), NaN fills outside both views intact.  Returns (out, SiLU output,
    ratio of the bound check)."""
    film, sN, rows = film_rows(L, form, seed)
    runs = [launch_silu(L, film, sN, **kw) for _ in range(2)]
    (out, silu, info), (out2, silu2, info2) = runs
    assert info == info2 and torch.equal(G.bits(out), G.bits(out2)) and torch.equal(G.bits(silu), G.bits(silu2)), \
        f"{tag}: two launches differ"
    for k, v in want.items():
        assert (info[k] != 0 if v == "nonzero" else info[k] == v), f"{tag}: launched {k} = {info[k]}, wanted {v} ({info})"
    Co = L.Cout
    got, s = out[..., :Co], silu[..., SILU_C0:SILU_C0 + Co]
    ref, mag = L.ref()
    slack = None
    if rows is not None:
        one, sh = 1 + rows[:, None, None, :Co], rows[:, None, None, Co:]
        slack = 0.5 * G.ulp16(ref.abs() + KAPPA * mag) * one.abs()        # the fp16 rounding before the FiLM
        ref, mag = ref * one + sh, mag * one.abs() + sh.abs()
    ratio = G.assert_within(tag, got, ref, mag, KAPPA, slack=slack)
    sref = F.silu(got.double())
    assert ((s.double() - sref).abs() <= G.ulp16(sref)).all(), f"{tag}: SiLU output beyond one fp16 ulp of SiLU(out)"
    assert torch.isnan(out[..., Co:]).all(), f"{tag}: written beyond the output view"
    assert torch.isnan(silu[..., :SILU_C0]).all() and torch.isnan(silu[..., SILU_C0 + Co:]).all(), \
        f"{tag}: written outside the SiLU view"
    return got, s, ratio


def resample_case(N, H, W, Cc, pool):
    """rs_op_avgpool2x2 / rs_op_upsample2x_ex with the SiLU output against float64; without it, the same first output."""
    g = G.gen(H * W + Cc)
    x = (torch.randn(N, H, W, Cc, device="cuda", generator=g) * 3).half()
    Ho, Wo = (H // 2, W // 2) if pool else (2 * H, 2 * W)
    y, s = G.nan16(N, Ho, Wo, Cc), G.nan16(N, Ho, Wo, Cc)
    fn = _lib.lib.rs_op_avgpool2x2 if pool else _lib.lib.rs_op_upsample2x_ex
    _lib.check(fn(x.data_ptr(), N, H, W, Cc, y.data_ptr(), s.data_ptr(), G.stream()))
    torch.cuda.synchronize()
    xd = x.permute(0, 3, 1, 2).double()
    ref = (F.avg_pool2d(xd, 2) if pool else F.interpolate(xd, scale_factor=2, mode="nearest")).permute(0, 2, 3, 1)
    if pool:
        assert ((y.double() - ref).abs() <= 0.5 * G.ulp16(ref) + 2.0 ** -22 * ref.abs()).all()
    else:
        assert torch.equal(y.double(), ref)
    sref = F.silu(y.double())
    assert ((s.double() - sref).abs() <= G.ulp16(sref)).all()
    y2 = G.nan16(N, Ho, Wo, Cc)
    fn(x.data_ptr(), N, H, W, Cc, y2.data_ptr(), None, G.stream())     # without the second output: the same first one
    torch.cuda.synchronize()
    assert torch.equal(G.bits(y), G.bits(y2))
