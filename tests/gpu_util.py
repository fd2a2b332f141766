"""Helpers shared by the GPU parity tests (thin wrappers over the C ABI single-operator entry points)."""
import gc
import time
from contextlib import contextmanager

import pytest
import torch
import torch.nn.functional as F

from resshift_b200 import _lib

L = _lib.lib

# a denoiser forward against the fp32 oracle (test_gpu_unet.py's module docstring)
FWD_MAX, FWD_MEAN = 1e-2, 2.5e-3


def stream():
    return _lib.current_stream()


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def free():
    gc.collect()
    torch.cuda.empty_cache()


def note(obs, key, ratio):
    """obs[key] = the worst ratio seen so far."""
    obs[key] = max(obs.get(key, 0.0), float(ratio))


@pytest.fixture(scope="module", autouse=True)
def module_clock():
    """In a module that imports it: the time its first test started, the peak memory statistics reset then."""
    torch.cuda.reset_peak_memory_stats()
    return time.time()


def nan16(*shape):
    return torch.full(shape, float("nan"), dtype=torch.float16, device="cuda")


@contextmanager
def fp32_matmuls():
    """Exact fp32 matmuls / convolutions (TF32 off) for reference computations; restored afterwards."""
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def box128(H, W):
    """The conv launcher's 128-pixel box over an H x W output map: (bw, bh, images per box, tile slots per image)."""
    def p2(x, cap):
        p = 1
        while p * 2 <= cap and x % (p * 2) == 0:
            p *= 2
        return p
    bw = p2(W, 128)
    bh = p2(H, 128 // bw)
    return bw, bh, 128 // (bw * bh), (W // bw) * (H // bh)


def nhwc16(x_nchw: torch.Tensor) -> torch.Tensor:
    return x_nchw.permute(0, 2, 3, 1).contiguous().half()


def nchw32(x_nhwc: torch.Tensor) -> torch.Tensor:
    return x_nhwc.permute(0, 3, 1, 2).float().contiguous()


def pack_weight(w: torch.Tensor) -> tuple:
    """fp32 [O, I, kh, kw] (or [O, I]) on GPU -> packed fp16 [O][kh*kw][Ipad]."""
    if w.dim() == 2:
        w = w[:, :, None, None]
    O, I, KH, KW = w.shape
    ipad = (I + 7) // 8 * 8
    dst = torch.empty(O * KH * KW * ipad, dtype=torch.float16, device=w.device)
    _lib.check(L.rs_op_pack_conv_weight(w.contiguous().data_ptr(), dst.data_ptr(), O, I, KH, KW, ipad, stream()))
    return dst, ipad


def conv2d(x_nhwc, w, bias, stride=1, residual=None, act=0, out_f32=False, bn=0, in_view=None, out_view=None):
    """x_nhwc fp16 [N,H,W,C] (or a channel-slice view of a wider buffer given as (buffer, c0, C))."""
    if in_view is not None:
        buf, c0, Cc = in_view
        N, H, W, ld = buf.shape
        xptr = buf.data_ptr() + 2 * c0
    else:
        N, H, W, Cc = x_nhwc.shape
        ld = Cc
        xptr = x_nhwc.data_ptr()
    wp, ipad = pack_weight(w)
    O = w.shape[0]
    k = w.shape[-1] if w.dim() == 4 else 1
    Ho, Wo = H // stride, W // stride
    dev = w.device
    out = None
    out_ptr, out_ld = None, 0
    if out_view is not None:
        obuf, oc0 = out_view
        out_ptr, out_ld = obuf.data_ptr() + 2 * oc0, obuf.shape[-1]
    elif not out_f32:
        out = torch.full((N, Ho, Wo, O), float("nan"), dtype=torch.float16, device=dev)
        out_ptr, out_ld = out.data_ptr(), O
    o32 = torch.full((N, O, Ho, Wo), float("nan"), dtype=torch.float32, device=dev) if out_f32 else None
    _lib.check(L.rs_op_conv2d(xptr, N, H, W, Cc, ld, wp.data_ptr(), ipad, _lib.ptr(bias), O, k, stride,
                              _lib.ptr(residual), 0 if residual is None else residual.shape[-1], out_ptr, out_ld,
                              _lib.ptr(o32), act, bn, stream()))
    torch.cuda.synchronize()
    return o32 if out_f32 else out


def ref_conv(x_nhwc16, w, bias, stride=1, residual=None, act=0):
    """float64 torch reference (NCHW) on the fp16-rounded operands: no TF32, no fp32 accumulation error of its own."""
    x = nchw32(x_nhwc16).double()
    wq = w.half().double()
    if wq.dim() == 2:
        wq = wq[:, :, None, None]
    y = F.conv2d(x, wq, None if bias is None else bias.double(), stride=stride, padding=wq.shape[-1] // 2)
    if act == 1:
        y = F.gelu(y)
    elif act == 2:
        y = F.silu(y)
    if residual is not None:
        y = y + nchw32(residual).double()
    return y


def ulp16(v: torch.Tensor) -> torch.Tensor:
    """Spacing of fp16 numbers at |v| (float64; the subnormal spacing 2^-24 below 2^-14)."""
    e = torch.floor(torch.log2(v.double().abs().clamp(min=2.0 ** -14)))
    return torch.exp2(e - 10)


def accumulation_ratio(got, ref, mag, fp16=True, slack=None):
    """max over elements of (|got - ref| - rounding - slack) / mag: the accumulation error relative to the magnitudes that
    entered each output (rounding = half an fp16 ulp of the stored value, or one fp32 rounding for fp32 outputs)."""
    err = (got.double() - ref).abs()
    rnd = 0.5 * ulp16(ref) if fp16 else 2.0 ** -24 * ref.abs()
    if slack is not None:
        rnd = rnd + slack
    return ((err - rnd).clamp(min=0) / mag.clamp(min=1e-30)).max().item()


def assert_within(tag, got, ref, mag, kappa, slack=None, fp16=True):
    """|got - ref| <= 1/2 ulp16(ref) + kappa * mag (+ slack) per element; ulp taken at |ref| + the error allowance so that
    a value pushed across a power of two may round to the coarser spacing.  NaN fails."""
    allow = kappa * mag + (0 if slack is None else slack)
    err = (got.double() - ref).abs()
    rnd = 0.5 * ulp16(ref.abs() + allow) if fp16 else 2.0 ** -24 * (ref.abs() + allow)
    bad = ~(err <= rnd + allow)
    ratio = accumulation_ratio(got, ref, mag, fp16, slack)
    print(f"[bound] {tag}: max (|d| - rounding) / mag = {ratio:.3e}")
    assert not bad.any(), f"{tag}: {int(bad.sum())} of {bad.numel()} elements outside the bound (ratio {ratio:.3e})"
    return ratio


def check_slot_pairs(tag, part, out16, cstride, coff):
    """(mean, M2) pairs part[N][slots][cstride][2] of the stored fp16 output out16 [N, H, W, C] (slot = (bw x bh) box128
    of one image, row-major over the map) at channel offset coff, against float64 statistics of the same values; the
    bounds of test_gpu_ops.py's combined statistics.  Channels outside [coff, coff + C) must still hold their NaN fill."""
    N, H, W, Co = out16.shape
    bw, bh, _, slots = box128(H, W)
    o = out16.double()
    t = o.reshape(N, H // bh, bh, W // bw, bw, Co).permute(0, 1, 3, 2, 4, 5).reshape(N, slots, bh * bw, Co)
    mean = t.mean(dim=2)
    m2 = ((t - mean[:, :, None]) ** 2).sum(dim=2)
    p = part[:N * slots * cstride * 2].view(N, slots, cstride, 2)
    got = p[:, :, coff:coff + Co].double()
    assert torch.isfinite(got).all(), f"{tag}: missing statistics"
    rest = torch.cat([p[:, :, :coff], p[:, :, coff + Co:]], dim=2)
    assert torch.isnan(rest).all(), f"{tag}: statistics written outside the sink's channel slice"
    assert torch.isnan(part[N * slots * cstride * 2:]).all(), f"{tag}: statistics written beyond the slots"
    assert (got[..., 0] - mean).abs().max().item() <= 1e-5 * (1 + o.abs().max().item()), tag
    assert ((got[..., 1] - m2).abs() / (m2 + 1e-6 * bw * bh)).max().item() <= 1e-4, tag


def bits(t: torch.Tensor) -> torch.Tensor:
    """The raw bits of a float tensor (NaN fills compare equal)."""
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def err_stats(got: torch.Tensor, ref: torch.Tensor) -> dict:
    d = (got.float() - ref.float()).abs()
    return {"max_abs": d.max().item(), "mean_abs": d.mean().item(), "ref_absmax": ref.abs().max().item(),
            "ref_std": ref.float().std().item(), "nan": int(torch.isnan(got.float()).sum().item())}
