"""The fused Swin MLP (rs_op_mlp_ex) as the GPU tests drive it, and its float64 reference with the bound of
test_gpu_mlp_instances.py's module docstring."""
import ctypes as C

import torch
import torch.nn.functional as F

from resshift_b200 import _lib
from tests import gpu_util as G

# the conv tests' allowance (conv_ref.KAPPA: 6.6 times the largest ratio observed there).  On an H100 80GB HBM3 (700 W)
# no MLP output exceeded 1/2 ulp16 + slack at all: every deviation from the float64 reference was explained by hidden
# values rounded to the neighbouring fp16 number, so the slack term dominates this bound
KAPPA = 2.0 ** -18
ACT_GAIN = 1.13


def mlp(x, res, w1p, b1, w2p, b2, E, Hd, sinks=()):
    N, H, W, _ = x.shape
    out = torch.full_like(x, float("nan"))
    parts = (C.c_void_p * 2)(*[s[0].data_ptr() for s in sinks] + [None] * (2 - len(sinks)))
    cst = (C.c_int32 * 2)(*[s[1] for s in sinks] + [0] * (2 - len(sinks)))
    cof = (C.c_int32 * 2)(*[s[2] for s in sinks] + [0] * (2 - len(sinks)))
    slots_out = C.c_int32()
    _lib.check(_lib.lib.rs_op_mlp_ex(x.data_ptr(), N, H, W, E, Hd, w1p.data_ptr(), b1.data_ptr(), w2p.data_ptr(), b2.data_ptr(),
                                     _lib.ptr(res), out.data_ptr(), parts, cst, cof, C.byref(slots_out), G.stream()))
    torch.cuda.synchronize()
    return out, slots_out.value


def reference(xin, res, w1, b1, w2, b2):
    """float64 output, mag2 and slack (test_gpu_mlp_instances.py's module docstring) of the MLP on the fp16 input
    xin [M, E]."""
    x = xin.double()
    w1q, w2q = w1.half().double(), w2.half().double()
    pre = x @ w1q.T + b1.double()
    dh = KAPPA * ACT_GAIN * (x.abs() @ w1q.abs().T + b1.double().abs()) + 2.0 ** -21 * pre.abs()
    h64 = F.gelu(pre)
    h16 = h64.half()
    hc = h16.cpu()                                          # (fp16 nextafter on the CPU)
    inf = torch.full_like(hc, float("inf"))
    up, dn = (torch.nextafter(hc, s * inf).to(h16.device).double() for s in (1, -1))
    hq = h16.double()
    near = (h64 + dh >= 0.5 * (hq + up)) | (h64 - dh <= 0.5 * (hq + dn))
    e = torch.where(near, torch.maximum(up - hq, hq - dn), torch.zeros_like(hq))
    out = hq @ w2q.T + b2.double() + res.double()
    mag = hq.abs() @ w2q.abs().T + b2.double().abs() + res.double().abs()
    return out, mag, e @ w2q.abs().T
