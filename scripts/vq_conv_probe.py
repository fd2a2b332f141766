"""Where does a 256x256 VQ-GAN conv layer spend its time?  Same layer (a) through the timeline entry (no statistics),
(b) with (mean, M2) pairs only, (c) finalised: the conv plus gn_finalize_kernel reducing the pairs to the 32 group
(mean, rstd) — each under the knobs in the environment (RS_CONV_PERSIST / RS_CONV_CG / ...).  A profiling aid, not a
benchmark."""
import ctypes as C
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch

from resshift_b200 import _lib
from tests import gpu_util as G
from scripts.conv_timeline import run as timeline

L = _lib.lib


def timed(fn, iters=10):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


def stats_variants(N, H, W, Ci, Co, k):
    x = torch.randn(N, H, W, Ci, device="cuda").half()
    w = torch.randn(Co, Ci, k, k, device="cuda") / (Ci * k * k) ** 0.5
    b = torch.randn(Co, device="cuda")
    wp, ipad = G.pack_weight(w)
    out = torch.empty(N, H, W, Co, dtype=torch.float16, device="cuda")
    slots_max = H * W // 128
    part = torch.empty(N * slots_max * Co * 2, dtype=torch.float32, device="cuda")
    gstat = torch.empty(N, 32, 2, dtype=torch.float32, device="cuda")
    slots = C.c_int32()
    st = G.stream()

    def pairs_only():
        _lib.check(L.rs_op_conv2d_stats(x.data_ptr(), N, H, W, Ci, Ci, wp.data_ptr(), ipad, b.data_ptr(), Co, k, 1, None, 0,
                                        out.data_ptr(), Co, 0, 0, part.data_ptr(), Co, 0, C.byref(slots), None, None, 0, st))

    def finalised():
        _lib.check(L.rs_op_conv2d_stats(x.data_ptr(), N, H, W, Ci, Ci, wp.data_ptr(), ipad, b.data_ptr(), Co, k, 1, None, 0,
                                        out.data_ptr(), Co, 0, 0, part.data_ptr(), Co, 0, C.byref(slots), gstat.data_ptr(),
                                        None, 0, st))
    fl = 2.0 * N * H * W * Co * Ci * k * k
    a = timed(pairs_only)
    bb = timed(finalised)
    print(f"    with (mean, M2) pairs: {a:8.1f} us ({fl / a / 1e6:7.1f} TFLOP/s) | + gn_finalize_kernel: {bb:8.1f} us")


if __name__ == "__main__":
    torch.manual_seed(0)
    for s in [(16, 256, 256, 128, 128, 3), (16, 256, 256, 8, 128, 3), (16, 128, 128, 256, 256, 3), (16, 256, 256, 256, 128, 1)]:
        timeline(*s, iters=5, tag=os.environ.get("TAG", "default"))
        stats_variants(*s)
