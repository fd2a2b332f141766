"""Per-CTA timeline + throughput of the conv/GEMM kernel for the benchmark's dominant layer shapes.
Run on the GPU box; prints one block per (shape, knob setting).  A profiling aid, not a benchmark."""
import ctypes as C
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np
import torch

from resshift_b200 import _lib
from tests import gpu_util as G

L = _lib.lib


def run(N, H, W, Ci, Co, k, bn=0, iters=20, tag=""):
    x = torch.randn(N, H, W, Ci, device="cuda").half()
    w = torch.randn(Co, Ci, k, k, device="cuda") / (Ci * k * k) ** 0.5
    b = torch.randn(Co, device="cuda")
    wp, ipad = G.pack_weight(w)
    out = torch.empty(N, H, W, Co, dtype=torch.float16, device="cuda")
    info = (C.c_int32 * 7)()
    scratch = torch.empty(8 * N * H * W * Co, dtype=torch.float32, device="cuda") if os.environ.get("TL_SPLIT") else None
    dbg = torch.zeros(8 * 8192, dtype=torch.int64, device="cuda")
    st = _lib.current_stream()
    # warm-up + timed launches
    _lib.check(L.rs_op_conv2d_timeline(x.data_ptr(), N, H, W, Ci, Ci, wp.data_ptr(), ipad, b.data_ptr(), Co, k, 1,
                                       out.data_ptr(), Co, bn, 3, dbg.data_ptr(), info, _lib.ptr(scratch), st))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _lib.check(L.rs_op_conv2d_timeline(x.data_ptr(), N, H, W, Ci, Ci, wp.data_ptr(), ipad, b.data_ptr(), Co, k, 1,
                                       out.data_ptr(), Co, bn, iters, dbg.data_ptr(), info, _lib.ptr(scratch), st))
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    fl = 2.0 * N * H * W * Co * Ci * k * k
    grid = info[0]
    d = dbg[:grid * 8].view(grid, 8).cpu().numpy().astype(np.float64)
    t0 = d[:, 0].min()
    start, setup, first, mma_end, acc, done = [(d[:, i] - t0) / 1e3 for i in range(6)]
    epi_done = (d[:, 6] - t0) / 1e3
    kb = k * k * ((Ci + 63) // 64)
    print(f"--- {tag} N={N} {H}x{W} Cin={Ci} Cout={Co} k={k} | grid={grid} BN={info[1]} cg={info[4]} S={info[5]} stages={info[2]} smem={info[3]} kblocks={kb}")
    print(f"    {ms*1e3:8.1f} us/launch  {fl/ms/1e9:8.1f} TFLOP/s   kernel span {done.max():.1f} us")
    med = np.median
    lead = d[:, 2] > 0          # in pair mode only the leader CTA issues MMAs (and stamps slots 2, 3)
    staged = d[:, 6] > 0
    print(f"    per CTA (us, median): setup {med(setup-start):.2f} | wait first operands {med((first-setup)[lead]):.2f} | "
          f"mainloop {med((mma_end-first)[lead]):.2f} ({med((mma_end-first)[lead])/kb*1e3:.0f} ns/kblock) | "
          f"drain->acc {med((acc-mma_end)[lead]):.2f} | epilogue {med(done-acc):.2f}"
          + (f" (compute {med((epi_done-acc)[staged]):.2f}, store+teardown {med((done-epi_done)[staged]):.2f})" if staged.any() else "")
          + f" | total {med(done-start):.2f}")
    order = np.argsort(start)
    waves = start[order]
    print(f"    CTA start times (us) pct 0/25/50/75/100: {np.percentile(start,[0,25,50,75,100]).round(1).tolist()}  "
          f"distinct SMs {len(set(d[:,7].astype(int).tolist()))}")


if __name__ == "__main__":
    torch.manual_seed(0)
    shapes = [(16, 64, 64, 160, 160, 3), (16, 64, 64, 480, 160, 3), (16, 64, 64, 192, 768, 1), (16, 32, 32, 320, 320, 3),
              (16, 16, 16, 320, 320, 3), (16, 8, 8, 640, 640, 3)]
    if os.environ.get("TL_SMALL"):
        shapes = [(16, 8, 8, 640, 640, 3), (16, 16, 16, 320, 320, 3), (16, 8, 8, 1280, 640, 3), (16, 16, 16, 640, 320, 3)]
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    for s in shapes:
        run(*s, tag=os.environ.get("TAG", "default"))
