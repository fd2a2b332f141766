"""Sweep the conv/GEMM tile configuration knobs (BN, cta pair, CTAs/SM, split-K) over the model's layer shapes at the
benchmark batch and print, per shape, the default pick's time next to the best forced configuration.
Calibration aid for pick_tile_config() (launch.cuh); run on the GPU box."""
import ctypes as C
import itertools
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch

from resshift_b200 import _lib
from tests import gpu_util as G

L = _lib.lib
KNOBS = ("RS_CONV_BN", "RS_CONV_CG", "RS_CONV_OCC", "RS_CONV_SPLITK")


def time_conv(t, iters=24):
    x, wp, ipad, b, out, scratch, dbg, (N, H, W, Ci, Co, k) = t
    info = (C.c_int32 * 7)()
    st = _lib.current_stream()
    rc = L.rs_op_conv2d_timeline(x.data_ptr(), N, H, W, Ci, Ci, wp.data_ptr(), ipad, b.data_ptr(), Co, k, 1,
                                 out.data_ptr(), Co, 0, 3, dbg.data_ptr(), info, scratch.data_ptr(), st)
    if rc != 0:
        torch.cuda.synchronize()
        return None, None
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    L.rs_op_conv2d_timeline(x.data_ptr(), N, H, W, Ci, Ci, wp.data_ptr(), ipad, b.data_ptr(), Co, k, 1,
                            out.data_ptr(), Co, 0, iters, dbg.data_ptr(), info, scratch.data_ptr(), st)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3, (info[1], info[4], info[5], info[2], info[0], info[6])


def main():
    N = int(os.environ.get("SWEEP_BATCH", "16"))
    shapes = [
        (64, 160, 160, 3), (64, 320, 160, 3), (64, 480, 160, 3), (64, 320, 320, 3), (64, 192, 576, 1), (64, 192, 192, 1),
        (64, 160, 192, 1), (64, 192, 160, 1), (64, 320, 160, 1),
        (32, 320, 320, 3), (32, 640, 320, 3), (32, 480, 320, 3), (32, 160, 320, 3), (32, 192, 576, 1), (32, 192, 192, 1),
        (32, 320, 192, 1), (32, 192, 320, 1),
        (16, 320, 320, 3), (16, 640, 320, 3), (16, 960, 320, 3), (16, 640, 640, 3), (16, 192, 576, 1), (16, 192, 192, 1),
        (8, 640, 640, 3), (8, 1280, 640, 3), (8, 960, 640, 3), (8, 320, 640, 3), (8, 192, 576, 1), (8, 192, 192, 1),
        (8, 640, 192, 1), (8, 192, 640, 1),
    ]
    only = os.environ.get("SWEEP_ONLY")
    total_def = total_best = 0.0
    for (HW, Ci, Co, k) in shapes:
        if only and f"{HW},{Ci},{Co},{k}" != only:
            continue
        x = torch.randn(N, HW, HW, Ci, device="cuda").half()
        w = torch.randn(Co, Ci, k, k, device="cuda") / (Ci * k * k) ** 0.5
        b = torch.randn(Co, device="cuda")
        wp, ipad = G.pack_weight(w)
        out = torch.empty(N, HW, HW, Co, dtype=torch.float16, device="cuda")
        scratch = torch.empty(8 * N * HW * HW * Co, dtype=torch.float32, device="cuda")
        dbg = torch.zeros(8 * 8192, dtype=torch.int64, device="cuda")
        t = (x, wp, ipad, b, out, scratch, dbg, (N, HW, HW, Ci, Co, k))
        for kn in KNOBS:
            os.environ.pop(kn, None)
        t_def, cfg_def = time_conv(t)
        co16 = (Co + 15) // 16 * 16
        bns = [c for c in range(256, 47, -16) if co16 % c == 0]
        m_tiles = N * HW * HW // 128
        splits = [1] if m_tiles * max(1, co16 // 160) >= 296 else [1, 2, 3, 4, 6, 8]
        results = []
        for bn, cg, occ, sk in itertools.product(bns, (1, 2), (1, 2), splits):
            os.environ.update(RS_CONV_BN=str(bn), RS_CONV_CG=str(cg), RS_CONV_OCC=str(occ), RS_CONV_SPLITK=str(sk))
            us, cfg = time_conv(t, iters=12)
            if us is not None and cfg[0] == bn and cfg[1] == cg and cfg[2] == sk:
                results.append((us, bn, cg, occ, sk, cfg[3], cfg[4]))
        for kn in KNOBS:
            os.environ.pop(kn, None)
        results.sort()
        best = results[0]
        total_def += t_def; total_best += best[0]
        top = "  ".join(f"[{r[0]:.1f}us BN={r[1]} cg={r[2]} occ={r[3]} S={r[4]} st={r[5]}]" for r in results[:4])
        print(f"{HW}x{HW} Cin={Ci} Cout={Co} k={k}: default {t_def:.1f}us (BN={cfg_def[0]} cg={cfg_def[1]} S={cfg_def[2]} st={cfg_def[3]} grid={cfg_def[4]}{' persist' if cfg_def[5] else ''})"
              f" | best {top}", flush=True)
    print(f"sum default {total_def:.1f} us, sum best {total_best:.1f} us")


if __name__ == "__main__":
    main()
