"""Per-launch time of the fused Swin MLP kernel (rs_op_mlp_ex) at the benchmark's batch and every level's shape.

For each shape (E = 192, hidden 768, levels 64x64, 32x32, 16x16 and 8x8): warm-up launches, then CUDA events around one
replay of a CUDA graph of `--iters` back-to-back launches, with the residual in place (out == res, as the Swin block
runs it) and one GroupNorm statistics sink.  Reported as us per launch and TFLOP/s from 4 * pixels * E * hidden.  The
card's name, power limit and max SM clock are printed with the numbers.  RESSHIFT_B200_LIB selects another build of
the library for A/B runs; `--dump DIR` writes each shape's output and sink pairs after one launch on a fresh residual,
so that two builds can be compared.

    python scripts/profile_mlp.py [--batch 16] [--iters 50] [--dump DIR]
"""
import argparse
import ctypes as C
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch

from resshift_b200 import _lib
from tests import gpu_util as G


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0) + " (power limit unknown)"


def run(N, H, W, E=192, Hd=768, iters=50, warmup=5, dump=None):
    g = torch.Generator(device="cuda").manual_seed(H * 1000 + W + E)
    x = torch.randn(N, H, W, E, device="cuda", generator=g).half()
    res0 = torch.randn(N, H, W, E, device="cuda", generator=g).half()
    w1 = torch.randn(Hd, E, device="cuda", generator=g) / E ** 0.5
    b1 = torch.randn(Hd, device="cuda", generator=g) * 0.5
    w2 = torch.randn(E, Hd, device="cuda", generator=g) / Hd ** 0.5 * 0.1
    b2 = torch.randn(E, device="cuda", generator=g) * 0.1
    w1p, _ = G.pack_weight(w1)
    w2p, _ = G.pack_weight(w2)
    res = res0.clone()
    part = torch.zeros(N * H * W * E * 2 // 64 + 64, device="cuda")   # at least N * slots * E pairs (slots <= H*W/64)
    parts = (C.c_void_p * 2)(part.data_ptr(), None)
    cst = (C.c_int32 * 2)(E, 0)
    cof = (C.c_int32 * 2)(0, 0)
    slots = C.c_int32()

    def launch():
        _lib.check(_lib.lib.rs_op_mlp_ex(x.data_ptr(), N, H, W, E, Hd, w1p.data_ptr(), b1.data_ptr(), w2p.data_ptr(),
                                         b2.data_ptr(), res.data_ptr(), res.data_ptr(), parts, cst, cof, C.byref(slots),
                                         G.stream()))

    launch()
    torch.cuda.synchronize()
    if dump is not None:
        n = N * slots.value * E * 2
        torch.save({"out": res.cpu(), "pairs": part[:n].cpu()}, Path(dump) / f"mlp_{N}x{H}x{W}_E{E}.pt")
    for _ in range(warmup):
        launch()
    torch.cuda.synchronize()
    # replayed from a CUDA graph, as the denoiser runs it: the host's per-call work (argument checks, tensor-map
    # encoding) would otherwise be timed instead of the kernel at the small shapes
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(iters):
            launch()
    graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    graph.replay()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    tflops = 4.0 * N * H * W * E * Hd / (us * 1e-6) / 1e12
    tiles = N * H * W // 128
    print(f"mlp N={N} {H}x{W} E={E} Hd={Hd} tiles={tiles}: {us:8.1f} us  {tflops:6.1f} TFLOP/s", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--dump", default=None)
    args = ap.parse_args()
    assert args.iters >= 20
    assert torch.cuda.is_available(), "profile_mlp.py needs a CUDA device"
    if args.dump:
        Path(args.dump).mkdir(parents=True, exist_ok=True)
    print(f"card: {card()}  library: {_lib.LIB_PATH}", flush=True)
    for hw in (64, 32, 16, 8):
        run(args.batch, hw, hw, iters=args.iters, dump=args.dump)


if __name__ == "__main__":
    main()
