"""Per-launch time of the fused Swin attention kernel (rs_op_swin_attn) at the benchmark's batch and every level's shape.

For each shape: warm-up launches, then CUDA events around one replay of a CUDA graph of `--iters` back-to-back launches
(in place, y == x, as the denoiser runs it), reported as us per launch and TFLOP/s from 22.0 MFLOP per 8x8 window at E = 192 (DESIGN.md §4:
qkv 14.16 + QK^T 1.57 + PV 1.57 + proj 4.72).  The card's name and power limit are printed with the numbers.
RESSHIFT_B200_LIB selects another build of the library for A/B runs.

    python scripts/profile_swin.py [--batch 16] [--iters 50]
"""
import argparse
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


def flop_per_window(E: int) -> float:
    T = 64
    return 2 * T * E * 3 * E + 2 * 2 * T * T * E + 2 * T * E * E


def run(N, H, W, shift, E=192, iters=50, warmup=5):
    heads = E // 32
    g = torch.Generator(device="cuda").manual_seed(1)
    x = (torch.randn(N, H, W, E, device="cuda", generator=g)).half()
    gamma = 1 + 0.1 * torch.randn(E, device="cuda", generator=g)
    beta = 0.1 * torch.randn(E, device="cuda", generator=g)
    wqkv = torch.randn(3 * E, E, device="cuda", generator=g) / E ** 0.5
    bqkv = torch.zeros(3 * E, device="cuda")
    wproj = torch.randn(E, E, device="cuda", generator=g) / E ** 0.5 * 0.1
    bproj = torch.zeros(E, device="cuda")
    table = torch.randn(225, heads, device="cuda", generator=g) * 0.5
    dense = torch.empty(heads * 64 * 64, dtype=torch.float32, device="cuda")
    _lib.check(G.L.rs_op_expand_relpos(table.data_ptr(), dense.data_ptr(), heads, G.stream()))
    rows = 128 if H * W >= 128 else 64
    slots = H * W // rows
    xs = x.float().reshape(N, slots, rows, E)
    mean_s = xs.mean(dim=2)
    part = torch.stack([mean_s, ((xs - mean_s[:, :, None]) ** 2).sum(dim=2)], dim=-1).contiguous()
    wq_p, _ = G.pack_weight(wqkv)
    wp_p, _ = G.pack_weight(wproj)
    pout = torch.empty(N, (H // 8) * (W // 8), E, 2, device="cuda")

    def launch():
        _lib.check(G.L.rs_op_swin_attn(x.data_ptr(), N, H, W, E, heads, shift, part.data_ptr(), slots, gamma.data_ptr(),
                                       beta.data_ptr(), wq_p.data_ptr(), bqkv.data_ptr(), dense.data_ptr(), wp_p.data_ptr(),
                                       bproj.data_ptr(), x.data_ptr(), pout.data_ptr(), None, None, G.stream()))

    for _ in range(warmup):
        launch()
    torch.cuda.synchronize()
    # the launches are replayed from a CUDA graph, as the denoiser runs them: the host's per-call work (argument
    # checks, tensor-map encoding) would otherwise be timed instead of the kernel at the small shapes
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
    windows = N * (H // 8) * (W // 8)
    tflops = windows * flop_per_window(E) / (us * 1e-6) / 1e12
    print(f"swin_attn N={N} {H}x{W} shift={shift} E={E} pairs={(windows + 1) // 2}: {us:8.1f} us  {tflops:6.1f} TFLOP/s", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    assert args.iters >= 20
    assert torch.cuda.is_available(), "profile_swin.py needs a CUDA device"
    print(f"card: {card()}  library: {_lib.LIB_PATH}", flush=True)
    print(f"{flop_per_window(192) / 1e6:.1f} MFLOP per 8x8 window at E = 192", flush=True)
    for hw in (64, 32, 16, 8):
        for shift in (0, 4):
            if shift and hw == 8:
                continue                       # one window per image: the model does not shift there
            run(args.batch, hw, hw, shift, iters=args.iters)


if __name__ == "__main__":
    main()
