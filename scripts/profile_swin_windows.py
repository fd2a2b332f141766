"""Per-launch time of the window-attention core (rs_op_window_attention_ex) for its four instances (windows of 8 or 16,
heads of 32 or 64) at E = 192, the benchmark's batch, 64x64 and 32x32 maps, unshifted and shifted.

For each case: warm-up launches, then CUDA events around one replay of a CUDA graph of `--iters` back-to-back launches (as
scripts/profile_swin.py does), reported as us per launch and as TFLOP/s from the 4 T^2 E FLOP of QK^T and PV per window of
T tokens (the softmax is not counted).  The card's name, power limit and maximum SM clock are printed with the numbers.

    python scripts/profile_swin_windows.py [--batch 16] [--iters 50]
"""
import argparse
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch

from resshift_b200 import _lib
from scripts.profile_swin import card


def run(N, H, W, ws, hd, shift, E=192, iters=50, warmup=5):
    heads, T = E // hd, ws * ws
    g = torch.Generator(device="cuda").manual_seed(1)
    qkv = torch.randn(N, H, W, 3 * E, device="cuda", generator=g).half()
    table = torch.randn((2 * ws - 1) ** 2, heads, device="cuda", generator=g) * 0.5
    dense = torch.empty(heads * T * T, dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.rs_op_expand_relpos_ex(table.data_ptr(), dense.data_ptr(), heads, ws, _lib.current_stream()))
    out = torch.empty(N, H, W, E, dtype=torch.float16, device="cuda")

    def launch():
        _lib.check(_lib.lib.rs_op_window_attention_ex(qkv.data_ptr(), N, H, W, heads, ws, hd, shift, dense.data_ptr(),
                                                      out.data_ptr(), _lib.current_stream()))

    for _ in range(warmup):
        launch()
    torch.cuda.synchronize()
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
    windows = N * (H // ws) * (W // ws)
    tflops = windows * 4.0 * T * T * E / (us * 1e-6) / 1e12
    gbs = N * H * W * 4 * E * 2 / (us * 1e-6) / 1e9          # qkv read once, out written once
    print(f"window_attn<{ws:2d}, {hd}> N={N} {H}x{W} shift={shift} heads={heads} windows={windows:5d}: {us:8.1f} us  "
          f"{tflops:6.1f} TFLOP/s  {gbs:6.0f} GB/s", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    assert args.iters >= 20
    assert torch.cuda.is_available(), "profile_swin_windows.py needs a CUDA device"
    print(f"card (name, power limit, max SM clock): {card()}  library: {os.path.relpath(_lib.LIB_PATH, ROOT)}", flush=True)
    for ws, hd in ((8, 32), (8, 64), (16, 32), (16, 64)):
        for hw in (64, 32):
            for shift in (0, ws // 2):
                run(args.batch, hw, hw, ws, hd, shift, iters=args.iters)


if __name__ == "__main__":
    main()
