"""Measures UNetModel's multi-head attention kernel (csrc/unet_attn.cuh) and the fused sampling loop of a realsr-width
UNetModel.  Prints the card's name, power limit and maximum SM clock first.

Kernel: every unet_attn instance (head dim D = 32, 64, 128) at the channel counts of a realsr-width UNetModel
(model_channels 160, channel_mult (1, 2, 2, 4): C = 160 / 320 / 320 / 640 at the 64x64 / 32x32 / 16x16 / 8x8 levels,
heads = C / D), batch 16, and batch 1 at T = 16384 (the 128x128 latent of a 512 chop).  CUDA events around `reps`
launches after a warm-up, median of 3 rounds.  Achieved rate = 4 T^2 D heads N (QK^T + PV) / time, next to two bounds:
  * MUFU: one exp2 per score at 16 / clk / SM (132 SMs at the card's max SM clock): T^2 heads N exp2;
  * tensor: 989 TFLOP/s, the H100 SXM data sheet's dense fp16 rate (never reached; a bound only).
torch's scaled_dot_product_attention on the same fp16 shapes ([N, heads, T, D] contiguous) is timed as a sanity
baseline.  (At D = 32 the kernel's P V product computes 64 columns and stores 32; the rate counts the algorithm's FLOPs.)

Loop: ms per 15-step fused loop (CUDA graph replay) of a realsr-width UNetModel (in 6, out 3, 160 channels,
num_head_channels 32, attention at 64/32/16/8, num_res_blocks 2, synthetic weights) at batch 16, 64x64 latent, and of
the shipped realsr UNetModelSwin at the same shape for scale.

    python scripts/profile_unetmodel.py [reps]
"""
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch
import torch.nn.functional as F

from resshift_b200 import _lib
from resshift_b200.config import DiffusionConfig, UNetConfig, UNetModelConfig
from resshift_b200.models.script_util import create_gaussian_diffusion
from resshift_b200.models.unet import UNetModel, UNetModelSwin
from resshift_b200.weights import random_state_dict

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
TENSOR_PEAK = 989e12
SMS = 132


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                              # noqa: BLE001 — the name alone still identifies the card
        q = ""
    return q or torch.cuda.get_device_name(0)


def max_sm_hz():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return float(q.splitlines()[0]) * 1e6
    except Exception:                              # noqa: BLE001
        return 1980e6


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(3):
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / reps)
    return statistics.median(out)


def kernel_table():
    hz = max_sm_hz()
    shapes = [(16, 64 * 64, 160), (16, 32 * 32, 320), (16, 16 * 16, 320), (16, 8 * 8, 640), (1, 128 * 128, 160)]
    print(f"{'D':>4} {'N':>3} {'T':>6} {'heads':>5} {'ms':>9} {'TFLOP/s':>8} {'MUFU-bound ms':>13} {'tensor-bound ms':>15} "
          f"{'of MUFU':>7} {'of tensor':>9} {'sdpa ms':>8}")
    for D in (32, 64, 128):
        for N, T, C in shapes:
            heads = C // D
            g = torch.Generator(device="cuda").manual_seed(0)
            qkv = torch.randn(N, T, 3 * C, device="cuda", generator=g).half()
            out = torch.empty(N, T, C, dtype=torch.float16, device="cuda")
            st = _lib.current_stream()

            def run():
                _lib.check(_lib.lib.rs_op_unet_attention(qkv.data_ptr(), N, T, heads, D, 0, out.data_ptr(), st))
            reps = max(3, REPS if T < 16384 else REPS // 4)
            ms = timed(run, reps)
            flops = 4.0 * T * T * D * heads * N
            mufu_ms = T * T * heads * N / (16.0 * SMS * hz) * 1e3
            tc_ms = flops / TENSOR_PEAK * 1e3
            q, k, v = (torch.randn(N, heads, T, D, device="cuda", generator=g).half() for _ in range(3))
            sdpa_ms = timed(lambda: F.scaled_dot_product_attention(q, k, v), reps)
            print(f"{D:>4} {N:>3} {T:>6} {heads:>5} {ms:>9.4f} {flops / ms / 1e9:>8.1f} {mufu_ms:>13.4f} {tc_ms:>15.4f} "
                  f"{mufu_ms / ms:>7.2f} {tc_ms / ms:>9.2f} {sdpa_ms:>8.4f}")
            del qkv, out, q, k, v
            torch.cuda.empty_cache()


def loop_ms(model, steps=15, B=16, hw=64):
    diff = create_gaussian_diffusion(**DiffusionConfig(steps=steps).to_kwargs())
    g = torch.Generator(device="cuda").manual_seed(0)
    y = torch.rand(B, 3, hw, hw, device="cuda", generator=g) * 2 - 1
    noises = torch.randn(steps + 1, B, 3, hw, hw, device="cuda", generator=g)
    ms = timed(lambda: diff.sample_latent(y, model, {"lq": y}, noises=noises), max(2, REPS // 4))
    return ms, model.num_launches(B, hw, hw)


def main():
    print(f"card (name, power limit, max SM clock): {card()}")
    kernel_table()
    ucfg = UNetModelConfig(image_size=64, in_channels=6, model_channels=160, out_channels=3, num_res_blocks=2,
                           attention_resolutions=(64, 32, 16, 8), channel_mult=(1, 2, 2, 4), num_head_channels=32)
    m = UNetModel(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 0))
    ms, n = loop_ms(m.cuda().eval())
    print(f"UNetModel realsr width, batch 16, 64x64 latent, 15-step fused loop: {ms:.2f} ms per loop, "
          f"{ms / 15:.3f} ms per denoise step, {n} launches per forward")
    del m
    torch.cuda.empty_cache()
    scfg = UNetConfig()
    s = UNetModelSwin(**scfg.to_kwargs())
    s.load_state_dict(random_state_dict(scfg, 0))
    ms, n = loop_ms(s.cuda().eval())
    print(f"UNetModelSwin realsr (shipped), same shape: {ms:.2f} ms per loop, {ms / 15:.3f} ms per denoise step, "
          f"{n} launches per forward")


if __name__ == "__main__":
    main()
