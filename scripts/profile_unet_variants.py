"""Times one batch-16, 4-step fused sampling loop (CUDA graph replay, 64x64 latent) of the realsr-width denoiser
(model_channels 160, swin_embed_dim 192, synthetic weights) for the shipped topology and for each constructor-option
variant of oracle/make_golden_variants.py.  CUDA events around `reps` replays after one warm-up, median of `rounds`.
Prints the card's name and power limit first.  It reports what a variant costs; it checks nothing.

    python scripts/profile_unet_variants.py [reps] [rounds]
"""
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch

from oracle.make_golden_variants import VARIANTS
from resshift_b200.config import DiffusionConfig, UNetConfig
from resshift_b200.models.script_util import create_gaussian_diffusion
from resshift_b200.models.unet import UNetModelSwin
from resshift_b200.weights import random_state_dict

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 10
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 3
B, T = 16, 4


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                              # noqa: BLE001 — the name alone still identifies the card
        q = ""
    return q or torch.cuda.get_device_name(0)


def loop_ms(ucfg):
    m = UNetModelSwin(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 0))
    m = m.cuda().eval()
    diff = create_gaussian_diffusion(**DiffusionConfig(steps=T, min_noise_level=0.2, sf=1).to_kwargs())
    g = torch.Generator(device="cuda").manual_seed(0)
    y = torch.rand(B, 3, 64, 64, device="cuda", generator=g) * 2 - 1
    mask = None
    if ucfg.cond_mask:
        mask = torch.ones(B, 1, 64, 64, device="cuda")
    kw = {"lq": y} if mask is None else {"lq": y, "mask": mask}
    noises = torch.randn(T + 1, B, 3, 64, 64, device="cuda", generator=g)
    diff.sample_latent(y, m, kw, noises=noises)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(ROUNDS):
        e0.record()
        for _ in range(REPS):
            diff.sample_latent(y, m, kw, noises=noises)
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / REPS)
    launches = m.num_launches(B, 64, 64)
    del m
    torch.cuda.empty_cache()
    return statistics.median(out), launches


def main():
    print(f"card: {card()}; realsr width, batch {B}, 64x64 latent, T = {T} fused loop, {REPS} replays x {ROUNDS} rounds (median)")
    print(f"{'variant':>16} {'loop ms':>9} {'vs shipped':>10} {'launches/forward':>17}")
    base, n0 = loop_ms(UNetConfig())
    print(f"{'shipped':>16} {base:>9.2f} {1.0:>10.3f} {n0:>17}")
    for name, kw in VARIANTS.items():
        ms, n = loop_ms(UNetConfig(**kw))
        print(f"{name:>16} {ms:>9.2f} {ms / base:>10.3f} {n:>17}")


if __name__ == "__main__":
    main()
