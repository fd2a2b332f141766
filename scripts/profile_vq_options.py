"""Times first stages built with the Encoder / Decoder options on one GPU (synthetic weights): encode and decode ms and
the launches of each plan, CUDA events around `reps` back-to-back calls after one warm-up call, median of `rounds`.
  - LDM's vq-f8 shape (ch 128, ch_mult 1-2-2-4, attention at resolution 32: the bottleneck level) at batch 16 x 256x256
    (a 32x32 level: GEMM-form attention, which loops over the images) and batch 1 x 1024x1024 (128x128: fused);
  - the shipped f4 shape without and with attn_resolutions (128, 64) at 512x512 (levels 1 and 2 at 256x256 and 128x128,
    every attention fused).
Prints the card's name and power limit first.

    python scripts/profile_vq_options.py [reps] [rounds]
"""
import statistics
import subprocess
import sys
from dataclasses import replace
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch

from resshift_b200.models.autoencoder import VQModelTorch
from resshift_b200.vq_arch import ldm_vq_preset, random_vq_state_dict, vq_preset

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 5
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 3


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                              # noqa: BLE001 — the name alone still identifies the card
        q = ""
    return q or torch.cuda.get_device_name(0)


def timed(fn):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(ROUNDS):
        e0.record()
        for _ in range(REPS):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / REPS)
    return statistics.median(out)


def main():
    print(f"card: {card()}; synthetic weights, {REPS} calls x {ROUNDS} rounds (median)")
    print(f"{'config':>22} {'batch x image':>14} {'fused enc/dec':>13} {'launches enc/dec':>16} {'encode ms':>10} {'decode ms':>10}")
    cases = [("vq-f8", ldm_vq_preset("vq-f8"), 16, 256), ("vq-f8", ldm_vq_preset("vq-f8"), 1, 1024),
             ("f4", vq_preset("f4"), 1, 512), ("f4 attn (128, 64)", replace(vq_preset("f4"), attn_resolutions=(128, 64)), 1, 512)]
    models = {}
    for tag, cfg, b, hw in cases:
        if tag not in models:
            m = VQModelTorch(**cfg.to_kwargs())
            m.load_state_dict(random_vq_state_dict(cfg, 0))
            models = {tag: m.cuda().eval()}                 # one model at a time
            torch.cuda.empty_cache()
        m = models[tag]
        x = torch.rand(b, 3, hw, hw, device="cuda") * 2 - 1
        z = m.encode(x)
        t_enc = timed(lambda: m.encode(x))
        t_dec = timed(lambda: m.decode(z))
        pe, pd = m.plan(0, b, hw, hw), m.plan(1, b, hw, hw)
        print(f"{tag:>22} {b:>4} x {hw:>4}^2 {len(pe.attentions):>6}/{len(pd.attentions):<6} {pe.launches:>8}/{pd.launches:<7} "
              f"{t_enc:>10.2f} {t_dec:>10.2f}", flush=True)
        del x, z
        m._plans.clear()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
