"""Time the fused sampling loop (CUDA graph replay) of every predict_type against xstart on the realsr-width
UNetModelSwin, batch 16, 64x64 latent, T = 15, in one process, alternating the configurations round by round so
that drift of the shared machine falls on all of them alike.

    python scripts/profile_predict_types.py [--rounds 5] [--reps 5] [--out predict_types.json]

Prints, per mean type, the median and spread of the loop time over the rounds and its ratio to xstart, with the card
name and power limit; writes the same as JSON.  Random weights (resshift_b200.weights.random_state_dict): the time of
the loop does not depend on the values.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

MEAN_TYPES = ("xstart", "epsilon", "epsilon_scale", "residual")


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, check=True).stdout.strip().splitlines()[0]
        return q
    except (OSError, subprocess.CalledProcessError, IndexError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5, help="loops per timed window")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from resshift_b200.config import DiffusionConfig, UNetConfig
    from resshift_b200.models.script_util import create_gaussian_diffusion
    from resshift_b200.models.unet import UNetModelSwin
    from resshift_b200.weights import random_state_dict

    if not torch.cuda.is_available():
        raise SystemExit("profile_predict_types needs a CUDA device")
    ucfg = UNetConfig()
    m = UNetModelSwin(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 0), strict=True)
    m = m.cuda().eval()
    B, H, W = args.batch, 64, 64
    g = torch.Generator(device="cuda").manual_seed(1)
    y = torch.rand(B, 3, H, W, device="cuda", generator=g) * 2 - 1
    diffs = {mt: create_gaussian_diffusion(**DiffusionConfig(steps=15, sf=1, predict_type=mt).to_kwargs())
             for mt in MEAN_TYPES}
    noises = diffs["xstart"].draw_noises(y)
    for d in diffs.values():            # capture each sampler's graph, warm up
        for _ in range(2):
            d.sample_latent(y, m, {"lq": y}, noises=noises)
    torch.cuda.synchronize()

    times = {mt: [] for mt in MEAN_TYPES}
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(args.rounds):
        order = MEAN_TYPES if r % 2 == 0 else MEAN_TYPES[::-1]
        for mt in order:
            start.record()
            for _ in range(args.reps):
                diffs[mt].sample_latent(y, m, {"lq": y}, noises=noises)
            end.record()
            end.synchronize()
            times[mt].append(start.elapsed_time(end) / args.reps)

    card = _card()
    res = {"card": card, "batch": B, "latent": [H, W], "T": 15, "rounds": args.rounds, "reps": args.reps, "loop_ms": {}}
    base = sorted(times["xstart"])[len(times["xstart"]) // 2]
    print(f"card: {card}; realsr-width UNetModelSwin, batch {B}, {H}x{W} latent, T = 15 (graph replay, incl. copies in)")
    for mt in MEAN_TYPES:
        ts = sorted(times[mt])
        med = ts[len(ts) // 2]
        res["loop_ms"][mt] = {"median": med, "min": ts[0], "max": ts[-1], "ratio_to_xstart": med / base}
        print(f"  {mt:14s} median {med:8.3f} ms  [min {ts[0]:8.3f}, max {ts[-1]:8.3f}]  ratio to xstart {med / base:.4f}")
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
