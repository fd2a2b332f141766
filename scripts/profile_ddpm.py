"""Time the fused DDIM and ancestral DDPM loops against the fused ResShift loop on the same plan: the realsr-width
UNetModelSwin, batch 16, 64x64 latent, T = 15 for every process, each as CUDA graph replay and eagerly, in one process,
alternating the configurations round by round so that drift of the shared machine falls on all of them alike.

    python scripts/profile_ddpm.py [--rounds 5] [--reps 5] [--out ddpm.json]

Prints, per configuration, the median and spread of the per-step time (loop time / T) over the rounds and its ratio to
the ResShift graph replay, with the card name and power limit; writes the same as JSON.  Each step is one denoiser
forward plus one elementwise launch for every process, so equal per-step times are what the design predicts.  Random
weights (resshift_b200.weights.random_state_dict): the time of the loop does not depend on the values.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

T = 15


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, check=True).stdout.strip().splitlines()[0]
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
    from resshift_b200.models.script_util import create_gaussian_diffusion, create_gaussian_diffusion_ddpm
    from resshift_b200.models.unet import UNetModelSwin
    from resshift_b200.weights import random_state_dict

    if not torch.cuda.is_available():
        raise SystemExit("profile_ddpm needs a CUDA device")
    ucfg = UNetConfig()
    m = UNetModelSwin(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 0), strict=True)
    m = m.cuda().eval()
    B, H, W = args.batch, 64, 64
    g = torch.Generator(device="cuda").manual_seed(1)
    y = torch.rand(B, 3, H, W, device="cuda", generator=g) * 2 - 1
    rs = create_gaussian_diffusion(**DiffusionConfig(steps=T, sf=1).to_kwargs())
    dd = create_gaussian_diffusion_ddpm(beta_start=0.0015, beta_end=0.0155, steps=1000, timestep_respacing=T)
    noises = rs.draw_noises(y)
    runs = {
        "resshift graph": lambda: rs.sample_latent(y, m, {"lq": y}, noises=noises),
        "ddim graph": lambda: dd.sample_latent(m, noises, {"lq": y}, "ddim", True, 0.0),
        "ancestral graph": lambda: dd.sample_latent(m, noises, {"lq": y}, "ancestral", True),
        "resshift eager": lambda: rs.sample_latent(y, m, {"lq": y}, noises=noises, use_graph=False),
        "ddim eager": lambda: dd.sample_latent(m, noises, {"lq": y}, "ddim", True, 0.0, use_graph=False),
    }
    names = list(runs)
    for fn in runs.values():            # capture each sampler's graph, warm up
        for _ in range(2):
            fn()
    torch.cuda.synchronize()

    times = {n: [] for n in names}
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(args.rounds):
        for n in (names if r % 2 == 0 else names[::-1]):
            start.record()
            for _ in range(args.reps):
                runs[n]()
            end.record()
            end.synchronize()
            times[n].append(start.elapsed_time(end) / args.reps / T)

    card = _card()
    res = {"card": card, "batch": B, "latent": [H, W], "T": T, "rounds": args.rounds, "reps": args.reps, "step_ms": {}}
    base = sorted(times["resshift graph"])[len(times["resshift graph"]) // 2]
    print(f"card: {card}; realsr-width UNetModelSwin, batch {B}, {H}x{W} latent, T = {T} per loop "
          f"(per-step time = loop time / T, including the copies in)")
    for n in names:
        ts = sorted(times[n])
        med = ts[len(ts) // 2]
        res["step_ms"][n] = {"median": med, "min": ts[0], "max": ts[-1], "ratio_to_resshift_graph": med / base}
        print(f"  {n:16s} median {med:8.3f} ms/step  [min {ts[0]:8.3f}, max {ts[-1]:8.3f}]  "
              f"ratio to resshift graph {med / base:.4f}")
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
