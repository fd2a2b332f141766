"""Time the fused ancestral loop of a learned-variance model (LEARNED_RANGE, out_channels = 6) against the same loop
on a fixed-variance model of otherwise identical shape (out_channels = 3) and against the learned model's torch route
(the same native UNet called step by step, the step in torch): the realsr-width UNetModelSwin, batch 16, 64x64 latent,
T = 15, in one process, alternating the configurations round by round so that drift of the shared machine falls on all
of them alike.

    python scripts/profile_ddpm_learned.py [--rounds 5] [--reps 5] [--out ddpm_learned.json]

Prints, per configuration, the median and spread of the per-step time (loop time / T) over the rounds and its ratio to
the fused learned loop, with the card name and power limit; writes the same as JSON.  Random weights
(resshift_b200.weights.random_state_dict): the time of the loop does not depend on the values.
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
    from resshift_b200.config import UNetConfig
    from resshift_b200.models.script_util import create_gaussian_diffusion_ddpm
    from resshift_b200.models.unet import UNetModelSwin
    from resshift_b200.weights import random_state_dict

    if not torch.cuda.is_available():
        raise SystemExit("profile_ddpm_learned needs a CUDA device")
    models = {}
    for out_ch in (6, 3):
        ucfg = UNetConfig(out_channels=out_ch)
        m = UNetModelSwin(**ucfg.to_kwargs())
        m.load_state_dict(random_state_dict(ucfg, 0), strict=True)
        models[out_ch] = m.cuda().eval()
    B, H, W = args.batch, 64, 64
    g = torch.Generator(device="cuda").manual_seed(1)
    y = torch.rand(B, 3, H, W, device="cuda", generator=g) * 2 - 1
    kw = dict(beta_start=0.0015, beta_end=0.0155, steps=1000, timestep_respacing=T)
    learned = create_gaussian_diffusion_ddpm(learn_sigma=True, **kw)
    fixed = create_gaussian_diffusion_ddpm(**kw)
    noises = learned.draw_noises((B, 3, H, W), device="cuda")
    mk = {"lq": y}
    ml, mf = models[6], models[3]
    wrapped = lambda xx, tt, **k: ml(xx, tt, **k)                   # noqa: E731  (not a native UNet: the torch route)
    assert learned._native_ok(ml, None, mk) and fixed._native_ok(mf, None, mk)
    assert not learned._native_ok(wrapped, None, mk) and not learned._native_ok(mf, None, mk)

    def torch_route():
        queue = list(noises[1:])
        orig = torch.randn_like
        torch.randn_like = lambda ref: queue.pop(0)
        try:
            return learned.p_sample_loop(wrapped, (B, 3, H, W), noise=noises[0], clip_denoised=False, model_kwargs=mk,
                                         device="cuda")
        finally:
            torch.randn_like = orig

    runs = {
        "learned graph": lambda: learned.sample_latent(ml, noises, mk, "ancestral", False),
        "fixed graph": lambda: fixed.sample_latent(mf, noises, mk, "ancestral", False),
        "learned torch route": torch_route,
    }
    names = list(runs)
    with torch.no_grad():
        for fn in runs.values():            # capture each sampler's graph, warm up
            for _ in range(2):
                fn()
        torch.cuda.synchronize()
        a, b = runs["learned graph"](), runs["learned torch route"]()
        same = bool(torch.equal(a, b))
        dmax = float((a - b).abs().max())

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
    res = {"card": card, "batch": B, "latent": [H, W], "T": T, "rounds": args.rounds, "reps": args.reps,
           "fused_equals_torch_route": same, "fused_vs_torch_route_max_abs": dmax, "step_ms": {}}
    base = sorted(times["learned graph"])[len(times["learned graph"]) // 2]
    print(f"card: {card}; realsr-width UNetModelSwin, batch {B}, {H}x{W} latent, T = {T} per loop, ancestral, eps, "
          f"no clip (per-step time = loop time / T, including the copies in)")
    print(f"learned (LEARNED_RANGE, out_channels 6) fused vs torch route: bit-identical {same}, max|d| {dmax:.3e}")
    for n in names:
        ts = sorted(times[n])
        med = ts[len(ts) // 2]
        res["step_ms"][n] = {"median": med, "min": ts[0], "max": ts[-1], "ratio_to_learned_graph": med / base}
        print(f"  {n:20s} median {med:8.3f} ms/step  [min {ts[0]:8.3f}, max {ts[-1]:8.3f}]  "
              f"ratio to learned graph {med / base:.4f}")
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
