"""Times the device pool (ResShiftSampler(devices=...)) on the workload of scripts/profile_tile_shards.py: the realsr x4
pipeline with random weights, one 1536x2048 LQ photo at the CLI's tiling (chop 512, stride 448, chop_bs 1,
padding_offset 64: 20 units of one 512x512 tile each).

    python scripts/profile_device_pool.py --steps 4
    python scripts/profile_device_pool.py --steps 15 --devices all

Prints the card name and power limit, then, alternating --reps times, the wall time of inference() on the photo (PNG in,
PNG out) through the default one-GPU path and through a pool of --devices (default: every visible GPU; on a one-GPU
machine that is a pool of one, whose cost over the default path is what it shows), and whether the PNG bytes are equal.
"""
import argparse
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import numpy as np
import torch

from profile_tile_shards import card
from resshift_b200.config import preset
from resshift_b200.sampler import ResShiftSampler, make_configs
from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
from resshift_b200.weights import random_state_dict


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=15)
    ap.add_argument("--height", type=int, default=1536)
    ap.add_argument("--width", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--devices", default="all")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profile_device_pool.py needs a CUDA device")
    import cv2
    ucfg, dcfg = preset("realsr", steps=a.steps)
    vcfg = vq_preset("f4")
    ae = {"target": "ldm.models.autoencoder.VQModelTorch", "params": vcfg.to_kwargs(), "ckpt_path": random_vq_state_dict(vcfg, 0)}
    configs = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    kw = dict(sf=4, use_amp=True, chop_size=512, chop_stride=448, chop_bs=1, padding_offset=ucfg.lq_size, seed=12345)
    default = ResShiftSampler(configs, devices="", **kw)
    pool = ResShiftSampler(configs, devices=a.devices, **kw)
    names = [f"cuda:{r.device.index}" for r in pool.pool.replicas]
    n_units = len(default._plan_units([(a.height, a.width)]))
    print(f"card: {card()}; {torch.cuda.device_count()} visible GPU(s); pool: {', '.join(names)}")
    print(f"realsr x4, T = {a.steps}, LQ {a.height}x{a.width}, chop 512 / stride 448 / chop_bs 1: {n_units} units",
          flush=True)

    with tempfile.TemporaryDirectory() as tmp:
        tmp = Path(tmp)
        rng = np.random.default_rng(0)
        (tmp / "in").mkdir()
        (tmp / "warm").mkdir()
        cv2.imwrite(str(tmp / "in" / "photo.png"), rng.integers(0, 256, (a.height, a.width, 3), dtype=np.uint8))
        cv2.imwrite(str(tmp / "warm" / "tile.png"), rng.integers(0, 256, (512, 512, 3), dtype=np.uint8))

        def run(s, out):
            s.setup_seed()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            s.inference(tmp / "in", tmp / out, bs=1)
            torch.cuda.synchronize()
            return time.perf_counter() - t0, (tmp / out / "photo.png").read_bytes()

        for s in (default, pool):                               # plans for the 512x512 unit on every replica
            s.inference(tmp / "warm", tmp / "warm_out", bs=1)
        for rep in range(a.reps):
            t_def, ref = run(default, f"def{rep}")
            t_pool, out = run(pool, f"pool{rep}")
            print(f"rep {rep}: default path {t_def:.3f} s; pool of {len(names)} {t_pool:.3f} s ({t_def / t_pool:.2f}x); "
                  f"PNG bytes equal: {out == ref}", flush=True)


if __name__ == "__main__":
    main()
