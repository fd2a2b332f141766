"""Times tile sharding (ResShiftSampler(shard_tiles=True)) on the realsr x4 pipeline with random weights: one
1536x2048 LQ image at the CLI's tiling (chop 512, stride 448, chop_bs 1, padding_offset 64: 4 x 5 = 20 tiles of 512x512,
each a 2048x2048 image through the f4 VQ-GAN and a 512x512 latent through the denoiser).

    python scripts/profile_tile_shards.py --steps 4
    torchrun --nproc_per_node N scripts/profile_tile_shards.py --steps 15

Prints, with the card name and power limit:
  * one GPU: the time per unit (one sample_func call on one tile), then the whole image through the default path and
    through shard mode at world 1, alternating --reps times, and whether the two outputs are bit-identical;
  * under torchrun: the wall time of shard mode on N ranks (barrier to barrier, including the gather and the assembly on
    rank 0) next to the default path on rank 0 alone, and whether the two outputs are bit-identical.
"""
import argparse
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch
import torch.distributed as dist

from resshift_b200.config import preset
from resshift_b200.parallel import gather_counts
from resshift_b200.sampler import ResShiftSampler, make_configs, plan_tiles, tile_counts
from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
from resshift_b200.weights import random_state_dict


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError) as e:
        q = f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"
    return q


def timed(fn):
    torch.cuda.synchronize()
    if dist.is_initialized():
        dist.barrier()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    if dist.is_initialized():
        dist.barrier()
    return out, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=15)
    ap.add_argument("--height", type=int, default=1536)
    ap.add_argument("--width", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profile_tile_shards.py needs a CUDA device")
    ucfg, dcfg = preset("realsr", steps=a.steps)
    vcfg = vq_preset("f4")
    ae = {"target": "ldm.models.autoencoder.VQModelTorch", "params": vcfg.to_kwargs(), "ckpt_path": random_vq_state_dict(vcfg, 0)}
    configs = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    s = ResShiftSampler(configs, sf=4, use_amp=True, chop_size=512, chop_stride=448, chop_bs=1, padding_offset=ucfg.lq_size,
                        seed=12345, shard_tiles=True)
    world, rank = s.num_gpus, s.rank
    h, w = a.height, a.width
    g = torch.Generator(device="cuda").manual_seed(0)
    lq = torch.rand(1, 3, h, w, device="cuda", generator=g) * 2 - 1
    units = s._plan_units([(h, w)])
    if rank == 0:
        print(f"card: {card()}; world {world}")
        print(f"realsr x4, T = {a.steps}, LQ {h}x{w}, chop 512 / stride 448 / chop_bs 1: {len(units)} units of "
              f"{plan_tiles(h, w, 512, 448, 1)[2]}x{plan_tiles(h, w, 512, 448, 1)[3]}", flush=True)

    ctx = torch.autocast("cuda")
    tile = lq[:, :, :512, :512].contiguous()
    unit_times = []
    for _ in range(3):                                          # the first call builds the plans
        with ctx:
            unit_times.append(timed(lambda: s.sample_func(tile).float())[1])
    if rank == 0:
        print(f"time per unit: {', '.join(f'{t:.3f}' for t in unit_times)} s (first call includes plan creation)", flush=True)

    schedule = s._schedule(len(units), world)

    def sharded():
        shares = s._run_rank([lq], [None], False, units, schedule, rank)
        tiles = gather_counts(shares[0], tile_counts(units, schedule, world)[0])
        return s._assemble(tiles, h, w) if rank == 0 else None

    def default():
        return s._sample_tiled(lq) if rank == 0 else None

    for rep in range(a.reps):
        s.setup_seed()
        ref, t_def = timed(default)
        s.setup_seed()
        out, t_sh = timed(sharded)
        if rank == 0:
            same = bool(torch.equal(out, ref))
            print(f"rep {rep}: default path on one GPU {t_def:.3f} s; shard mode on {world} rank(s) {t_sh:.3f} s "
                  f"({t_def / t_sh:.2f}x); bit-identical: {same}", flush=True)
    if dist.is_initialized():
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
