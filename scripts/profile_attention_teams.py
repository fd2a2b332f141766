"""Measures what attention teams (DESIGN.md §6) work with: the fused VQ-GAN bottleneck attention on a fraction of its
query rows, and one 512x512 realsr x4 unit (the CLI's default chop: a 2048x2048 image through the f4 VQ-GAN, whose
bottleneck attention has T = 262144 positions at C = 512), with random weights.

    python scripts/profile_attention_teams.py [--iters 3]

Prints, with the card name and power limit:
  * rs_op_vq_attention_rows at T = 262144, C = 512, N = 1 on the first 1, 1/2, 1/4 and 1/8 of the rows (CUDA events over
    --iters launches after a warm-up);
  * the wall time of one unit (sample_func on one 512x512 LQ tile) at T = 4 and T = 15 steps;
  * the predicted time of that unit on a team of k ranks: the unit minus its two full attention launches plus two
    launches on 1/k of the rows.  The row exchange between the ranks is not in this figure.
With two or more GPUs visible it also spawns one process per GPU (NCCL) and times a real team run of the unit at the
first --steps value, barrier to barrier, against the same unit on one GPU, and checks that both are bit-identical.
"""
import argparse
import os
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch
import torch.distributed as dist

from resshift_b200 import _lib
from resshift_b200.config import preset
from resshift_b200.parallel import gather_counts
from resshift_b200.sampler import ResShiftSampler, make_configs, tile_counts
from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
from resshift_b200.weights import random_state_dict

T_POS, C_BOT = 262144, 512


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError) as e:
        q = f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"
    return q


def events(fn, iters):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def attention_rows_ms(frac_den, iters):
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, v = (torch.randn(1, T_POS, C_BOT, device="cuda", generator=g).half() for _ in range(3))
    out = torch.empty_like(q)
    st, rows = _lib.current_stream(), T_POS // frac_den
    f = lambda: _lib.check(_lib.lib.rs_op_vq_attention_rows(q.data_ptr(), k.data_ptr(), v.data_ptr(), 1, T_POS, C_BOT, C_BOT,
                                                            0, rows, out.data_ptr(), st))
    return events(f, iters)


def sampler(steps, **kw):
    ucfg, dcfg = preset("realsr", steps=steps)
    vcfg = vq_preset("f4")
    ae = {"target": "ldm.models.autoencoder.VQModelTorch", "params": vcfg.to_kwargs(), "ckpt_path": random_vq_state_dict(vcfg, 0)}
    configs = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    return ResShiftSampler(configs, sf=4, use_amp=True, chop_size=512, chop_stride=448, chop_bs=1,
                           padding_offset=ucfg.lq_size, seed=12345, shard_tiles=True, **kw)


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


def lq_tile():
    g = torch.Generator(device="cuda").manual_seed(0)
    return torch.rand(1, 3, 512, 512, device="cuda", generator=g) * 2 - 1


def team_worker(rank, world, port, steps, reps):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), LOCAL_RANK=str(rank),
                      WORLD_SIZE=str(world))
    s = sampler(steps)                                        # setup_dist: NCCL, one GPU per rank
    lq = lq_tile()
    units = s._plan_units([(512, 512)])
    schedule = s._schedule(len(units), world)                # one unit: a team of every rank

    def team():
        shares = s._run_rank([lq], [None], False, units, schedule, rank)
        tiles = gather_counts(shares[0], tile_counts(units, schedule, world)[0])
        return s._assemble(tiles, 512, 512) if rank == 0 else None

    def one():
        return s._sample_tiled(lq) if rank == 0 else None

    for rep in range(reps + 1):                               # rep 0 builds the plans
        s.setup_seed()
        ref, t_one = timed(one)
        s.setup_seed()
        out, t_team = timed(team)
        if rank == 0 and rep > 0:
            print(f"team of {world} (NCCL), T = {steps}: {t_team:.3f} s; the unit on one GPU {t_one:.3f} s "
                  f"({t_one / t_team:.2f}x); bit-identical: {bool(torch.equal(out, ref))}", flush=True)
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--steps", type=int, nargs="+", default=[4, 15])
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profile_attention_teams.py needs a CUDA device")
    print(f"card: {card()}")
    print(f"== fused attention on a row range, T = {T_POS}, C = {C_BOT}, N = 1 (CUDA events, {a.iters} launches after warm-up)")
    att = {}
    for k in (1, 2, 4, 8):
        att[k] = attention_rows_ms(k, a.iters)
        print(f"rows 1/{k}: {att[k]:9.2f} ms  ({4.0 * T_POS * T_POS * C_BOT / k / att[k] / 1e9:6.1f} TFLOP/s, "
              f"{att[1] / att[k] if k > 1 else 1.0:.2f}x less than all rows)", flush=True)

    for steps in a.steps:
        s = sampler(steps)
        tile = lq_tile()
        times = []
        for _ in range(3):                                    # the first call builds the plans
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with torch.autocast("cuda"):
                s.sample_func(tile).float()
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        unit = min(times[1:])
        print(f"== realsr x4 unit, 512x512 LQ (2048x2048 through the f4 VQ-GAN), T = {steps}: "
              f"{', '.join(f'{t:.3f}' for t in times)} s (first call includes plan creation)")
        rest = unit - 2 * att[1] / 1e3
        print(f"   two attention launches {2 * att[1] / 1e3:.3f} s = {100 * 2 * att[1] / 1e3 / unit:.1f} % of the unit; "
              f"the rest {rest:.3f} s")
        for k in (2, 4, 8):
            pred = rest + 2 * att[k] / 1e3
            print(f"   predicted on a team of {k}: {pred:.3f} s ({unit / pred:.2f}x), without the row exchange", flush=True)
        del s
        torch.cuda.empty_cache()

    n = torch.cuda.device_count()
    if n >= 2:
        import torch.multiprocessing as mp
        port = 29500 + os.getpid() % 2000
        mp.spawn(team_worker, args=(n, port, a.steps[0], a.reps), nprocs=n, join=True)
    else:
        print(f"== one GPU visible: no team run (multi-GPU figures above are predictions, not measurements)")


if __name__ == "__main__":
    main()
