"""Attention teams in tile-shard mode: when a chunk has fewer work units than ranks, unit u runs on team u of the ranks,
every member runs the whole unit, and the VQ-GAN bottleneck attention's query rows (more than 8192 positions) are split
across the team and exchanged.  The PNGs must be byte-identical to a one-GPU default run.

1. One unit, three ranks: 3 processes on one GPU under gloo, one 128x128 LQ image (x4: a 512x512 image, a 128x128
   bottleneck, T = 16384): one team of three.
2. Two units, three ranks: a 128x128 and a 128x192 image (T = 24576): teams of two and one.
3. The first case on two GPUs under NCCL (a team of two)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _sampler(**kw):
    from resshift_b200.config import preset
    from resshift_b200.sampler import ResShiftSampler, make_configs
    from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
    from resshift_b200.weights import random_state_dict
    ucfg, dcfg = preset("tiny")
    dcfg.sf = 4
    vcfg = vq_preset("tiny")
    ae = {"target": "ldm.models.autoencoder.VQModelTorch", "params": vcfg.to_kwargs(), "ckpt_path": random_vq_state_dict(vcfg, 0)}
    configs = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    return ResShiftSampler(configs, sf=4, use_amp=True, seed=123, chop_size=512, chop_stride=448, padding_offset=16, **kw)


def _write_pngs(d, shapes):
    import cv2
    rng = np.random.default_rng(5)
    d.mkdir()
    for name, (h, w) in shapes.items():
        cv2.imwrite(str(d / f"{name}.png"), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))


def _worker(rank, world, port, backend, in_dir, out_dir, bs, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world))
    import cv2
    import torch.distributed as dist
    try:
        if backend == "gloo":                                 # (NCCL: the sampler's setup_dist initialises it)
            dist.init_process_group("gloo", rank=rank, world_size=world)
        s = _sampler(shard_tiles=True)
        assert s.num_gpus == world and s.rank == rank and dist.get_backend() == backend
        ran, writes = [], []
        orig_unit, orig_write = s._sample_unit, cv2.imwrite
        s._sample_unit = lambda *a: (ran.append(tuple(a[0].shape[2:])), orig_unit(*a))[1]
        cv2.imwrite = lambda *a: (writes.append(a[0]), orig_write(*a))[1]
        s.inference(in_dir, out_dir, bs=bs)
        q.put((rank, ran, len(writes), list(s.autoencoder.attention_rows), ""))
    except Exception:                                         # noqa: BLE001 — report instead of hanging the parent
        import traceback
        q.put((rank, None, -1, None, traceback.format_exc()))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _run(tmp_path, backend, world, shapes):
    import torch.multiprocessing as mp
    in_dir, out_dir, ref_dir = tmp_path / "in", tmp_path / "out", tmp_path / "ref"
    _write_pngs(in_dir, shapes)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() + 3) % 2000
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, str(in_dir), str(out_dir), len(shapes), q))
             for r in range(world)]
    try:
        for p in procs:
            p.start()
        res = sorted((q.get(timeout=900) for _ in procs), key=lambda r: r[0])
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.terminate()
                p.join()
    assert all(r[1] is not None for r in res), [r[4] for r in res]

    s = _sampler(shard_tiles=False)
    s.inference(in_dir, ref_dir, bs=len(shapes))
    names = sorted(p.name for p in ref_dir.iterdir())
    assert names == sorted(f"{n}.png" for n in shapes) and sorted(p.name for p in out_dir.iterdir()) == names
    for n in names:
        assert (out_dir / n).read_bytes() == (ref_dir / n).read_bytes(), n
    assert [r[2] for r in res] == [len(shapes)] + [0] * (world - 1)           # only rank 0 writes
    return res


def _check_team_rows(res, T):
    """Every member of a team of len(res) computed a non-empty row range in the encode and in the decode; the ranges are
    disjoint and cover all T rows."""
    for which in (0, 1):
        ranges = sorted(next((rb, re) for w, rb, re in r[3] if w == which) for r in res)
        assert all(len(r[3]) == 2 for r in res), [r[3] for r in res]
        assert all(re > rb for rb, re in ranges)
        assert ranges[0][0] == 0 and ranges[-1][1] == T and all(a[1] == b[0] for a, b in zip(ranges, ranges[1:])), ranges


def test_one_unit_three_ranks_gloo(tmp_path):
    res = _run(tmp_path, "gloo", 3, {"a": (128, 128)})
    assert [r[1] for r in res] == [[(128, 128)]] * 3                           # every member ran the whole unit
    _check_team_rows(res, 16384)


def test_two_units_three_ranks_gloo(tmp_path):
    """Units in file order: a (128x128) to ranks 0-1, b (128x192) to rank 2 alone (a team of one: no split)."""
    res = _run(tmp_path, "gloo", 3, {"a": (128, 128), "b": (128, 192)})
    assert [r[1] for r in res] == [[(128, 128)], [(128, 128)], [(128, 192)]]
    _check_team_rows(res[:2], 16384)
    assert res[2][3] == []


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_one_unit_two_gpus_nccl(tmp_path):
    res = _run(tmp_path, "nccl", 2, {"a": (128, 128)})
    _check_team_rows(res, 16384)
