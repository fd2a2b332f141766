"""Tile sharding (ResShiftSampler(shard_tiles=True)): the sample_func calls of a chunk of images are dealt across ranks,
every rank draws every unit's noise in the one-GPU order, and rank 0 averages the gathered tiles.  The output must be
bit-identical to a one-GPU run of the default path, whatever the number of ranks.

1. Virtual ranks in one process: each rank's share (_run_rank) after the same reseed, assembled in rank order, against
   the default _sample_tiled.
2. inference(bs=3) with two processes on one GPU under gloo, and 3. under NCCL on two GPUs: the PNG bytes against a
   one-GPU default inference().
4. A configuration that takes the generic per-step route is refused before any work."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CHOP = dict(tiny=dict(chop_size=64, chop_stride=48, padding_offset=64),           # 200x148 -> 4 x 3 = 12 tiles
            inpaint=dict(chop_size=256, chop_stride=192, padding_offset=256))     # 400x300 -> 2 x 2 = 4 tiles


def _sampler(kind, **kw):
    from resshift_b200.config import preset
    from resshift_b200.sampler import ResShiftSampler, make_configs
    from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
    from resshift_b200.weights import random_state_dict
    unet, sf = ("tiny", 4) if kind == "tiny" else ("tiny_inpaint", 1)
    ucfg, dcfg = preset(unet)
    dcfg.sf = sf
    vcfg = vq_preset("tiny")
    ae = {"target": "ldm.models.autoencoder.VQModelTorch", "params": vcfg.to_kwargs(), "ckpt_path": random_vq_state_dict(vcfg, 0)}
    configs = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    return ResShiftSampler(configs, sf=sf, use_amp=True, seed=123, **{**CHOP[kind], **kw})


@pytest.fixture(scope="module")
def samplers():
    return {k: _sampler(k) for k in CHOP}


def _chunk(kind):
    """Per shape group: lq [b, 3, h, w] in [-1, 1] and the mask (inpainting) or None.  The x4 chunk is three images in
    two shape groups: two that tile and one that fits in a tile (reflect-padded to 64x64)."""
    g = torch.Generator(device="cuda").manual_seed(8)
    shapes = [(2, 200, 148), (1, 60, 50)] if kind == "tiny" else [(1, 400, 300)]
    lqs = [torch.rand(b, 3, h, w, device="cuda", generator=g) * 2 - 1 for b, h, w in shapes]
    masks = [None] * len(lqs) if kind == "tiny" else \
        [(torch.rand(b, 1, h, w, device="cuda", generator=g) > 0.5).float() * 2 - 1 for b, h, w in shapes]
    return lqs, masks


CASES = [("tiny", 1, False), ("tiny", 1, True), ("tiny", 5, False), ("tiny", 5, True), ("inpaint", 1, False),
         ("inpaint", 5, True)]


@pytest.mark.parametrize("kind,chop_bs,noise_repeat", CASES)
def test_virtual_ranks_of_the_schedule_equal_one_gpu_default(samplers, kind, chop_bs, noise_repeat):
    from resshift_b200.parallel import unit_schedule
    from resshift_b200.sampler import tile_counts
    s = samplers[kind]
    s.chop_bs = chop_bs
    lqs, masks = _chunk(kind)
    s.setup_seed()
    ref = [s._sample_tiled(lq, mask=m, noise_repeat=noise_repeat) for lq, m in zip(lqs, masks)]

    ran = []
    orig = s._sample_unit

    def counted(y0, mask, noises, spec, replica):
        assert replica is None                                        # shard mode runs the sampler's own models
        ran.append(y0.shape[0])
        # the z_y shape and dtype derived from the configs (what every rank draws noise for) against the real encoder
        pad = s.padding_offset
        hp, wp = -(-y0.shape[2] // pad) * pad, -(-y0.shape[3] // pad) * pad
        z = s.base_diffusion.encode_first_stage(torch.zeros(y0.shape[0], 3, hp, wp, device="cuda"), s.autoencoder, up_sample=True)
        assert (tuple(z.shape), z.dtype) == spec
        return orig(y0, mask, noises, spec, replica)

    units = s._plan_units([tuple(lq.shape[2:]) for lq in lqs])
    if kind == "tiny":
        assert len(units) == {1: 13, 5: 4}[chop_bs]                   # 12 tiles of the pair (groups of 5, 5, 2) + 1
    s._sample_unit = counted
    try:
        for world in (1, 2, 5, 13):
            schedule = unit_schedule(len(units), world, teams=False)  # virtual ranks cannot exchange attention rows
            ran.clear()
            shares = []
            for rank in range(world):
                s.setup_seed()
                shares.append(s._run_rank(lqs, masks, noise_repeat, units, schedule, rank))
            assert ran == [lqs[u[0]].shape[0] * len(u[1]) for u in units]      # each unit ran once, in order
            counts = tile_counts(units, schedule, world)
            for g, (lq, r) in enumerate(zip(lqs, ref)):
                assert [sh[g].shape[0] for sh in shares] == counts[g]
                out = s._assemble(torch.cat([sh[g] for sh in shares]), *lq.shape[2:])
                assert out.shape == r.shape and torch.equal(out, r), (world, g, (out - r).abs().max().item())
    finally:
        s._sample_unit = orig


def _write_pngs(d):
    import cv2
    rng = np.random.default_rng(4)
    d.mkdir()
    for name, (h, w) in {"a_big": (200, 148), "b_small": (60, 50), "c_small": (40, 64)}.items():
        cv2.imwrite(str(d / f"{name}.png"), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))


def _worker(rank, world, port, backend, in_dir, out_dir, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world))
    import cv2
    import torch.distributed as dist
    try:
        if backend == "gloo":                                 # (NCCL: the sampler's setup_dist initialises it)
            dist.init_process_group("gloo", rank=rank, world_size=world)
        s = _sampler("tiny", chop_bs=2, shard_tiles=True)
        assert s.num_gpus == world and s.rank == rank and dist.get_backend() == backend
        ran, writes = [], []
        orig_unit, orig_write = s._sample_unit, cv2.imwrite
        s._sample_unit = lambda *a: (ran.append(a[0].shape[0]), orig_unit(*a))[1]
        cv2.imwrite = lambda *a: (writes.append(a[0]), orig_write(*a))[1]
        s.inference(in_dir, out_dir, bs=3)
        q.put((rank, len(ran), len(writes), ""))
    except Exception:                                         # noqa: BLE001 — report instead of hanging the parent
        import traceback
        q.put((rank, -1, -1, traceback.format_exc()))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _run_two_ranks(tmp_path, backend):
    import torch.multiprocessing as mp
    in_dir, out_dir, ref_dir = tmp_path / "in", tmp_path / "out", tmp_path / "ref"
    _write_pngs(in_dir)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, backend, str(in_dir), str(out_dir), q)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        res = sorted(q.get(timeout=900) for _ in procs)
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.terminate()
                p.join()
    assert all(r[1] >= 0 for r in res), res
    # 6 units of two tiles for the 200x148 image + one unit per small image: rank 0 runs units 0-3, rank 1 units 4-7
    assert [r[:3] for r in res] == [(0, 4, 3), (1, 4, 0)], res

    s = _sampler("tiny", chop_bs=2, shard_tiles=False)
    s.inference(in_dir, ref_dir, bs=3)
    names = sorted(p.name for p in ref_dir.iterdir())
    assert names == ["a_big.png", "b_small.png", "c_small.png"] and sorted(p.name for p in out_dir.iterdir()) == names
    for n in names:
        assert (out_dir / n).read_bytes() == (ref_dir / n).read_bytes(), n


def test_two_ranks_gloo_one_gpu_equal_one_gpu_default(tmp_path):
    _run_two_ranks(tmp_path, "gloo")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_gpus_nccl_equal_one_gpu_default(tmp_path):
    _run_two_ranks(tmp_path, "nccl")


def test_generic_route_is_refused_before_inference_or_run_rank_works(tmp_path, monkeypatch):
    """Without an autoencoder the reference clips x0 (clip_denoised=True), which takes the generic per-step route: its
    noise is drawn step by step inside the loop, so it cannot be drawn ahead for skipped units."""
    from resshift_b200.config import preset
    from resshift_b200.sampler import ResShiftSampler, make_configs
    from resshift_b200.weights import random_state_dict
    ucfg, dcfg = preset("tiny")
    dcfg.sf = 1
    configs = make_configs(ucfg, dcfg, autoencoder=None, state_dict=random_state_dict(ucfg, 0))
    monkeypatch.setenv("RS_SHARD_TILES", "1")
    s = ResShiftSampler(configs, sf=1, use_amp=True, seed=123, chop_size=64, chop_stride=48, padding_offset=64)
    assert s.shard_tiles

    def fail(*a, **k):
        raise AssertionError("work started before the configuration was refused")

    s._ingest_u8 = s._sample_unit = s.base_diffusion.encode_first_stage = s.base_diffusion.draw_noises = fail
    _write_pngs(tmp_path / "in")
    with pytest.raises(RuntimeError, match="generic per-step route"):
        s.inference(tmp_path / "in", tmp_path / "out", bs=3)
    assert not (tmp_path / "out").exists()
    with pytest.raises(RuntimeError, match="generic per-step route"):
        s._run_rank([torch.zeros(1, 3, 64, 64, device="cuda")], [None], False, s._plan_units([(64, 64)]), [(0, 1)], 0)
