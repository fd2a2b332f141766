"""Device pool (ResShiftSampler(devices=...)): one process runs a chunk's work units on several model replicas, one
thread and one stream each, with every unit's noise drawn on the primary in one-GPU order.  The PNGs must be
byte-identical to a one-GPU default inference().

On one GPU the pools are virtual (the same device listed several times: separate replicas, streams and threads):
1. the three-image x4 chunk in two shape groups, chop_bs 1 and 5, noise_repeat off and on, pools of 2 and 3 — every
   unit runs exactly once, on more than one replica;
2. inpainting with masks and mask_back (with chop_bs 5 the chunk is one unit: a team without a fused attention);
3. one 128x128 LQ image (T = 16384) on a pool of 3: one team that splits the bottleneck attention's query rows;
4. an exception inside a worker reaches the caller and stops the other workers, also inside a team exchange.
With two GPUs: devices="all", a second device in the same process, and a plan run on the wrong device."""
import threading

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CHOP = dict(tiny=dict(chop_size=64, chop_stride=48, padding_offset=64),           # 200x148 -> 4 x 3 = 12 tiles
            inpaint=dict(chop_size=256, chop_stride=192, padding_offset=256),     # 400x300 -> 2 x 2 = 4 tiles
            team=dict(chop_size=512, chop_stride=448, padding_offset=16))         # 128x128 x4: one unit, T = 16384


def _sampler(kind, devices=None, **kw):
    from resshift_b200.config import preset
    from resshift_b200.sampler import ResShiftSampler, make_configs
    from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
    from resshift_b200.weights import random_state_dict
    unet, sf = ("tiny_inpaint", 1) if kind == "inpaint" else ("tiny", 4)
    ucfg, dcfg = preset(unet)
    dcfg.sf = sf
    vcfg = vq_preset("tiny")
    ae = {"target": "ldm.models.autoencoder.VQModelTorch", "params": vcfg.to_kwargs(), "ckpt_path": random_vq_state_dict(vcfg, 0)}
    configs = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    return ResShiftSampler(configs, sf=sf, use_amp=True, seed=123, devices=devices, **{**CHOP[kind], **kw})


@pytest.fixture(scope="module")
def samplers():
    """kind -> {pool size (0: the default path): sampler}"""
    return {kind: {0: _sampler(kind), 2: _sampler(kind, "0,0"), 3: _sampler(kind, [0, 0, 0])} for kind in CHOP}


IMAGES = dict(tiny={"a1": (200, 148), "a2": (200, 148), "b": (60, 50)},       # two shape groups
              inpaint={"p": (400, 300), "q": (400, 300)},
              team={"t": (128, 128)},
              team2={"t": (128, 128), "u": (128, 128)})                      # one unit of two images: N = 2


def _write(d, kind, images=None):
    import cv2
    rng = np.random.default_rng(7)
    (d / "in").mkdir()
    (d / "mask").mkdir()
    for name, (h, w) in IMAGES[images or kind].items():
        cv2.imwrite(str(d / "in" / f"{name}.png"), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        cv2.imwrite(str(d / "mask" / f"{name}.png"), (rng.random((h, w)) > 0.5).astype(np.uint8) * 255)


def _infer(s, d, kind, out, noise_repeat=False, images=None):
    """inference() from the sampler's seed (as right after its construction: the generators are process-wide)."""
    s.setup_seed()
    mask = d / "mask" if kind == "inpaint" else None
    s.inference(d / "in", d / out, mask_path=mask, mask_back=True, bs=len(IMAGES[images or kind]),
                noise_repeat=noise_repeat)
    return {p.name: p.read_bytes() for p in sorted((d / out).iterdir())}


def _instrument(s):
    """Wraps s._sample_unit: records (replica index, batch, h, w) of every call."""
    ran, orig = [], s._sample_unit

    def counted(y0, mask, noises, spec, replica):
        ran.append((None if replica is None else replica.index, y0.shape[0]) + tuple(y0.shape[2:]))
        return orig(y0, mask, noises, spec, replica)
    s._sample_unit = counted
    return ran, orig


@pytest.mark.parametrize("pool", [2, 3])
@pytest.mark.parametrize("chop_bs,noise_repeat", [(1, False), (1, True), (5, False), (5, True)])
def test_x4_chunk_equals_one_gpu(samplers, tmp_path, pool, chop_bs, noise_repeat):
    ref_s, s = samplers["tiny"][0], samplers["tiny"][pool]
    ref_s.chop_bs = s.chop_bs = chop_bs
    _write(tmp_path, "tiny")
    ref = _infer(ref_s, tmp_path, "tiny", "ref", noise_repeat)
    ran, orig = _instrument(s)
    try:
        out = _infer(s, tmp_path, "tiny", "out", noise_repeat)
    finally:
        s._sample_unit = orig
    assert sorted(ref) == ["a1.png", "a2.png", "b.png"] and out == ref
    units = s._plan_units([(200, 148), (60, 50)])
    assert len(units) == {1: 13, 5: 4}[chop_bs]                    # 12 tiles of the pair (groups of 5, 5, 2) + 1
    expected = sorted((2 if g == 0 else 1) * len(starts) for g, starts, _, _ in units)
    assert sorted(r[1] for r in ran) == expected                 # every unit ran exactly once
    assert all(r[0] is not None for r in ran), ran
    if chop_bs == 1:
        # 13 units: a worker holds at most one unit beyond the one its device runs, so the others get units too
        # (with 4 units, dealing by progress may in principle leave a replica without one)
        assert len({r[0] for r in ran}) > 1, ran


@pytest.mark.parametrize("pool", [2, 3])
@pytest.mark.parametrize("chop_bs", [1, 5])
def test_inpainting_with_mask_back_equals_one_gpu(samplers, tmp_path, pool, chop_bs):
    ref_s, s = samplers["inpaint"][0], samplers["inpaint"][pool]
    ref_s.chop_bs = s.chop_bs = chop_bs
    _write(tmp_path, "inpaint")
    ref = _infer(ref_s, tmp_path, "inpaint", "ref")
    ran, orig = _instrument(s)
    try:
        out = _infer(s, tmp_path, "inpaint", "out")
    finally:
        s._sample_unit = orig
    assert sorted(ref) == ["p.png", "q.png"] and out == ref
    n_units = len(s._plan_units([(400, 300)]))
    assert n_units == {1: 4, 5: 1}[chop_bs]
    # one unit: a team of every replica, each running the whole unit (no fused attention to split at this size)
    assert len(ran) == (n_units if n_units >= pool else pool)
    if n_units < pool:
        assert sorted(r[0] for r in ran) == list(range(pool))


def _check_team(ref_s, s, tmp_path, images):
    """inference() of one unit (the images of ``images``, one 128x128 shape group) on the team of all of s's replicas:
    PNG bytes equal the default path's, every member ran the whole unit, and the members' attention rows tile [0, T)."""
    _write(tmp_path, "team", images)
    ref = _infer(ref_s, tmp_path, "team", "ref", images=images)
    ran, orig = _instrument(s)
    try:
        out = _infer(s, tmp_path, "team", "out", images=images)
    finally:
        s._sample_unit = orig
    n = len(IMAGES[images])
    assert sorted(ref) == sorted(f"{k}.png" for k in IMAGES[images]) and out == ref
    assert sorted(ran) == [(r, n, 128, 128) for r in range(len(s.pool.replicas))]
    rows = [rep.autoencoder.attention_rows for rep in s.pool.replicas]
    for which in (0, 1):                                        # encode, decode: disjoint, non-empty, covering [0, T)
        ranges = sorted(next((rb, re) for w, rb, re in r if w == which) for r in rows)
        assert all(len(r) == 2 for r in rows), rows
        assert all(re > rb for rb, re in ranges)
        assert ranges[0][0] == 0 and ranges[-1][1] == 16384 and all(a[1] == b[0] for a, b in zip(ranges, ranges[1:])), ranges


@pytest.mark.parametrize("images", ["team", "team2"])
def test_one_unit_runs_on_a_team_of_three(samplers, tmp_path, images):
    """One image (attention view [1, T, C]) and two of the same shape in one unit ([2, T, C]: the rows of a member are
    a strided slice, staged through a dense buffer by the exchange)."""
    _check_team(samplers["team"][0], samplers["team"][3], tmp_path, images)


def _pool_threads():
    return [t for t in threading.enumerate() if t.name.startswith("rs-device-pool-")]


@pytest.mark.parametrize("kind,pool,failing", [("tiny", 2, "second call"), ("team", 3, "member 1")])
def test_worker_error_reaches_the_caller(samplers, tmp_path, kind, pool, failing):
    """The error of one worker is raised by inference(); the other workers stop (team members waiting in the exchange
    are released); nothing is left running, and the pool computes correctly afterwards."""
    ref_s, s = samplers[kind][0], samplers[kind][pool]
    ref_s.chop_bs = s.chop_bs = 1
    _write(tmp_path, kind)
    calls, orig = [], s._sample_unit

    def boom(y0, mask, noises, spec, replica):
        calls.append(replica.index)
        if (failing == "second call" and len(calls) == 2) or (failing == "member 1" and replica.index == 1):
            raise RuntimeError("boom in a pool worker")
        return orig(y0, mask, noises, spec, replica)
    s._sample_unit = boom
    try:
        with pytest.raises(RuntimeError, match="boom in a pool worker"):
            _infer(s, tmp_path, kind, "out")
    finally:
        s._sample_unit = orig
    assert _pool_threads() == []
    assert _infer(s, tmp_path, kind, "out2") == _infer(ref_s, tmp_path, kind, "ref")


def test_pool_of_one_is_the_default_path(samplers, tmp_path):
    s = _sampler("tiny", devices="0")
    s.chop_bs = samplers["tiny"][0].chop_bs = 1
    assert len(s.pool.replicas) == 1
    _write(tmp_path, "tiny")
    assert _infer(s, tmp_path, "tiny", "out") == _infer(samplers["tiny"][0], tmp_path, "tiny", "ref")


# ---------------------------------------------------------------------------------------------------------------------
two_gpus = pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")


@two_gpus
def test_all_devices_equal_one_gpu(samplers, tmp_path):
    s = _sampler("tiny", devices="all")
    assert [r.device.index for r in s.pool.replicas] == list(range(torch.cuda.device_count()))
    s.chop_bs = samplers["tiny"][0].chop_bs = 1
    _write(tmp_path, "tiny")
    assert _infer(s, tmp_path, "tiny", "out") == _infer(samplers["tiny"][0], tmp_path, "tiny", "ref")


@two_gpus
@pytest.mark.parametrize("images", ["team", "team2"])
def test_team_across_two_devices(samplers, tmp_path, images):
    """One unit on a team of cuda:0 and cuda:1: the exchange copies attention rows between devices, for one image and
    for two in the unit (a strided [2, T, C] row slice)."""
    _check_team(samplers["team"][0], _sampler("team", devices="0,1"), tmp_path, images)


@two_gpus
def test_arena_of_another_device_is_refused():
    import ctypes as C
    from resshift_b200 import _lib
    from resshift_b200.vq_arch import vq_preset
    from resshift_b200.models.autoencoder import VQModelTorch
    vq = VQModelTorch(**vq_preset("tiny").to_kwargs())
    h = C.c_void_p()
    _lib.check(_lib.lib.rs_vq_create(C.byref(_lib.make_vq_config(vq.cfg)), C.byref(h)))
    try:
        arena = torch.empty(_lib.lib.rs_unet_arena_bytes(h) + 256, dtype=torch.uint8, device="cuda:1")
        ptr = (arena.data_ptr() + 255) // 256 * 256
        with torch.cuda.device(0):
            with pytest.raises(_lib.RsError, match="the arena is memory of cuda:1 but cuda:0 is current"):
                _lib.check(_lib.lib.rs_unet_set_arena(h, ptr))
        with torch.cuda.device(1):
            _lib.check(_lib.lib.rs_unet_set_arena(h, ptr))
    finally:
        _lib.lib.rs_unet_destroy(h)
    # a model on cuda:1 first used while cuda:0 is current: its engine belongs to cuda:1
    unet, vq = _models("cuda:1")
    with torch.cuda.device(0):
        vq._ensure_engine(torch.device("cuda:1"))
        unet._ensure_engine(torch.device("cuda:1"))
    with torch.cuda.device(1):
        ref = _run_models(unet, vq, "cuda:1")
        torch.cuda.synchronize()
    assert all(torch.isfinite(r).all() for r in ref)


def _models(device):
    from resshift_b200.config import preset
    from resshift_b200.models.autoencoder import VQModelTorch
    from resshift_b200.models.unet import UNetModelSwin
    from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
    from resshift_b200.weights import random_state_dict
    ucfg, _ = preset("tiny")
    vcfg = vq_preset("tiny")
    unet = UNetModelSwin(**ucfg.to_kwargs())
    unet.load_state_dict(random_state_dict(ucfg, 0))
    vq = VQModelTorch(**vcfg.to_kwargs())
    vq.load_state_dict(random_vq_state_dict(vcfg, 0))
    return unet.to(device).eval(), vq.to(device).eval()


def _run_models(unet, vq, device):
    g = torch.Generator().manual_seed(3)
    img = (torch.rand(1, 3, 512, 512, generator=g) * 2 - 1).to(device)          # 128x128 bottleneck: fused attention
    x = torch.randn(2, 3, 64, 64, generator=g).to(device)
    lq = (torch.rand(2, 3, 64, 64, generator=g) * 2 - 1).to(device)
    t = torch.tensor([3, 1], device=device)
    h = vq.encode(img)
    assert vq.plan(0, 1, 512, 512).attention is not None
    return h.cpu(), unet(x, t, lq=lq).cpu()


@two_gpus
def test_second_device_in_the_same_process():
    """The large kernels' shared-memory opt-in is a per-device attribute: after cuda:0 has run, the fused VQ attention
    and the denoiser must launch on cuda:1 as well, with the same results."""
    ref = _run_models(*_models("cuda:0"), "cuda:0")
    with torch.cuda.device(1):
        out = _run_models(*_models("cuda:1"), "cuda:1")
        torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(ref, out))


@two_gpus
def test_plan_run_on_another_device_is_an_error():
    from resshift_b200 import _lib
    unet, vq = _models("cuda:0")
    _run_models(unet, vq, "cuda:0")
    plan = unet.plan(2, 64, 64)
    x = torch.zeros(2, 3, 64, 64, device="cuda:0")
    t = torch.zeros(2, device="cuda:0")
    with torch.cuda.device(1):
        rc = _lib.lib.rs_plan_forward(plan.handle, x.data_ptr(), t.data_ptr(), x.data_ptr(), None, x.data_ptr(),
                                      _lib.current_stream())
        assert rc != 0 and b"bound on cuda:0 but cuda:1 is current" in _lib.lib.rs_last_error()
        with pytest.raises(_lib.RsError, match="a plan runs on the device it was bound on"):
            vq.encode(torch.zeros(1, 3, 512, 512, device="cuda:0"))
    torch.cuda.synchronize(0)
