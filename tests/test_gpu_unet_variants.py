"""GPU parity of UNetModelSwin built with the constructor options the shipped yaml files leave at one value
(use_scale_shift_norm=False, resblock_updown, conv_resample=False, patch_norm, cond_mask at latent size, dropout > 0):
forwards against the reference's goldens (tests/golden/unet_variants.npz) and the fp32 oracle, the fused 4-step loop,
every conv epilogue with the per-image bias, and the sampler's multi-GPU modes.  Bounds are those of test_gpu_unet.py."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import unet_variants_oracle as uo
from oracle.make_golden_variants import OUT_STRIDE, VARIANTS, trajectory_inputs, variant_config, variant_inputs
from resshift_b200.config import UNetConfig
from resshift_b200.weights import random_state_dict

FWD_MAX, FWD_MEAN = 1e-2, 2.5e-3
LOOP_MAX, LOOP_MEAN = 1e-2, 3e-3


def _model(ucfg, seed=0):
    from resshift_b200.models.unet import UNetModelSwin
    m = UNetModelSwin(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, seed), strict=True)
    return m.cuda().eval()


def _check(tag, got, ref, bmax=FWD_MAX, bmean=FWD_MEAN):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    print(f"[parity] {tag}: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e}")
    assert not torch.isnan(got).any()
    assert d.max().item() <= bmax and d.mean().item() <= bmean, tag


def _cuda(*ts):
    return [None if t is None else t.cuda() for t in ts]


@pytest.mark.parametrize("tag", list(VARIANTS) + ["combined_64x128"])
def test_forward_vs_reference_golden(golden_dir, tag):
    g = np.load(golden_dir / "unet_variants.npz")
    ucfg, _ = variant_config(tag.split("_64x128")[0])
    seed, h, w = (int(v) for v in g[f"{tag}/seed"])
    x, lq, mask = _cuda(*variant_inputs(ucfg, 2, h, w, seed))
    out = _model(ucfg)(x, torch.from_numpy(g[f"{tag}/t"]).cuda(), lq=lq, mask=mask)
    _check(f"golden {tag}", out.reshape(-1)[::OUT_STRIDE], torch.from_numpy(g[f"{tag}/out_sub"]))


@pytest.mark.parametrize("name", list(VARIANTS))
def test_forward_vs_oracle_fresh_inputs(name):
    ucfg, _ = variant_config(name)
    x, lq, mask = variant_inputs(ucfg, 2, 64, 64, 9000)
    t = torch.tensor([0, 3])
    ref = uo.unet_forward(random_state_dict(ucfg, 0), ucfg, x, t, lq=lq, mask=mask)
    x, lq, mask, t = _cuda(x, lq, mask, t)
    _check(f"oracle {name}", _model(ucfg)(x, t, lq=lq, mask=mask), ref)


def test_combined_fused_loop_vs_reference_trajectory(golden_dir):
    from resshift_b200.models.script_util import create_gaussian_diffusion
    g = np.load(golden_dir / "unet_variants.npz")
    ucfg, dcfg = variant_config("combined")
    m = _model(ucfg)
    diff = create_gaussian_diffusion(**dcfg.to_kwargs())
    assert diff._native_ok(m, clip_denoised=False, denoised_fn=None, model_kwargs={"lq": None})
    y, noises = _cuda(*trajectory_inputs(2, dcfg.steps))
    finals = [diff.sample_latent(y, m, {"lq": y}, noises=noises).clone() for _ in range(2)]   # capture, then replay
    assert torch.equal(finals[0], finals[1])
    _check("loop combined", finals[0].reshape(-1)[::OUT_STRIDE], torch.from_numpy(g["loop/final_sub"]), LOOP_MAX, LOOP_MEAN)


@pytest.fixture(scope="module")
def realsr_combined():
    ucfg = UNetConfig(**VARIANTS["combined"])               # realsr width: model_channels 160, swin_embed_dim 192
    return ucfg, random_state_dict(ucfg, 0), _model(ucfg)


def test_realsr_width_combined_vs_fp32_oracle_on_gpu(realsr_combined):
    ucfg, sd, m = realsr_combined
    gen = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(2, 3, 64, 64, device="cuda", generator=gen)
    lq = torch.rand(2, 3, 64, 64, device="cuda", generator=gen) * 2 - 1
    t = torch.tensor([1, 12], device="cuda")
    tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        ref = uo.unet_forward({k: v.cuda() for k, v in sd.items()}, ucfg, x, t, lq=lq)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    _check("realsr-width combined", m(x, t, lq=lq), ref)


def test_realsr_width_combined_batch16_images_are_independent(realsr_combined):
    """Batch 16 with 16 different timesteps (one per-image bias row each).  Image i is bit-identical whatever its batch
    neighbours are; a batch-1 run agrees to rounding only, as for the shipped topology (the planner picks other tile
    shapes / split-K factors for other batch sizes)."""
    _, _, m = realsr_combined
    gen = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn(16, 3, 64, 64, device="cuda", generator=gen)
    lq = torch.rand(16, 3, 64, 64, device="cuda", generator=gen) * 2 - 1
    t = torch.arange(16, device="cuda") % 15
    full = m(x, t, lq=lq).clone()
    assert not torch.isnan(full).any()
    x2, lq2, t2 = torch.randn_like(x), torch.rand_like(lq) * 2 - 1, torch.flip(t, (0,))
    for i in range(16):
        x2[i], lq2[i], t2[i] = x[i], lq[i], t[i]
        other = m(x2, t2, lq=lq2)
        assert torch.equal(other[i], full[i]), f"image {i} depends on its batch neighbours"
        x2[i], lq2[i], t2[i] = torch.randn_like(x[i]), torch.rand_like(lq[i]) * 2 - 1, t[15 - i]
    for i in (0, 9):
        _check(f"batch-16 vs batch-1 image {i}", m(x[i:i + 1], t[i:i + 1], lq=lq[i:i + 1]), full[i:i + 1], 1e-2, 1e-3)


@pytest.mark.parametrize("knob", [("RS_CONV_EPI", "direct"), ("RS_CONV_PERSIST", "1"), ("RS_CONV_SPLITK", "2"),
                                  ("RS_CONV_CG", "2"), ("RS_CONV_IMPL", "simt")])
def test_scale_shift_off_through_every_epilogue(monkeypatch, knob):
    """The per-image bias (h + emb_out in in_layers.2's epilogue) with each epilogue forced at plan build."""
    monkeypatch.setenv(*knob)
    ucfg, _ = variant_config("scale_shift_off")
    x, lq, _ = variant_inputs(ucfg, 2, 64, 64, 9100)
    t = torch.tensor([3, 0])
    ref = uo.unet_forward(random_state_dict(ucfg, 0), ucfg, x, t, lq=lq)
    x, lq, t = _cuda(x, lq, t)
    _check(f"scale_shift_off {knob[0]}={knob[1]}", _model(ucfg)(x, t, lq=lq), ref)


def test_create_ex_with_shipped_options_equals_create(monkeypatch):
    from resshift_b200 import _lib
    ucfg, _ = variant_config("scale_shift_off")
    ucfg.use_scale_shift_norm = True                        # the tiny preset: the shipped options {1, 0, 1, 0}
    x, lq, _ = _cuda(*variant_inputs(ucfg, 2, 64, 64, 9200))
    t = torch.tensor([2, 1], device="cuda")
    a = _model(ucfg)(x, t, lq=lq)
    monkeypatch.setattr(_lib.lib, "rs_unet_create_ex", lambda cfg, opt, out: _lib.lib.rs_unet_create(cfg, out))
    b = _model(ucfg)(x, t, lq=lq)
    assert torch.equal(a, b)
    o = _lib.make_options(ucfg)
    assert (o.use_scale_shift_norm, o.resblock_updown, o.conv_resample, o.patch_norm) == (1, 0, 1, 0)


# ------------------------------------------------------------------------------------------------ the whole pipeline

def _sampler(devices=None):
    from resshift_b200.sampler import ResShiftSampler, make_configs
    from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
    ucfg, dcfg = variant_config("combined")
    dcfg.sf = 4
    vcfg = vq_preset("tiny")
    ae = {"target": "ldm.models.autoencoder.VQModelTorch", "params": vcfg.to_kwargs(), "ckpt_path": random_vq_state_dict(vcfg, 0)}
    configs = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    return ResShiftSampler(configs, sf=4, use_amp=True, seed=123, devices=devices, chop_size=64, chop_stride=48,
                           padding_offset=64)


def test_sampler_virtual_ranks_and_pool_equal_one_gpu(tmp_path):
    import cv2
    from resshift_b200.parallel import unit_schedule
    from resshift_b200.sampler import tile_counts
    s = _sampler()
    assert s.base_diffusion._native_ok(s.model, clip_denoised=False, denoised_fn=None, model_kwargs={"lq": None})
    gen = torch.Generator(device="cuda").manual_seed(8)
    lqs = [torch.rand(b, 3, h, w, device="cuda", generator=gen) * 2 - 1 for b, h, w in [(2, 200, 148), (1, 60, 50)]]
    s.setup_seed()
    ref = [s._sample_tiled(lq, mask=None, noise_repeat=False) for lq in lqs]
    units = s._plan_units([tuple(lq.shape[2:]) for lq in lqs])
    for world in (2, 5):
        schedule = unit_schedule(len(units), world, teams=False)
        shares = []
        for rank in range(world):
            s.setup_seed()
            shares.append(s._run_rank(lqs, [None, None], False, units, schedule, rank))
        counts = tile_counts(units, schedule, world)
        for gi, (lq, r) in enumerate(zip(lqs, ref)):
            assert [sh[gi].shape[0] for sh in shares] == counts[gi]
            assert torch.equal(s._assemble(torch.cat([sh[gi] for sh in shares]), *lq.shape[2:]), r), (world, gi)

    rng = np.random.default_rng(7)
    (tmp_path / "in").mkdir()
    for name, (h, w) in {"a1": (200, 148), "a2": (200, 148), "b": (60, 50)}.items():
        cv2.imwrite(str(tmp_path / "in" / f"{name}.png"), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
    outs = []
    for smp, d in ((s, "ref"), (_sampler("0,0"), "pool")):
        smp.setup_seed()
        smp.inference(tmp_path / "in", tmp_path / d, bs=3)
        outs.append({p.name: p.read_bytes() for p in sorted((tmp_path / d).iterdir())})
    assert len(outs[0]) == 3 and outs[0] == outs[1]
