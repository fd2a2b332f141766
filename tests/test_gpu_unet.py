"""GPU parity of the whole hot path (denoiser forward + residual-shift loop) against
(a) the committed golden vectors produced by the reference itself and (b) the CPU oracle on fresh seeded
inputs; plus size-independent properties at the benchmark batch size.

Tolerance.  BASELINE.json's north_star states the bar for this floating-point path: results match the
reference "within fp16 tolerance (per-pixel |delta| <= 1e-2 ...)".  The kernels store activations in fp16
(fp32 accumulation, fp32 GroupNorm / softmax statistics) exactly like the reference under
torch.cuda.amp.autocast (reference sampler.py:185), while the oracle / goldens are fp32.  Against fp32 the
expected deviation of an fp16-activation network of this depth is a few 1e-3 on outputs of std ~0.6; the
tests hold every comparison to the north-star figure itself — max|d| <= 1e-2 — for one forward AND for the
final latent / per-step tensors of the sampling loops (errors compound through x_t), with mean|d| <= 2.5e-3
(forward) and 3e-3 (loop).  Measured values are printed.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from resshift_b200.config import preset
from resshift_b200.weights import random_state_dict

FWD_MAX, FWD_MEAN = 1e-2, 2.5e-3
LOOP_MAX, LOOP_MEAN = 1e-2, 3e-3


def _model(name, seed=0):
    from resshift_b200.models.unet import UNetModelSwin
    ucfg, dcfg = preset(name)
    m = UNetModelSwin(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, seed), strict=True)
    return ucfg, dcfg, m.cuda().eval()


def _report(tag, got, ref):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    print(f"[parity] {tag}: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e} ref_std={ref.float().std().item():.3f}")
    return d.max().item(), d.mean().item()


@pytest.mark.parametrize("name,fname", [("tiny", "unet_tiny.npz"), ("tiny_inpaint", "unet_tiny_inpaint.npz"),
                                         ("tiny_faceir", "unet_tiny_faceir.npz"), ("realsr", "unet_realsr.npz"),
                                         ("faceir", "unet_faceir.npz"), ("inpaint", "unet_inpaint.npz"),
                                         ("realsr", "unet_realsr_64x128.npz"), ("tiny", "unet_tiny_128x64.npz")])
def test_forward_vs_reference_golden(golden_dir, name, fname):
    from tests.golden_util import golden_inputs
    g = np.load(golden_dir / fname)
    ucfg, _, m = _model(name)
    x, t, lq, mask = golden_inputs(g)
    x, t, lq = x.cuda(), t.cuda(), lq.cuda()
    mask = None if mask is None else mask.cuda()
    out = m(x, t, lq=lq, mask=mask)
    assert not torch.isnan(out).any()
    mx, mn = _report(f"forward {name}", out, torch.from_numpy(g["out"]))
    assert mx <= FWD_MAX and mn <= FWD_MEAN


def test_forward_blocks_vs_golden(golden_dir):
    """Block-by-block comparison (sub-sampled probes of the reference) to localise a divergence."""
    os.environ["RS_NO_REUSE"] = "1"
    try:
        g = np.load(golden_dir / "unet_tiny.npz")
        ucfg, _, m = _model("tiny")
        x, t, lq = (torch.from_numpy(g[k]).cuda() for k in ("x", "t", "lq"))
        m(x, t, lq=lq)
        worst = 0.0
        for key in g.files:
            if not key.startswith("probe_sub/"):
                continue
            blk = key.split("/", 1)[1]
            got = m.probe(x.shape[0], 64, 64, blk).reshape(-1)[::37].cpu().numpy()
            d = np.abs(got - g[key]).max()
            print(f"[parity] block {blk}: max|d|={d:.3e} (ref absmax {np.abs(g[key]).max():.2f})")
            worst = max(worst, d / max(1.0, np.abs(g[key]).max()))
        assert worst <= 2e-2
    finally:
        os.environ.pop("RS_NO_REUSE", None)


def test_norm2_fused_into_mlp_is_bit_identical_to_separate_groupnorm():
    """The fused Swin MLP kernel applying norm2 to its X tile in shared memory (RS_MLP_NORM_FUSE=1) must reproduce, bit for bit,
    the plan that runs gn_apply_kernel first (RS_MLP_NORM_FUSE=0): same partial sums, same affine, same rounding."""
    outs = []
    for fuse in ("1", "0"):
        os.environ["RS_MLP_NORM_FUSE"] = fuse
        try:
            ucfg, _, m = _model("realsr")
            g = torch.Generator(device="cuda").manual_seed(7)
            x = torch.randn(3, 3, 64, 64, device="cuda", generator=g)
            lq = torch.rand(3, 3, 64, 64, device="cuda", generator=g) * 2 - 1
            t = torch.tensor([2, 9, 14], device="cuda")
            outs.append((m(x, t, lq=lq).clone(), m.num_launches(3, 64, 64)))
            del m
        finally:
            os.environ.pop("RS_MLP_NORM_FUSE", None)
    assert outs[0][1] == outs[1][1] - 18, (outs[0][1], outs[1][1])      # one launch less per Swin block
    assert not torch.isnan(outs[0][0]).any() and torch.equal(outs[0][0], outs[1][0])


def test_fused_swin_attention_plan_matches_four_launch_plan(monkeypatch):
    """The fused Swin attention kernel (norm1 + qkv + window attention + proj + residual in one launch) against the
    four-launch form of the same half, at plan level and WITH workspace reuse: forced on every level
    (RS_SWIN_FUSE_MIN_PAIRS=1: 18 blocks x 3 launches fewer) vs off.  Same roundings, different summation orders: the
    outputs agree to rounding; the fused plan is bit-reproducible and right against the oracle.  Batch 3 puts several
    images and an odd window count (8x8 level: 3 windows) into one CTA's range."""
    from oracle import unet_oracle as uo
    outs = {}
    for thr in ("1", "1000000"):
        monkeypatch.setenv("RS_SWIN_FUSE_MIN_PAIRS", thr)
        ucfg, _, m = _model("realsr")
        g = torch.Generator(device="cuda").manual_seed(11)
        x = torch.randn(3, 3, 64, 64, device="cuda", generator=g)
        lq = torch.rand(3, 3, 64, 64, device="cuda", generator=g) * 2 - 1
        t = torch.tensor([1, 8, 14], device="cuda")
        a = m(x, t, lq=lq).clone()
        b = m(x, t, lq=lq).clone()
        assert torch.equal(a, b) and not torch.isnan(a).any()
        outs[thr] = (a, m.num_launches(3, 64, 64))
        del m
    assert outs["1"][1] == outs["1000000"][1] - 54, (outs["1"][1], outs["1000000"][1])
    d = (outs["1"][0] - outs["1000000"][0]).abs()
    print(f"[property] fused vs four-launch Swin attention: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e}")
    assert d.max().item() <= 1e-2 and d.mean().item() <= 1.5e-3
    sd = random_state_dict(ucfg, 0)
    ref = uo.unet_forward(sd, ucfg, x.cpu(), t.cpu(), lq=lq.cpu())
    mx, mn = _report("forward realsr, fused Swin attention on every level", outs["1"][0], ref)
    assert mx <= FWD_MAX and mn <= FWD_MEAN


def test_forward_vs_oracle_fresh_inputs():
    """Oracle on new seeded inputs (not in the goldens), batch 3 with distinct timesteps."""
    from oracle import unet_oracle as uo
    ucfg, _, m = _model("tiny", seed=3)
    sd = random_state_dict(ucfg, 3)
    g = torch.Generator().manual_seed(99)
    x = torch.randn(3, 3, 64, 64, generator=g)
    lq = torch.rand(3, 3, 64, 64, generator=g) * 2 - 1
    t = torch.tensor([0, 2, 3])
    ref = uo.unet_forward(sd, ucfg, x, t, lq=lq)
    out = m(x.cuda(), t.cuda(), lq=lq.cuda())
    mx, mn = _report("forward tiny fresh", out, ref)
    assert mx <= FWD_MAX and mn <= FWD_MEAN


@pytest.mark.parametrize("name", ["faceir", "inpaint"])
def test_forward_full_size_other_tasks_vs_oracle(name):
    """BASELINE configs 4 / 5 at full width: face restoration (8 latent channels, 512x512 LQ through the three-stage
    feature extractor) and inpainting (LQ + mask at 256x256, two-stage extractor), batch 2 with distinct timesteps,
    against the CPU oracle on fresh seeded inputs."""
    from oracle import unet_oracle as uo
    ucfg, _, m = _model(name, seed=5)
    sd = random_state_dict(ucfg, 5)
    g = torch.Generator().manual_seed(55)
    x = torch.randn(2, ucfg.out_channels, 64, 64, generator=g)
    lq = torch.rand(2, 3, ucfg.lq_size, ucfg.lq_size, generator=g) * 2 - 1
    mask = (torch.rand(2, 1, ucfg.lq_size, ucfg.lq_size, generator=g) > 0.5).float() * 2 - 1 if ucfg.cond_mask else None
    t = torch.tensor([0, 3])
    ref = uo.unet_forward(sd, ucfg, x, t, lq=lq, mask=mask)
    out = m(x.cuda(), t.cuda(), lq=lq.cuda(), mask=None if mask is None else mask.cuda())
    assert not torch.isnan(out).any()
    mx, mn = _report(f"forward {name} full size", out, ref)
    assert mx <= FWD_MAX and mn <= FWD_MEAN


def test_forward_rectangular_latent():
    """Non-square latent (chopped tiles / padded inputs): H=64, W=128."""
    from oracle import unet_oracle as uo
    ucfg, _, m = _model("tiny", seed=4)
    sd = random_state_dict(ucfg, 4)
    g = torch.Generator().manual_seed(100)
    x = torch.randn(1, 3, 64, 128, generator=g)
    lq = torch.rand(1, 3, 64, 128, generator=g) * 2 - 1
    t = torch.tensor([1])
    ref = uo.unet_forward(sd, ucfg, x, t, lq=lq)
    out = m(x.cuda(), t.cuda(), lq=lq.cuda())
    mx, mn = _report("forward tiny 64x128", out, ref)
    assert mx <= FWD_MAX and mn <= FWD_MEAN


def _loop(golden_dir, name, steps, fname, use_graph):
    from resshift_b200.models.script_util import create_gaussian_diffusion
    from tests.golden_util import golden_loop_inputs
    g = np.load(golden_dir / fname)
    ucfg, dcfg, m = _model(name)
    dcfg.steps, dcfg.sf = steps, 1
    diff = create_gaussian_diffusion(**dcfg.to_kwargs())
    y, noises = (v.cuda() for v in golden_loop_inputs(g))
    final = diff.sample_latent(y, m, {"lq": y}, noises=noises, use_graph=use_graph)
    return g, diff, m, y, noises, final


@pytest.mark.parametrize("use_graph", [False, True])
def test_loop_tiny_vs_reference_golden(golden_dir, use_graph):
    g, diff, m, y, noises, final = _loop(golden_dir, "tiny", 4, "loop_tiny_T4.npz", use_graph)
    mx, mn = _report(f"loop tiny T4 graph={use_graph}", final, torch.from_numpy(g["final"]))
    assert mx <= LOOP_MAX and mn <= LOOP_MEAN


def test_loop_realsr_15_vs_reference_golden(golden_dir):
    g, diff, m, y, noises, final = _loop(golden_dir, "realsr", 15, "loop_realsr_T15.npz", True)
    mx, mn = _report("loop realsr T15 (final latent)", final, torch.from_numpy(g["final"]))
    assert mx <= LOOP_MAX and mn <= LOOP_MEAN
    # per-step taps through the progressive generator (same native loop, with taps)
    import resshift_b200.models.gaussian_diffusion as gd
    orig = diff.draw_noises
    diff.draw_noises = lambda z_y, noise=None, noise_repeat=False: noises
    try:
        rec = list(diff.p_sample_loop_progressive(y, m, first_stage_model=None, noise=noises[0], clip_denoised=False,
                                                  model_kwargs={"lq": y}))
    finally:
        diff.draw_noises = orig
    assert len(rec) == 15
    for k in (0, 7, 14):
        mx, mn = _report(f"loop realsr pred_xstart step {k}", rec[k]["pred_xstart"], torch.from_numpy(g[f"pred_xstart/{k}"]))
        assert mx <= LOOP_MAX and mn <= LOOP_MEAN
        mx, mn = _report(f"loop realsr sample step {k}", rec[k]["sample"], torch.from_numpy(g[f"sample/{k}"]))
        assert mx <= LOOP_MAX and mn <= LOOP_MEAN
    assert torch.equal(rec[-1]["sample"], final)


def test_loop_realsr_15_batch2_vs_reference_golden(golden_dir):
    """Two images through the 15-step loop against the reference's own trajectory (noise re-drawn from the seed)."""
    g, diff, m, y, noises, final = _loop(golden_dir, "realsr", 15, "loop_realsr_T15_b2.npz", True)
    mx, mn = _report("loop realsr T15 batch 2 (final latent)", final, torch.from_numpy(g["final"]))
    assert mx <= LOOP_MAX and mn <= LOOP_MEAN


def test_sampler_tables_survive_forward_reload_and_second_schedule():
    """The schedule / FiLM tables live in the plan's workspace and are shared by model.forward (rows 0..B-1) and by
    every sampler of the plan: a sampler must re-derive them after (a) a plain forward on the same plan, (b) a second
    diffusion with another T / kappa on the same plan, (c) new weights (load_state_dict -> repack)."""
    from resshift_b200.models.script_util import create_gaussian_diffusion
    ucfg, dcfg, m = _model("tiny")
    dcfg.sf = 1
    diff = create_gaussian_diffusion(**dcfg.to_kwargs())
    g = torch.Generator(device="cuda").manual_seed(21)
    y = torch.rand(4, 3, 64, 64, device="cuda", generator=g) * 2 - 1
    noises = torch.randn(diff.num_timesteps + 1, 4, 3, 64, 64, device="cuda", generator=g)
    a = diff.sample_latent(y, m, {"lq": y}, noises=noises)
    # (a) forward with unrelated timesteps in between overwrites FiLM rows 0..3
    m(torch.randn(4, 3, 64, 64, device="cuda", generator=g), torch.tensor([3, 3, 1, 0], device="cuda"), lq=y)
    assert torch.equal(diff.sample_latent(y, m, {"lq": y}, noises=noises), a)
    # (b) another schedule on the same plan, then the first again
    d2 = preset("tiny")[1]
    d2.sf, d2.steps, d2.kappa = 1, 6, 1.0
    diff2 = create_gaussian_diffusion(**d2.to_kwargs())
    n2 = torch.randn(diff2.num_timesteps + 1, 4, 3, 64, 64, device="cuda", generator=g)
    b = diff2.sample_latent(y, m, {"lq": y}, noises=n2)
    assert torch.equal(diff.sample_latent(y, m, {"lq": y}, noises=noises), a)
    assert torch.equal(diff2.sample_latent(y, m, {"lq": y}, noises=n2), b)
    # (c) new weights: results must equal those of a fresh model holding the new weights
    sd2 = random_state_dict(ucfg, 9)
    m.load_state_dict(sd2, strict=True)
    c = diff.sample_latent(y, m, {"lq": y}, noises=noises)
    _, _, fresh = _model("tiny", seed=9)
    assert torch.equal(c, diff.sample_latent(y, fresh, {"lq": y}, noises=noises))
    assert not torch.equal(c, a)


def test_native_loop_rejects_mismatched_inputs():
    from resshift_b200.models.script_util import create_gaussian_diffusion
    ucfg, dcfg, m = _model("tiny")
    dcfg.sf = 1
    diff = create_gaussian_diffusion(**dcfg.to_kwargs())
    y = torch.rand(2, 3, 64, 64, device="cuda")
    noises = torch.randn(diff.num_timesteps + 1, 2, 3, 64, 64, device="cuda")
    with pytest.raises(ValueError):
        diff.sample_latent(y, m, {"lq": y[:, :, :32]}, noises=noises)             # wrong LQ size
    with pytest.raises(ValueError):
        diff.sample_latent(y, m, {"lq": y, "mask": y[:, :1]}, noises=noises)      # mask on a model without cond_mask
    with pytest.raises(ValueError):
        diff.sample_latent(y, m, {"lq": y}, noises=noises[:-1])                   # wrong number of noise tensors


def test_loop_faceir_4_steps_vs_oracle():
    """The native 4-step schedule of the face-restoration task (8 latent channels, feature extractor hoisted out of the
    loop) against the CPU oracle loop on the same z_y, noises and 512x512 LQ."""
    from oracle import diffusion_oracle as do
    from oracle import unet_oracle as uo
    from resshift_b200.models.script_util import create_gaussian_diffusion
    ucfg, dcfg, m = _model("faceir", seed=6)
    sd = random_state_dict(ucfg, 6)
    diff = create_gaussian_diffusion(**dcfg.to_kwargs())
    g = torch.Generator().manual_seed(66)
    zy = torch.randn(2, 8, 64, 64, generator=g) * 0.5
    lq = torch.rand(2, 3, 512, 512, generator=g) * 2 - 1
    noises = torch.stack([torch.randn(2, 8, 64, 64, generator=g) for _ in range(dcfg.steps + 1)])
    tabs = do.schedule_tables(do.eta_schedule(dcfg.steps, dcfg.min_noise_level, dcfg.etas_end, dcfg.kappa,
                                              dcfg.schedule_kwargs["power"]), dcfg.kappa)
    ref = do.p_sample_loop(lambda x, t: uo.unet_forward(sd, ucfg, x, t, lq=lq), zy, list(noises), tabs, dcfg.kappa)
    final = diff.sample_latent(zy.cuda(), m, {"lq": lq.cuda()}, noises=noises.cuda(), use_graph=True)
    assert not torch.isnan(final).any()
    mx, mn = _report("loop faceir T4", final, ref)
    assert mx <= LOOP_MAX and mn <= LOOP_MEAN


def test_batch_independence_at_bench_size():
    """BASELINE config 2 size (batch 16, full width).  Tiles of different images share CTAs at the 8x8 level and
    GroupNorm statistics are per image, so image i must not depend on its batch neighbours: bit-exact when only the
    OTHER images change (every reduction has a fixed order, no atomics).  Against a batch-1 run the result agrees to
    rounding noise only, because the planner picks other tile shapes / split-K factors for other batch sizes."""
    ucfg, _, m = _model("realsr")
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(16, 3, 64, 64, device="cuda", generator=g)
    lq = torch.rand(16, 3, 64, 64, device="cuda", generator=g) * 2 - 1
    t = torch.full((16,), 9, device="cuda")
    full = m(x, t, lq=lq).clone()
    assert not torch.isnan(full).any()
    again = m(x, t, lq=lq)
    assert torch.equal(full, again)                                   # run-to-run bit reproducible
    keep = [0, 5, 15]
    x2, lq2 = torch.randn_like(x), torch.rand_like(lq) * 2 - 1
    for i in keep:
        x2[i], lq2[i] = x[i], lq[i]
    other = m(x2, t, lq=lq2)
    for i in keep:
        assert torch.equal(other[i], full[i]), f"image {i} depends on its batch neighbours"
    for i in (5,):
        one = m(x[i:i + 1], t[i:i + 1], lq=lq[i:i + 1])
        d = (one - full[i:i + 1]).abs()
        print(f"[property] batch-16 vs batch-1 run of image {i}: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e}")
        assert d.max().item() <= 1e-2 and d.mean().item() <= 1e-3
    # and the batched result itself is right: image 5 against the CPU oracle
    from oracle import unet_oracle as uo
    sd = random_state_dict(ucfg, 0)
    ref = uo.unet_forward(sd, ucfg, x[5:6].cpu(), t[5:6].cpu(), lq=lq[5:6].cpu())
    mx, mn = _report("forward realsr, image 5 of a batch of 16", full[5:6], ref)
    assert mx <= FWD_MAX and mn <= FWD_MEAN


def test_concurrent_batch_slices_are_bit_identical(monkeypatch):
    """RS_LOWRES_STREAMS=2: the few-tile levels run as two batch slices on side streams (fork / join by events, captured
    into the sampler's graph as parallel branches).  Per-image results do not depend on batch neighbours, but slices
    get other tile configurations than the full batch, so the check is agreement to rounding — plus exact
    reproducibility of the sliced plan itself, eager and graph-replayed, with per-image timesteps (FiLM rows)."""
    from resshift_b200.models.script_util import create_gaussian_diffusion
    outs = {}
    for nb in ("1", "2"):
        monkeypatch.setenv("RS_LOWRES_STREAMS", nb)
        ucfg, dcfg, m = _model("tiny")
        dcfg.sf = 1
        diff = create_gaussian_diffusion(**dcfg.to_kwargs())
        g = torch.Generator(device="cuda").manual_seed(5)
        x = torch.randn(4, 3, 64, 64, device="cuda", generator=g)
        lq = torch.rand(4, 3, 64, 64, device="cuda", generator=g) * 2 - 1
        t = torch.tensor([3, 0, 2, 1], device="cuda")
        noises = torch.randn(diff.num_timesteps + 1, 4, 3, 64, 64, device="cuda", generator=g)
        f1 = m(x, t, lq=lq).clone()
        assert torch.equal(f1, m(x, t, lq=lq))
        a = diff.sample_latent(lq, m, {"lq": lq}, noises=noises, use_graph=True)
        assert torch.equal(a, diff.sample_latent(lq, m, {"lq": lq}, noises=noises, use_graph=False))
        outs[nb] = (f1, a)
        del m
    d = (outs["1"][0] - outs["2"][0]).abs().max().item()
    e = (outs["1"][1] - outs["2"][1]).abs().max().item()
    print(f"[streams] forward |d|max {d:.3e}, loop |d|max {e:.3e}")
    assert d <= 1e-2 and e <= 1e-2


def test_graph_replay_is_deterministic_and_matches_eager():
    from resshift_b200.models.script_util import create_gaussian_diffusion
    ucfg, dcfg, m = _model("tiny")
    dcfg.sf = 1
    diff = create_gaussian_diffusion(**dcfg.to_kwargs())
    g = torch.Generator(device="cuda").manual_seed(11)
    y = torch.rand(4, 3, 64, 64, device="cuda", generator=g) * 2 - 1
    noises = torch.randn(diff.num_timesteps + 1, 4, 3, 64, 64, device="cuda", generator=g)
    a = diff.sample_latent(y, m, {"lq": y}, noises=noises, use_graph=True)
    b = diff.sample_latent(y, m, {"lq": y}, noises=noises, use_graph=True)
    c = diff.sample_latent(y, m, {"lq": y}, noises=noises, use_graph=False)
    assert torch.equal(a, b)          # graph replay is bit-reproducible
    assert torch.equal(a, c)          # and identical to the eagerly enqueued loop


def test_sampler_class_end_to_end_with_identity_autoencoder():
    """ResShiftSampler.sample_func surface (reference sampler.py:119-165) with a stand-in first stage."""
    from resshift_b200.sampler import ResShiftSampler, make_configs
    ucfg, dcfg = preset("tiny")
    dcfg.sf = 1
    configs = make_configs(ucfg, dcfg, autoencoder=None, state_dict=random_state_dict(ucfg, 0))
    s = ResShiftSampler(configs, sf=1, use_amp=True, chop_size=64, chop_stride=64, padding_offset=64, seed=123)
    y0 = torch.rand(2, 3, 60, 50, device="cuda") * 2 - 1        # gets reflect-padded to 64x64
    out = s.sample_func(y0, noise_repeat=False, mask=None)
    assert out.shape == (2, 3, 60, 50) and out.abs().max().item() <= 1.0
