"""KL first stage (AutoencoderKLTorch / EncoderKLTorch) on the native kernels, and VQModelTorch.decode_code.

1. encode (moments, mode, sample with given noise) and decode against the fp32 oracle on the GPU (TF32 off): the tiny
   configuration, the SD-style f8 at 512x512 (T = 4096: GEMM + row softmax), at 1024x1024 (T = 16384: fused attention)
   and at 384x640.  Bounds as for the VQ-GAN: max|d| <= 1e-2, mean|d| <= 2e-3 (for the sampled z, per unit of
   1 + |noise|).
2. encode(x) with the default sample_posterior draws its noise exactly as the reference does: torch.randn on the CPU
   default generator, leaving that generator in the same state.
3. attention_team members of 2 and 3 give results bit-identical to plain encode / decode (T > 8192).
4. decode_code is bit-identical to decode(embedding[idx], force_not_quantize=True).
5. ResShiftSampler with autoencoder target "ldm.models.autoencoder.AutoencoderKLTorch": inference() end to end; shard
   mode (virtual ranks) and device pools of 2 and 3 (virtual, one chunk forming a team) give the PNG bytes / tiles of the
   one-GPU default run, noise_repeat off and on."""
import numpy as np
import pytest
import torch

from oracle import kl_oracle as ko
from tests.gpu_util import fp32_matmuls

pytestmark = pytest.mark.gpu

MAX_ABS, MEAN_ABS = 1e-2, 2e-3


@pytest.fixture(scope="module")
def fp32_reference():
    with fp32_matmuls():
        yield


_MODELS = {}


def _kl(name):
    from resshift_b200.models.autoencoder import AutoencoderKLTorch
    from resshift_b200.vq_arch import kl_preset, random_kl_state_dict
    if name not in _MODELS:
        cfg = kl_preset(name)
        sd = random_kl_state_dict(cfg, 0)
        m = AutoencoderKLTorch(**cfg.to_kwargs())
        m.load_state_dict(sd, strict=True)
        _MODELS[name] = (cfg, {k: v.cuda() for k, v in sd.items()}, m.cuda().eval())
    return _MODELS[name]


def _close(got, ref, what, scale=None):
    d = (got.float() - ref.float()).abs()
    if scale is not None:
        d = d / scale
    assert not torch.isnan(got).any(), what
    assert d.max().item() <= MAX_ABS and d.mean().item() <= MEAN_ABS, \
        f"{what}: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e} (ref std {ref.float().std().item():.3f})"


# (name, batch, H, W, fused attention)
SIZES = [("tiny", 2, 64, 96, False), ("f8", 1, 512, 512, False), ("f8", 1, 1024, 1024, True), ("f8", 1, 384, 640, False)]


@pytest.mark.parametrize("name,b,h,w,fused", SIZES)
def test_encode_decode_against_fp32_oracle(fp32_reference, name, b, h, w, fused):
    cfg, sd, m = _kl(name)
    f = cfg.downscale
    g = torch.Generator().manual_seed(5)
    x = (torch.rand(b, 3, h, w, generator=g) * 2 - 1).cuda()
    noise = torch.randn(b, cfg.embed_dim, h // f, w // f, generator=g)
    assert (m.plan(0, b, h, w).attention is not None) == fused and (m.plan(1, b, h, w).attention is not None) == fused
    z_ref, mom_ref = ko.kl_encode(x, sd, cfg, return_moments=True)
    z, mom = m.encode(x, sample_posterior=False, return_moments=True)
    _close(mom, mom_ref, "moments")
    _close(z, z_ref, "mode")
    zs, mom2 = m.encode(x, return_moments=True, posterior_noise=noise)
    # z = mean + std * noise: its error is err(mean) + |noise| err(std), so the bound applies per unit of (1 + |noise|)
    _close(zs, ko.kl_encode(x, sd, cfg, noise=noise), "sample", scale=1 + noise.abs().cuda())
    assert torch.equal(mom2, mom)
    _close(m.decode(z_ref), ko.kl_decode(z_ref, sd, cfg), "decode")
    del z_ref, mom_ref
    torch.cuda.empty_cache()


def test_default_encode_draws_noise_like_the_reference():
    cfg, sd, m = _kl("tiny")
    x = (torch.rand(2, 3, 64, 96, generator=torch.Generator().manual_seed(3)) * 2 - 1).cuda()
    torch.manual_seed(77)
    z = m.encode(x)
    after = torch.get_rng_state()
    torch.manual_seed(77)
    noise = torch.randn(z.shape)                 # DiagonalGaussianDistribution.sample: torch.randn(mean.shape), CPU
    assert torch.equal(torch.get_rng_state(), after)
    assert torch.equal(m.encode(x, posterior_noise=noise), z)
    assert torch.equal(m.forward(x, sample_posterior=False), m.decode(m.encode(x, sample_posterior=False)))
    state = torch.get_rng_state()
    m.encode(x, sample_posterior=False)          # mode() draws nothing
    assert torch.equal(torch.get_rng_state(), state)
    with pytest.raises(ValueError, match="posterior_noise"):
        m.encode(x, posterior_noise=noise[:1])


def test_encoder_only_class_equals_full_class():
    from resshift_b200.models.autoencoder import EncoderKLTorch
    cfg, sd, m = _kl("tiny")
    enc = EncoderKLTorch(**cfg.to_kwargs())
    enc.load_state_dict({k: v for k, v in sd.items() if k.startswith(("encoder.", "quant_conv."))}, strict=True)
    enc = enc.cuda().eval()
    x = (torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(4)) * 2 - 1).cuda()
    noise = torch.randn(1, cfg.embed_dim, 16, 16)
    a, am = enc.encode(x, return_moments=True, posterior_noise=noise)
    b, bm = m.encode(x, return_moments=True, posterior_noise=noise)
    assert torch.equal(a, b) and torch.equal(am, bm)


@pytest.mark.parametrize("size", [2, 3])
def test_attention_team_members_equal_plain_calls(size):
    """Virtual members in one process: each member computes its rows, the exchange fills in the others' rows from a
    full-row run; every member's result must equal the plain call bit for bit."""
    cfg, sd, m = _kl("tiny")
    x = (torch.rand(1, 3, 512, 512, generator=torch.Generator().manual_seed(6)) * 2 - 1).cuda()
    noise = torch.randn(1, cfg.embed_dim, 128, 128)
    assert m.plan(0, 1, 512, 512).attention.shape == (1, 16384, 128)
    z, mom = m.encode(x, return_moments=True, posterior_noise=noise)
    dec = m.decode(z)

    full = {}
    def capture(key):
        def ex(view, rb, re):
            assert (rb, re) == (0, view.shape[1])
            full[key] = view.clone()
        return ex
    with m.attention_team(0, 1, capture("enc")):
        assert torch.equal(m.encode(x, return_moments=True, posterior_noise=noise)[0], z)
    with m.attention_team(0, 1, capture("dec")):
        assert torch.equal(m.decode(z), dec)

    for member in range(size):
        def fill(key):
            def ex(view, rb, re):
                view[:, :rb] = full[key][:, :rb]
                view[:, re:] = full[key][:, re:]
            return ex
        with m.attention_team(member, size, fill("enc")):
            zm, mm = m.encode(x, return_moments=True, posterior_noise=noise)
        with m.attention_team(member, size, fill("dec")):
            dm = m.decode(z)
            assert [r[0] for r in m.attention_rows] == [1]
        assert torch.equal(zm, z) and torch.equal(mm, mom) and torch.equal(dm, dec), (size, member)


def test_vq_decode_code_equals_decode_of_codebook_rows():
    from resshift_b200.models.autoencoder import VQModelTorch
    from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
    cfg = vq_preset("tiny")
    m = VQModelTorch(**cfg.to_kwargs())
    m.load_state_dict(random_vq_state_dict(cfg, 0), strict=True)
    m = m.cuda().eval()
    g = torch.Generator().manual_seed(9)
    for b, lh, lw in [(2, 16, 16), (1, 16, 24), (1, 128, 128)]:                  # the last one: fused attention
        idx = torch.randint(0, cfg.n_embed, (b, lh, lw), generator=g).cuda()
        emb = m.quantize.embedding.weight
        ref = m.decode(emb[idx].permute(0, 3, 1, 2).contiguous(), force_not_quantize=True)
        assert torch.equal(m.decode_code(idx), ref)
        assert torch.equal(m.decode_code(idx.to(torch.int32)), ref)
    bad = idx.clone()
    bad[0, 64, 64] = cfg.n_embed
    assert torch.isnan(m.decode_code(bad)).any()                    # refused in place: NaN, no out-of-bounds read


# ------------------------------------------------------------------------------------------------ the whole pipeline

CHOP = dict(tiny=dict(chop_size=64, chop_stride=48, padding_offset=64),           # 200x148 -> 4 x 3 = 12 tiles
            team=dict(chop_size=512, chop_stride=448, padding_offset=16))         # 128x128 x4: one unit, T = 16384


def _sampler(kind, devices=None, **kw):
    from resshift_b200.config import preset
    from resshift_b200.sampler import ResShiftSampler, make_configs
    from resshift_b200.vq_arch import VQConfig, random_kl_state_dict
    from resshift_b200.weights import random_state_dict
    ucfg, dcfg = preset("tiny")
    dcfg.sf = 4
    # embed_dim = the denoiser's in / out channels (3); the tiny VQ topology, f = 4
    kcfg = VQConfig(embed_dim=ucfg.in_channels, z_channels=4, resolution=64, ch=32, ch_mult=(1, 2, 4),
                    num_res_blocks=(1, 2, 2), double_z=True, kl=True)
    ae = {"target": "ldm.models.autoencoder.AutoencoderKLTorch", "params": kcfg.to_kwargs(),
          "ckpt_path": random_kl_state_dict(kcfg, 0)}
    configs = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    return ResShiftSampler(configs, sf=4, use_amp=True, seed=123, devices=devices, **{**CHOP[kind], **kw})


@pytest.fixture(scope="module")
def samplers():
    return {kind: {0: _sampler(kind), 2: _sampler(kind, "0,0"), 3: _sampler(kind, [0, 0, 0])} for kind in CHOP}


IMAGES = dict(tiny={"a1": (200, 148), "a2": (200, 148), "b": (60, 50)}, team={"t": (128, 128)})


def _write(d, kind):
    import cv2
    rng = np.random.default_rng(7)
    (d / "in").mkdir()
    for name, (h, w) in IMAGES[kind].items():
        cv2.imwrite(str(d / "in" / f"{name}.png"), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))


def _infer(s, d, kind, out, noise_repeat=False):
    s.setup_seed()
    s.inference(d / "in", d / out, bs=len(IMAGES[kind]), noise_repeat=noise_repeat)
    return {p.name: p.read_bytes() for p in sorted((d / out).iterdir())}


def test_reference_target_builds_the_native_kl_class(samplers):
    from resshift_b200.models.autoencoder import AutoencoderKLTorch
    s = samplers["tiny"][0]
    assert type(s.autoencoder) is AutoencoderKLTorch


@pytest.mark.parametrize("pool", [2, 3])
@pytest.mark.parametrize("kind,chop_bs,noise_repeat", [("tiny", 1, False), ("tiny", 5, True), ("team", 1, False),
                                                        ("team", 1, True)])
def test_device_pool_equals_one_gpu(samplers, tmp_path, kind, pool, chop_bs, noise_repeat):
    ref_s, s = samplers[kind][0], samplers[kind][pool]
    ref_s.chop_bs = s.chop_bs = chop_bs
    _write(tmp_path, kind)
    ref = _infer(ref_s, tmp_path, kind, "ref", noise_repeat)
    assert sorted(ref) == sorted(f"{n}.png" for n in IMAGES[kind])
    rows = []
    if kind == "team":
        orig = s.pool.run

        def run(*a):
            out = orig(*a)
            rows.extend(r.autoencoder.attention_rows for r in s.pool.replicas)
            return out
        s.pool.run = run
    try:
        out = _infer(s, tmp_path, kind, "out", noise_repeat)
    finally:
        s.pool.__dict__.pop("run", None)
    assert out == ref
    if kind == "team":                      # one unit on a team of every replica: the attention rows were split
        assert all(len(r) == 2 for r in rows) and len({r[0][1:] for r in rows}) == pool, rows


@pytest.mark.parametrize("chop_bs,noise_repeat", [(1, False), (1, True), (5, False), (5, True)])
def test_virtual_ranks_equal_one_gpu_default(samplers, chop_bs, noise_repeat):
    from resshift_b200.parallel import unit_schedule
    from resshift_b200.sampler import tile_counts
    s = samplers["tiny"][0]
    s.chop_bs = chop_bs
    g = torch.Generator(device="cuda").manual_seed(8)
    lqs = [torch.rand(b, 3, h, w, device="cuda", generator=g) * 2 - 1 for b, h, w in [(2, 200, 148), (1, 60, 50)]]
    masks = [None, None]
    s.setup_seed()
    ref = [s._sample_tiled(lq, mask=None, noise_repeat=noise_repeat) for lq in lqs]
    units = s._plan_units([tuple(lq.shape[2:]) for lq in lqs])
    for world in (2, 5):
        schedule = unit_schedule(len(units), world, teams=False)
        shares = []
        for rank in range(world):
            s.setup_seed()
            shares.append(s._run_rank(lqs, masks, noise_repeat, units, schedule, rank))
        counts = tile_counts(units, schedule, world)
        for gi, (lq, r) in enumerate(zip(lqs, ref)):
            assert [sh[gi].shape[0] for sh in shares] == counts[gi]
            out = s._assemble(torch.cat([sh[gi] for sh in shares]), *lq.shape[2:])
            assert torch.equal(out, r), (world, gi, (out - r).abs().max().item())


def test_posterior_sampling_autoencoder_without_noise_input_is_refused(samplers):
    """An autoencoder whose encode samples a posterior it cannot take from the caller (the reference's own class, for
    one) would draw that noise only for the units a rank runs: shard mode and pools refuse it."""
    s = samplers["tiny"][0]

    class Foreign(torch.nn.Module):
        def encode(self, x, sample_posterior=True, return_moments=False):
            raise AssertionError("not reached")

    orig = s.autoencoder
    s.autoencoder = Foreign()
    try:
        with pytest.raises(RuntimeError, match="samples its posterior"):
            s._check_shardable()
    finally:
        s.autoencoder = orig
