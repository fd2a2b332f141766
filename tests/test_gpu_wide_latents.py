"""First stages with 16- to 64-channel latents on the wide kernels of csrc/vq_kernels.cuh, and the sampling loop on them.

u = 2^-24 (one fp32 rounding to nearest).

1. pointwise_conv_wide_kernel (rs_op_pointwise_conv, VQ quant_conv) and kl_posterior_wide_kernel (rs_op_kl_posterior,
   KL quant_conv + DiagonalGaussianDistribution) against float64 on the same fp16 weights, with the bounds
   test_gpu_sampler_kernels.py holds the narrow kernels to: a chain of Cin fmaf from the bias, Cin u (|b| + sum |w x|);
   z = mean + fp32(expf(0.5 clamp(logvar)) noise) against float64 of the kernel's own moments, 5u |std noise| + u |z|;
   mode() bit-equal to the mean.  Logvars planted past both clamp limits and at their neighbours; HW not a multiple of
   the 32-position CTA tile; two images.
2. vq_quantize_wide_kernel (E = 16, 32, 64) through VQModelTorch.decode, with codebooks built so that the answer is
   known: every code planted once (indices exact), exact ties across the kernel's shared-memory chunk boundary and
   inside a chunk (the first minimum wins), random latents against the float64 argmin wherever its margin exceeds the
   fp32 evaluation's error.  `quantize` (post_quant_conv of the codes, the decoder's input) within 1/2 ulp16 + E u (|b| +
   sum |w| |e|) of float64, its pad channels +0 exactly; decode_code bit-identical to decoding the gathered rows, NaN at
   exactly the out-of-range indices.
3. Whole passes: the tiny 16- / 64-channel presets against the reference's outputs (tests/golden/wide_latents.npz) and
   LDM's kl-f16 / kl-f32 (level attention) at 512x512 and 1024x1024 against the fp32 options oracle on the GPU (TF32
   off; every attention of these takes the GEMM form, as no level has more than 8192 positions); max|d| <= 1e-2,
   mean|d| <= 2e-3 as test_gpu_kl.py (the sampled z per unit of 1 + |noise|).
4. ResShiftSampler.inference with a 16-channel KL first stage and a UNetModelSwin with 16 latent channels on a tiled
   image: bit-reproducible, and device pools "0,0" / [0,0,0] and shard mode (virtual ranks) give the one-GPU PNG bytes /
   tiles, noise_repeat off and on.
"""
import numpy as np
import pytest
import torch

from oracle import kl_oracle as ko
from oracle import vq_oracle as vo
from oracle import vq_options_oracle as voo
from resshift_b200.vq_arch import VQConfig, kl_preset, random_kl_state_dict, random_vq_state_dict, wide_vq_preset
from tests.gpu_util import fp32_matmuls

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from resshift_b200 import _lib
    from tests import gpu_util as G

U = 2.0 ** -24
MAX_ABS, MEAN_ABS = 1e-2, 2e-3


@pytest.fixture(scope="module")
def fp32_reference():
    with fp32_matmuls():
        yield


def _check(tag, got, ref, bound):
    """|got - ref| <= bound per element (float64).  NaN fails."""
    err = (got.double() - ref).abs()
    ratio = (err / bound.clamp(min=1e-300)).max().item()
    print(f"[bound] {tag}: max |d| / bound = {ratio:.3e}")
    bad = ~(err <= bound)
    assert not bad.any(), f"{tag}: {int(bad.sum())} of {bad.numel()} elements outside the bound (ratio {ratio:.3e})"


def _close(got, ref, what, scale=None):
    d = (got.float() - ref.float().to(got.device)).abs()
    if scale is not None:
        d = d / scale
    print(f"[wide] {what}: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e}")
    assert not torch.isnan(got).any(), what
    assert d.max().item() <= MAX_ABS and d.mean().item() <= MEAN_ABS, \
        f"{what}: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e} (ref std {ref.float().std().item():.3f})"


# ------------------------------------------------------------------------------------------------ 1. quant_conv kernels

def _fp16_weights(O, I, ld, g, scale=0.5):
    w = torch.randn(O, I, device="cuda", generator=g) * scale
    buf = torch.zeros(O, ld, dtype=torch.float16, device="cuda")
    buf[:, :I] = w.half()
    return buf, buf[:, :I].double()


@pytest.mark.parametrize("Cout", [16, 64])
@pytest.mark.parametrize("Cin", [16, 32, 64])
def test_pointwise_wide_vs_float64(Cin, Cout):
    N, HW, ld = 2, 999, Cin + 8                      # HW = 31 tiles of 32 + 7
    g = torch.Generator(device="cuda").manual_seed(Cin * 100 + Cout)
    x = torch.randn(N, Cin, HW, device="cuda", generator=g) * 3
    wbuf, w = _fp16_weights(Cout, Cin, ld, g, 0.3)
    b = torch.randn(Cout, device="cuda", generator=g)
    y = torch.full((N, Cout, HW), float("nan"), device="cuda")
    _lib.check(_lib.lib.rs_op_pointwise_conv(x.data_ptr(), wbuf.data_ptr(), ld, b.data_ptr(), Cin, Cout, N, HW, y.data_ptr(),
                                             G.stream()))
    torch.cuda.synchronize()
    ref = torch.einsum("oc,nch->noh", w, x.double()) + b.double()[None, :, None]
    mag = torch.einsum("oc,nch->noh", w.abs(), x.double().abs()) + b.double().abs()[None, :, None]
    _check(f"wide pointwise Cin={Cin} Cout={Cout} HW={HW}", y, ref, Cin * U * mag)


LOGVARS = [-40.0, -30.0, 20.0, 25.0, float(np.nextafter(np.float32(-30), np.float32(0))),
           float(np.nextafter(np.float32(-30), np.float32(-100))), float(np.nextafter(np.float32(20), np.float32(0))),
           float(np.nextafter(np.float32(20), np.float32(100)))]


def _posterior_ref(m64, noise, E):
    mean, lv = m64[:, :E], m64[:, E:].clamp(-30.0, 20.0)
    sn = torch.exp(0.5 * lv) * noise.double()
    return mean + sn, 5 * U * sn.abs() + U * (mean + sn).abs()


# (Cin = 2 z_channels, E): both wide, the widest, a narrow encoder with a wide latent and the reverse
@pytest.mark.parametrize("Cin,E,HW", [(32, 16, 333), (128, 64, 333), (64, 32, 1024), (8, 16, 100), (32, 4, 77)])
def test_kl_posterior_wide_vs_float64(Cin, E, HW):
    N, ld = 2, (Cin + 7) // 8 * 8
    g = torch.Generator(device="cuda").manual_seed(Cin * 1000 + E * 10 + HW)
    h = torch.randn(N, Cin, HW, device="cuda", generator=g) * 2
    wbuf, _ = _fp16_weights(2 * E, Cin, ld, g, 0.3)
    b = torch.randn(2 * E, device="cuda", generator=g)
    # planted logvars: the rows of these channels have zero weights, so the moment is the bias exactly
    planted = [LOGVARS[c % len(LOGVARS)] for c in range(E)]
    for c in range(E):
        b[E + c] = planted[c]
        wbuf[E + c].zero_()
    w = wbuf[:, :Cin].double()
    noise = torch.randn(N, E, HW, device="cuda", generator=g)
    z = torch.full((N, E, HW), float("nan"), device="cuda")
    mom = torch.full((N, 2 * E, HW), float("nan"), device="cuda")
    _lib.check(_lib.lib.rs_op_kl_posterior(h.data_ptr(), wbuf.data_ptr(), ld, b.data_ptr(), Cin, E, noise.data_ptr(),
                                           z.data_ptr(), mom.data_ptr(), N, HW, G.stream()))
    torch.cuda.synchronize()
    ref = torch.einsum("oc,nch->noh", w, h.double()) + b.double()[None, :, None]
    mag = torch.einsum("oc,nch->noh", w.abs(), h.double().abs()) + b.double().abs()[None, :, None]
    _check(f"wide kl moments Cin={Cin} E={E} HW={HW}", mom, ref, Cin * U * mag)
    assert torch.equal(mom[:, E:], b[E:][None, :, None].expand(N, E, HW)), "planted logvars"
    zr, bound = _posterior_ref(mom.double(), noise, E)
    _check(f"wide kl z Cin={Cin} E={E} HW={HW}", z, zr, bound)
    z0 = torch.full_like(z, float("nan"))
    _lib.check(_lib.lib.rs_op_kl_posterior(h.data_ptr(), wbuf.data_ptr(), ld, b.data_ptr(), Cin, E, None, z0.data_ptr(),
                                           None, N, HW, G.stream()))
    torch.cuda.synchronize()
    assert torch.equal(G.bits(z0), G.bits(mom[:, :E].contiguous())), "mode() is the mean"


def test_wide_refusals():
    x = torch.zeros(1, 200, 4, device="cuda")
    w = torch.zeros(256, 256, dtype=torch.float16, device="cuda")
    L = _lib.lib

    def refused(rc, what):
        assert rc != 0, f"accepted: {what}"
        assert what in L.rs_last_error().decode(), L.rs_last_error()
    for cin in (12, 72):
        refused(L.rs_op_pointwise_conv(x.data_ptr(), w.data_ptr(), 256, x.data_ptr(), cin, 3, 1, 4, x.data_ptr(), G.stream()),
                "Cin must be at most 8")
    refused(L.rs_op_pointwise_conv(x.data_ptr(), w.data_ptr(), 256, x.data_ptr(), 16, 72, 1, 4, x.data_ptr(), G.stream()),
            "Cout at most 64")
    refused(L.rs_op_pointwise_conv(x.data_ptr(), w.data_ptr(), 20, x.data_ptr(), 16, 8, 1, 4, x.data_ptr(), G.stream()),
            "w_ld a multiple of 8")
    refused(L.rs_op_kl_posterior(x.data_ptr(), w.data_ptr(), 256, x.data_ptr(), 136, 4, None, x.data_ptr(), None, 1, 4,
                                 G.stream()), "Cin must be at most 16")
    for e in (12, 72):
        refused(L.rs_op_kl_posterior(x.data_ptr(), w.data_ptr(), 256, x.data_ptr(), 32, e, None, x.data_ptr(), None, 1, 4,
                                     G.stream()), "2E must be at most 16")


# ------------------------------------------------------------------------------------------------ 2. quantiser

def _chunk(E):
    """Codes per shared-memory chunk of vq_quantize_wide_kernel<E> (kQuantWideChunk)."""
    return (32 * 1024 // (4 * (E + 5))) // 32 * 32


def _vq_cfg(E, z=None, n_embed=1024):
    return VQConfig(embed_dim=E, n_embed=n_embed, z_channels=E if z is None else z, resolution=64, ch=32, ch_mult=(1, 2, 4),
                    num_res_blocks=(1, 2, 2))


def _vq_model(cfg, sd):
    from resshift_b200.models.autoencoder import VQModelTorch
    m = VQModelTorch(**cfg.to_kwargs())
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def _separated_codebook(n, E, seed):
    """n codes in E >= 16 dimensions with the spread of random_vq_state_dict's codebook: random codes in 16 or more
    dimensions are far apart (checked below)."""
    g = torch.Generator().manual_seed(seed)
    return (0.6 * torch.randn(n, E, generator=g)).cuda()


def _state_dict(cfg, codebook, seed=0):
    sd = {n: t.cuda() for n, t in random_vq_state_dict(cfg, seed).items()}
    sd["quantize.embedding.weight"] = codebook
    sd["post_quant_conv.bias"] = 0.5 * torch.randn(sd["post_quant_conv.bias"].shape, device="cuda",
                                                   generator=torch.Generator(device="cuda").manual_seed(3))
    return sd


def _plant(codebook, codes, shape):
    N, H, W = shape
    return codebook[codes].reshape(N, H, W, -1).permute(0, 3, 1, 2).contiguous()


def _post_quant_ref(e, sd):
    """float64 post_quant_conv of per-pixel vectors e [N, h, w, E] -> (NCHW output, its accumulation magnitude)."""
    w = sd["post_quant_conv.weight"]
    cz, E = w.shape[0], w.shape[1]
    w = w.reshape(cz, E).half().double()
    b = sd["post_quant_conv.bias"].double()
    return (e @ w.t() + b).permute(0, 3, 1, 2), (e.abs() @ w.abs().t() + b.abs()).permute(0, 3, 1, 2)


def _check_quantize_output(tag, m, cfg, sd, shape, rows):
    """`quantize` = float64 post_quant_conv(rows) within 1/2 ulp16 + E u (|b| + sum |w| |e|); pad channels +0."""
    B, H, W = shape
    f = cfg.downscale
    ref, mag = _post_quant_ref(rows, sd)
    G.assert_within(f"{tag} quantize", m.probe(1, B, H * f, W * f, "quantize"), ref, cfg.embed_dim * U * mag, 1.0)
    padded = m.probe(1, B, H * f, W * f, "quantize.padded")
    assert padded.shape[1] == (cfg.z_channels + 7) // 8 * 8
    assert torch.equal(G.bits(padded[:, cfg.z_channels:]), torch.zeros_like(G.bits(padded[:, cfg.z_channels:]))), \
        "pad channels are +0"


@pytest.mark.parametrize("E", [16, 32, 64])
def test_planted_codes_every_code(fp32_reference, E):
    """Every code of a 1024-code codebook once, in random order, on 2 x 16 x 32 latents; two codes duplicated across the
    chunk boundary and inside a chunk: latents on either copy take the lower index."""
    cfg = _vq_cfg(E)
    cb = _separated_codebook(cfg.n_embed, E, seed=E)
    k = _chunk(E)
    first = {k: k - 1, 700: 5, k // 2 + 1: k // 2}
    for dup, orig in first.items():
        cb[dup] = cb[orig]
    d = torch.cdist(cb.double(), cb.double()).pow(2)
    d.fill_diagonal_(float("inf"))
    for dup, orig in first.items():
        d[dup, orig] = d[orig, dup] = float("inf")
    print(f"[wide quantizer] E={E}: chunk {k} codes, min squared distance between distinct codes {d.min().item():.2e}")
    assert d.min().item() >= 1e-2
    sd = _state_dict(cfg, cb)
    m = _vq_model(cfg, sd)
    codes = torch.randperm(cfg.n_embed, generator=torch.Generator().manual_seed(6)).cuda()
    expected = torch.tensor([first.get(int(c), int(c)) for c in codes.cpu()]).cuda()
    shape = (2, 16, 32)
    z = _plant(cb, codes, shape)
    got = m.decode(z)
    idx = m.last_indices.reshape(-1).long()
    wrong = (idx != expected).nonzero().flatten()
    assert wrong.numel() == 0, f"{wrong.numel()} wrong indices, first at {wrong[:8].tolist()}: got {idx[wrong[:8]].tolist()}"
    ref, ref_idx = vo.vq_decode(z, sd, cfg, return_indices=True)
    assert torch.equal(ref_idx.reshape(-1), expected), "the oracle disagrees with the planted codes"
    _close(got, ref, f"E={E} planted decode")
    _check_quantize_output(f"E={E} planted", m, cfg, sd, shape, cb.double()[idx].reshape(*shape, E))


@pytest.mark.parametrize("E", [16, 32, 64])
def test_random_latents_vs_float64_argmin(E):
    """Random z against random_vq_state_dict's codebook: where the float64 margin between the best and second-best code
    exceeds 1e-5 (|z|^2 + max |e|^2) the index is the float64 argmin, and everywhere it is a code within that bound."""
    cfg = _vq_cfg(E, n_embed=4096)
    sd = {n: t.cuda() for n, t in random_vq_state_dict(cfg, 0).items()}
    m = _vq_model(cfg, sd)
    z = torch.randn(2, E, 24, 40, device="cuda", generator=torch.Generator(device="cuda").manual_seed(10)) * 0.6
    m.decode(z)
    idx = m.last_indices.reshape(-1).long()
    zf = z.permute(0, 2, 3, 1).reshape(-1, E).double()
    e = sd["quantize.embedding.weight"].double()
    zz, ee = (zf * zf).sum(1), (e * e).sum(1)
    d = zz[:, None] + ee[None, :] - 2 * zf @ e.t()
    top = d.topk(2, dim=1, largest=False)
    dmin, best, second = top.values[:, 0], top.indices[:, 0], top.indices[:, 1]
    bound = 1e-5 * (zz + torch.maximum(ee[best], ee[second]))
    clear = (top.values[:, 1] - dmin) > bound
    print(f"[wide quantizer] E={E} random z: {int((~clear).sum())} of {idx.numel()} positions below the margin; "
          f"{int((idx != best).sum())} differ from the float64 argmin")
    assert torch.equal(idx[clear], best[clear])
    assert (d.gather(1, idx[:, None]).squeeze(1) - dmin <= bound).all()
    _check_quantize_output(f"E={E} random", m, cfg, sd, (2, 24, 40), e[idx].reshape(2, 24, 40, E))
    m.decode(z, force_not_quantize=True)
    assert (m.last_indices == -1).all()
    _check_quantize_output(f"E={E} force_not_quantize", m, cfg, sd, (2, 24, 40), z.double().permute(0, 2, 3, 1))


@pytest.mark.parametrize("E,z", [(16, 16), (64, 64), (16, 4)])
def test_decode_code(E, z):
    """decode_code is bit-identical to decode(codebook[idx], force_not_quantize=True); an index outside [0, n_e) gives NaN
    at exactly its position in `quantize` (z = 4 < E: the wide quantiser writing a 4-channel row padded to 8)."""
    cfg = _vq_cfg(E, z=z, n_embed=512)
    sd = _state_dict(cfg, _separated_codebook(cfg.n_embed, E, seed=11))
    m = _vq_model(cfg, sd)
    g = torch.Generator().manual_seed(9)
    B, H, W = 2, 16, 24
    idx = torch.randint(0, cfg.n_embed, (B, H, W), generator=g).cuda()
    emb = m.quantize.embedding.weight
    ref = m.decode(emb[idx].permute(0, 3, 1, 2).contiguous(), force_not_quantize=True)
    assert torch.equal(G.bits(m.decode_code(idx)), G.bits(ref))
    _check_quantize_output(f"E={E} z={z} decode_code", m, cfg, sd, (B, H, W), emb.detach().double()[idx])
    bad = idx.clone()
    hits = [(0, 3, 5, cfg.n_embed), (B - 1, H - 2, 1, -1)]
    for n_, y_, x_, v_ in hits:
        bad[n_, y_, x_] = v_
    m.decode_code(bad)
    f = cfg.downscale
    nan = torch.isnan(m.probe(1, B, H * f, W * f, "quantize"))
    want = torch.zeros_like(nan)
    for n_, y_, x_, _ in hits:
        want[n_, :, y_, x_] = True
    assert torch.equal(nan, want), "NaN outside exactly the out-of-range positions"
    padded = m.probe(1, B, H * f, W * f, "quantize.padded")
    assert (G.bits(padded[:, z:]) == 0).all(), "pad channels are +0 even where the code is out of range"


# ------------------------------------------------------------------------------------------------ 3. whole passes

def _kl_model(cfg, sd):
    from resshift_b200.models.autoencoder import AutoencoderKLTorch
    m = AutoencoderKLTorch(**cfg.to_kwargs())
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


@pytest.mark.parametrize("name", ["tiny16", "tiny64"])
def test_tiny_kl_against_reference(golden_dir, name):
    g = np.load(golden_dir / "wide_latents.npz")
    cfg = kl_preset(name)
    m = _kl_model(cfg, random_kl_state_dict(cfg, 0))
    x = torch.from_numpy(g[f"kl_{name}_x"]).cuda()
    z, mom = m.encode(x, sample_posterior=False, return_moments=True)
    _close(mom, torch.from_numpy(g[f"kl_{name}_moments"]), f"kl {name} moments")
    _close(z, torch.from_numpy(g[f"kl_{name}_mode"]), f"kl {name} mode")
    noise = torch.randn(z.shape, generator=torch.Generator().manual_seed(int(g["sample_seed"])))
    zs = m.encode(x, posterior_noise=noise)
    _close(zs, torch.from_numpy(g[f"kl_{name}_sample"]), f"kl {name} sample", scale=1 + noise.abs().cuda())
    _close(m.decode(torch.from_numpy(g[f"kl_{name}_mode"]).cuda()), torch.from_numpy(g[f"kl_{name}_dec"]), f"kl {name} decode")


@pytest.mark.parametrize("name", ["tiny16", "tiny64"])
def test_tiny_vq_against_reference(golden_dir, name):
    g = np.load(golden_dir / "wide_latents.npz")
    cfg = wide_vq_preset(name)
    sd = random_vq_state_dict(cfg, 0)
    m = _vq_model(cfg, {k: v.cuda() for k, v in sd.items()})
    _close(m.encode(torch.from_numpy(g[f"vq_{name}_x"]).cuda()), torch.from_numpy(g[f"vq_{name}_enc"]), f"vq {name} encode")
    z = torch.from_numpy(g[f"vq_{name}_z"]).cuda()
    dec = m.decode(z)
    # the indices are the reference's wherever the float64 margin to the second-best code exceeds the fp32 evaluation's
    # error (1e-5 (|z|^2 + max |e|^2)); this data has no position below it
    zf = z.permute(0, 2, 3, 1).reshape(-1, cfg.embed_dim).double()
    e = sd["quantize.embedding.weight"].double().cuda()
    zz, ee = (zf * zf).sum(1), (e * e).sum(1)
    top = (zz[:, None] + ee[None, :] - 2 * zf @ e.t()).topk(2, dim=1, largest=False)
    assert ((top.values[:, 1] - top.values[:, 0]) > 1e-5 * (zz + ee.max())).all()
    assert torch.equal(m.last_indices.cpu(), torch.from_numpy(g[f"vq_{name}_idx"])), "code indices"
    _close(dec, torch.from_numpy(g[f"vq_{name}_dec"]), f"vq {name} decode")
    _close(m.decode(z, force_not_quantize=True), torch.from_numpy(g[f"vq_{name}_dec_nq"]), f"vq {name} decode unquantised")


_LDM = {}


@pytest.mark.parametrize("name,size", [("f16", 512), ("f16", 1024), ("f32", 512), ("f32", 1024)])
def test_ldm_kl_against_fp32_oracle(fp32_reference, name, size):
    if name not in _LDM:
        _LDM.clear()
        cfg = kl_preset(name)
        sd = random_kl_state_dict(cfg, 0)
        _LDM[name] = (cfg, {k: v.cuda() for k, v in sd.items()}, _kl_model(cfg, sd))
    cfg, sd, m = _LDM[name]
    f = cfg.downscale
    g = torch.Generator().manual_seed(5)
    x = (torch.rand(1, 3, size, size, generator=g) * 2 - 1).cuda()
    noise = torch.randn(1, cfg.embed_dim, size // f, size // f, generator=g)
    print(f"[wide] kl-{name} {size}x{size}: fused attentions encode {len(m.plan(0, 1, size, size).attentions)}, "
          f"decode {len(m.plan(1, 1, size, size).attentions)}")
    # level attention (kl-f16 at 16, kl-f32 at 16 and 8): the options oracle
    mom_ref = voo.kl_moments(x, sd, cfg)
    mean, std = ko.posterior(mom_ref)
    z_ref = mean.contiguous()
    z, mom = m.encode(x, sample_posterior=False, return_moments=True)
    _close(mom, mom_ref, f"kl-{name} {size} moments")
    _close(z, z_ref, f"kl-{name} {size} mode")
    zs = m.encode(x, posterior_noise=noise)
    _close(zs, mean + std * noise.cuda(), f"kl-{name} {size} sample", scale=1 + noise.abs().cuda())
    _close(m.decode(z_ref), voo.kl_decode(z_ref, sd, cfg), f"kl-{name} {size} decode")
    del z_ref, mom_ref
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ 4. the sampler

CHOP = dict(chop_size=64, chop_stride=48, padding_offset=64)          # 200x148 -> 4 x 3 = 12 tiles
IMAGES = {"a1": (200, 148), "a2": (200, 148), "b": (60, 50)}


def _sampler(devices=None):
    from resshift_b200.config import preset
    from resshift_b200.sampler import ResShiftSampler, make_configs
    from resshift_b200.weights import random_state_dict
    ucfg, dcfg = preset("tiny")
    ucfg.in_channels = ucfg.out_channels = 16
    dcfg.sf = 4
    kcfg = VQConfig(embed_dim=16, z_channels=16, resolution=64, ch=32, ch_mult=(1, 2, 4), num_res_blocks=(1, 2, 2),
                    double_z=True, kl=True)
    ae = {"target": "ldm.models.autoencoder.AutoencoderKLTorch", "params": kcfg.to_kwargs(),
          "ckpt_path": random_kl_state_dict(kcfg, 0)}
    configs = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    return ResShiftSampler(configs, sf=4, use_amp=True, seed=123, devices=devices, **CHOP)


@pytest.fixture(scope="module")
def samplers():
    return {0: _sampler(), 2: _sampler("0,0"), 3: _sampler([0, 0, 0])}


def _write(d):
    import cv2
    rng = np.random.default_rng(7)
    (d / "in").mkdir()
    for name, (h, w) in IMAGES.items():
        cv2.imwrite(str(d / "in" / f"{name}.png"), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))


def _infer(s, d, out, noise_repeat=False):
    s.setup_seed()
    s.inference(d / "in", d / out, bs=len(IMAGES), noise_repeat=noise_repeat)
    return {p.name: p.read_bytes() for p in sorted((d / out).iterdir())}


def test_sampler_is_reproducible(samplers, tmp_path):
    from resshift_b200.models.autoencoder import AutoencoderKLTorch
    s = samplers[0]
    assert type(s.autoencoder) is AutoencoderKLTorch and s.autoencoder.cfg.embed_dim == 16
    _write(tmp_path)
    first = _infer(s, tmp_path, "first")
    assert sorted(first) == sorted(f"{n}.png" for n in IMAGES)
    assert _infer(s, tmp_path, "second") == first


@pytest.mark.parametrize("pool", [2, 3])
@pytest.mark.parametrize("chop_bs,noise_repeat", [(1, False), (5, True)])
def test_device_pool_equals_one_gpu(samplers, tmp_path, pool, chop_bs, noise_repeat):
    ref_s, s = samplers[0], samplers[pool]
    ref_s.chop_bs = s.chop_bs = chop_bs
    _write(tmp_path)
    assert _infer(s, tmp_path, "out", noise_repeat) == _infer(ref_s, tmp_path, "ref", noise_repeat)


@pytest.mark.parametrize("chop_bs,noise_repeat", [(1, False), (5, True)])
def test_virtual_ranks_equal_one_gpu(samplers, chop_bs, noise_repeat):
    from resshift_b200.parallel import unit_schedule
    from resshift_b200.sampler import tile_counts
    s = samplers[0]
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
