"""The nearest-code quantiser (vq_quantize_kernel, csrc/vq_kernels.cuh) through VQModelTorch.decode and last_indices,
with codebooks built here so that the right answer is known exactly: latents planted on codebook rows, exact ties across
and inside the kernel's 1024-code shared-memory chunks, latents whose position count leaves the last CTA partly empty,
and random latents against a float64 argmin with a stated rounding bound.

The decoded images are compared with the oracle on the GPU in fp32 (TF32 off) at the repository's tolerance, max|d| <=
1e-2 and mean|d| <= 2e-3: with planted codes there are no near-ties that could excuse a difference.
"""
import pytest
import torch

from oracle import vq_oracle as vo
from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
from tests.gpu_util import fp32_matmuls

pytestmark = pytest.mark.gpu

TOL_MAX, TOL_MEAN = 1e-2, 2e-3


@pytest.fixture
def fp32_reference():
    with fp32_matmuls():
        yield


def _report(tag, got, ref):
    d = (got.float() - ref.float().to(got.device)).abs()
    print(f"[vq quantizer] {tag}: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e} ref_std={ref.float().std().item():.3f}")
    return d.max().item(), d.mean().item()


def _vq(name, sd):
    from resshift_b200.models.autoencoder import VQModelTorch
    m = VQModelTorch(**vq_preset(name).to_kwargs())
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def _min_pair_dist2(cb, chunk=2048):
    """Smallest squared distance between two rows of cb (float64)."""
    c = cb.double()
    best = float("inf")
    for r0 in range(0, c.shape[0], chunk):
        d = torch.cdist(c[r0:r0 + chunk], c).pow(2)
        idx = torch.arange(r0, min(r0 + chunk, c.shape[0]), device=c.device)
        d[idx - r0, idx] = float("inf")
        best = min(best, d.min().item())
    return best


def _separated_codebook(n, E, seed):
    """n codes in E dimensions, no two closer than about 0.06, in shuffled order.  E = 3: a jittered 32 x 16 x 16
    grid with spacing 0.08 (random codes in 3-D have near-duplicates); otherwise normal with the spread of
    random_vq_state_dict's codebook."""
    g = torch.Generator().manual_seed(seed)
    if E == 3:
        assert n == 8192
        ax = [(torch.arange(k, dtype=torch.float32) - (k - 1) / 2) * 0.08 for k in (32, 16, 16)]
        cb = torch.stack(torch.meshgrid(*ax, indexing="ij"), dim=-1).reshape(-1, 3)
        cb = cb + (torch.rand(cb.shape, generator=g) - 0.5) * 0.02
        cb = cb[torch.randperm(n, generator=g)]
    else:
        cb = 0.6 * torch.randn(n, E, generator=g)
    return cb.cuda()


def _state_dict(cfg, codebook, seed=0):
    sd = {n: t.cuda() for n, t in random_vq_state_dict(cfg, seed).items()}
    sd["quantize.embedding.weight"] = codebook
    return sd


def _plant(codebook, codes, shape):
    """Latent [N, E, H, W] whose position p (in N, H, W order) is codebook row codes[p]."""
    N, H, W = shape
    return codebook[codes].reshape(N, H, W, -1).permute(0, 3, 1, 2).contiguous()


def _decode_vs_oracle(tag, m, sd, cfg, z, expected):
    """Quantised decode: the indices must be `expected` exactly (the oracle's too), the image the oracle's."""
    got = m.decode(z)
    idx = m.last_indices.reshape(-1).long()
    ref, ref_idx = vo.vq_decode(z, sd, cfg, return_indices=True)
    assert torch.equal(ref_idx.reshape(-1), expected), "the oracle disagrees with the planted codes"
    wrong = (idx != expected).nonzero().flatten()
    assert wrong.numel() == 0, f"{wrong.numel()} wrong indices, first at positions {wrong[:8].tolist()}: " \
                               f"got {idx[wrong[:8]].tolist()}, expected {expected[wrong[:8]].tolist()}"
    mx, mn = _report(tag, got, ref)
    assert mx <= TOL_MAX and mn <= TOL_MEAN


PLANTED = [("f4", 2), ("f8_face", 1)]


@pytest.mark.parametrize("name,batch", PLANTED, ids=[n for n, _ in PLANTED])
def test_planted_codes_every_code(fp32_reference, name, batch):
    """z set to codebook rows: every code of the codebook (8192 for f4, E = 3; 4096 for f8_face, E = 8) once, in random
    order, on 64x64 latents."""
    cfg = vq_preset(name)
    cb = _separated_codebook(cfg.n_embed, cfg.embed_dim, seed=5)
    sep = _min_pair_dist2(cb)
    print(f"[vq quantizer] {name}: {cfg.n_embed} codes, E = {cfg.embed_dim}, min squared distance between codes {sep:.2e}")
    assert sep >= 1e-3
    sd = _state_dict(cfg, cb)
    m = _vq(name, sd)
    codes = torch.randperm(cfg.n_embed, generator=torch.Generator().manual_seed(6)).cuda()
    assert batch * 64 * 64 == cfg.n_embed
    z = _plant(cb, codes, (batch, 64, 64))
    _decode_vs_oracle(f"{name} planted {cfg.n_embed} codes, decode", m, sd, cfg, z, codes)


def test_exact_ties_take_the_first_minimum(fp32_reference):
    """Identical codebook rows: 1023 and 1024 (the last code of the first 1024-code chunk and the first of the next), 17,
    1041 and 3093 (later chunks), 500 and 501 (inside one chunk).  Latents on any of them must get the lowest index,
    as torch.argmin does."""
    cfg = vq_preset("f4")
    cb = _separated_codebook(cfg.n_embed, cfg.embed_dim, seed=7)
    first = {1024: 1023, 1041: 17, 3093: 17, 501: 500}
    for dup, orig in first.items():
        cb[dup] = cb[orig]
    sd = _state_dict(cfg, cb)
    m = _vq("f4", sd)
    g = torch.Generator().manual_seed(8)
    tied = torch.tensor([1023, 1024, 17, 1041, 3093, 500, 501])
    codes = torch.cat([tied.repeat(16), torch.randint(0, cfg.n_embed, (192 - 16 * len(tied),), generator=g)])
    codes = codes[torch.randperm(codes.numel(), generator=g)]
    expected = torch.tensor([first.get(int(c), int(c)) for c in codes])
    z = _plant(cb, codes.cuda(), (1, 8, 24))
    _decode_vs_oracle("f4 exact ties, decode 8x24", m, sd, cfg, z, expected.cuda())


@pytest.mark.parametrize("h,w", [(8, 24), (8, 40)], ids=["192-positions", "320-positions"])
def test_partial_last_cta(fp32_reference, h, w):
    """N*H*W = 192 (one CTA of 256 threads, 64 idle) and 320 = 256 + 64 (the second CTA mostly idle), codes at both
    ends of the codebook and of the first chunk among the planted ones."""
    cfg = vq_preset("f4")
    cb = _separated_codebook(cfg.n_embed, cfg.embed_dim, seed=9)
    sd = _state_dict(cfg, cb)
    m = _vq("f4", sd)
    n = h * w
    g = torch.Generator().manual_seed(n)
    codes = torch.cat([torch.tensor([0, 1023, 1024, 8191]), torch.randint(0, cfg.n_embed, (n - 4,), generator=g)])
    codes = codes[torch.randperm(n, generator=g)].cuda()
    _decode_vs_oracle(f"f4 planted, decode {h}x{w} ({n} positions)", m, sd, cfg, _plant(cb, codes, (1, h, w)), codes)


def test_random_latents_vs_float64_argmin():
    """Random z against the shipped-size f4 codebook (8192 codes of random_vq_state_dict).  The kernel evaluates
    |z|^2 + |e|^2 - 2 z.e in fp32: each distance is off by at most about 1e-6 (|z|^2 + |e|^2), so where the float64
    margin between the best and second-best code exceeds bound = 1e-5 (|z|^2 + max(|e_best|^2, |e_second|^2)) the index
    must be the float64 argmin, and everywhere it must be a code within the bound of the minimum."""
    cfg = vq_preset("f4")
    sd = {n: t.cuda() for n, t in random_vq_state_dict(cfg, 0).items()}
    m = _vq("f4", sd)
    z = torch.randn(2, cfg.embed_dim, 64, 64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(10)) * 0.6
    m.decode(z)
    idx = m.last_indices.reshape(-1).long()
    zf = z.permute(0, 2, 3, 1).reshape(-1, cfg.embed_dim).double()
    e = sd["quantize.embedding.weight"].double()
    zz, ee = (zf * zf).sum(1), (e * e).sum(1)
    d = zz[:, None] + ee[None, :] - 2 * zf @ e.t()
    top = d.topk(2, dim=1, largest=False)
    dmin, best, second = top.values[:, 0], top.indices[:, 0], top.indices[:, 1]
    bound = 1e-5 * (zz + torch.maximum(ee[best], ee[second]))
    clear = (top.values[:, 1] - dmin) > bound
    print(f"[vq quantizer] random z: {int((~clear).sum())} of {idx.numel()} positions have a float64 margin below the bound "
          f"(median bound {bound.median().item():.1e}); {int((idx != best).sum())} differ from the float64 argmin")
    assert torch.equal(idx[clear], best[clear])
    assert (d.gather(1, idx[:, None]).squeeze(1) - dmin <= bound).all()


def test_force_not_quantize_writes_minus_one():
    cfg = vq_preset("f4")
    m = _vq("f4", random_vq_state_dict(cfg, 0))
    z = torch.randn(3, cfg.embed_dim, 16, 24, device="cuda", generator=torch.Generator(device="cuda").manual_seed(11)) * 0.6
    m.decode(z)
    assert (m.last_indices >= 0).all()
    m.decode(z, force_not_quantize=True)
    assert m.last_indices.shape == (3, 16, 24)
    assert (m.last_indices == -1).all()
