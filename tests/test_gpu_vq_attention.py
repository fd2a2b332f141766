"""The VQ-GAN bottleneck attention beyond 8192 positions (csrc/vq_attn.cuh): the fused online-softmax kernel through its
single-operator entry point, the encode / decode plans at sizes whose attention has more than 8192 positions, and the
x4 pipeline on a 128x128 LQ tile (a 512x512 image, a 128x128 bottleneck).

The operator tests hold it per element to float64 (the bound of tests/test_gpu_attention.py); the plan references run
in fp32 with TF32 off.  The oracle's attention is evaluated in chunks of query rows here (rows are
independent: the same math without the T x T temporaries, which are 17 GB each in fp32 at T = 65536).
Tolerances are the repository's: max|d| <= 1e-2, mean|d| <= 2e-3.  The default CLI tile (T = 262144, the 2048x2048
encode and decode) is held to float64 and to the oracle by test_gpu_cli_tile.py.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from oracle import vq_oracle as vo
from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
from tests.gpu_util import fp32_matmuls

TOL_MAX, TOL_MEAN = 1e-2, 2e-3

# rs_plan_num_launches of the f4 256x256 (64x64 latent, T = 4096) plans at batch 1, as before the fused kernel existed:
# bottlenecks up to 8192 positions keep the GEMM + row-softmax program launch for launch
F4_256_ENCODE_LAUNCHES = 58
F4_256_DECODE_LAUNCHES = 77


def _attention_chunked(q, k, v, rows=4096):
    """softmax(q^T k / sqrt(c)) applied to v on NCHW q, k, v, ``rows`` queries at a time (oracle attn_block's math)."""
    b, c, h, w = q.shape
    qt = q.reshape(b, c, h * w).permute(0, 2, 1)
    kf = k.reshape(b, c, h * w)
    vf = v.reshape(b, c, h * w)
    out = torch.empty_like(vf)
    for r0 in range(0, h * w, rows):
        w_ = F.softmax(torch.bmm(qt[:, r0:r0 + rows], kf) * (int(c) ** (-0.5)), dim=2)
        out[:, :, r0:r0 + rows] = torch.bmm(vf, w_.permute(0, 2, 1))
    return out.reshape(b, c, h, w)


def _attn_block_chunked(x, sd, p):
    """oracle.vq_oracle.attn_block with the attention evaluated by _attention_chunked."""
    h_ = vo._norm(x, sd, f"{p}.norm")
    q, k, v = (vo._conv(h_, sd, f"{p}.{n}") for n in ("q", "k", "v"))
    return x + vo._conv(_attention_chunked(q, k, v), sd, f"{p}.proj_out")


def test_chunked_oracle_attention_matches_unchunked():
    """CPU: the chunked evaluation used as the reference below equals the oracle's single-bmm AttnBlock at T = 16384."""
    cfg = vq_preset("tiny")
    sd = random_vq_state_dict(cfg, 0)
    top = cfg.ch * cfg.ch_mult[-1]
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1, top, 128, 128, generator=g)
    with torch.no_grad():
        a = vo.attn_block(x, sd, "encoder.mid.attn_1")
        b = _attn_block_chunked(x, sd, "encoder.mid.attn_1")
    d = (a - b).abs().max().item()
    print(f"[chunked oracle] T=16384 C={top}: max|d| = {d:.3e}")
    assert d <= 1e-5 * max(1.0, a.abs().max().item())


# ----------------------------------------------------------------------------------------------------------------- GPU

@pytest.fixture
def fp32_reference():
    with fp32_matmuls():
        yield


@pytest.fixture
def chunked_oracle(monkeypatch, fp32_reference):
    monkeypatch.setattr(vo, "attn_block", _attn_block_chunked)


def _report(tag, got, ref):
    d = (got.float() - ref.float().to(got.device)).abs()
    print(f"[vq attention] {tag}: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e} ref_std={ref.float().std().item():.3f}")
    return d.max().item(), d.mean().item()


def _op(q, k, v, ld=None):
    """rs_op_vq_attention on fp16 [N, T, C] tensors (q / k / v may be column slices of wider rows: row stride ld)."""
    from resshift_b200 import _lib
    N, T, Cc = q.shape
    out = torch.empty(N, T, Cc, dtype=torch.float16, device="cuda")
    _lib.check(_lib.lib.rs_op_vq_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), N, T, Cc, ld or Cc, out.data_ptr(),
                                           _lib.current_stream()))
    torch.cuda.synchronize()
    return out


def _ref_rows(q, k, v, rows, chunk=1024):
    """fp32 softmax(q k^T / sqrt(C)) v for the query rows `rows` of every image; q, k, v [N, T, C]."""
    Cc = q.shape[-1]
    kf, vf = k.float(), v.float()
    out = []
    for r0 in range(0, rows.numel(), chunk):
        r = rows[r0:r0 + chunk]
        s = torch.bmm(q[:, r].float(), kf.transpose(1, 2)) * Cc ** -0.5
        out.append(torch.bmm(torch.softmax(s, dim=-1), vf))
    return torch.cat(out, dim=1)


def _qkv(N, T, Cc, seed, ld=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ld = ld or Cc
    bufs = [torch.randn(N, T, ld, device="cuda", generator=g).half() for _ in range(3)]
    return [b[..., :Cc] for b in bufs]


OP_CASES = [(c, t) for c in (128, 256, 512) for t in (64, 384, 4096, 16384)] + [(512, 65536)]


@pytest.mark.gpu
@pytest.mark.parametrize("C,T", OP_CASES, ids=[f"C{c}-T{t}" for c, t in OP_CASES])
def test_op_vs_fp32(fp32_reference, C, T):
    """Per element against float64 on the fp16 operands (the bound of tests/test_gpu_attention.py)."""
    from tests.attn_ref import vq_check
    q, k, v = (t.contiguous() for t in _qkv(2, T, C, seed=C + T))
    vq_check("randn", q, k, v, _op(q, k, v))


@pytest.mark.gpu
def test_op_strided_rows(fp32_reference):
    """q, k, v as column slices of wider rows (row stride ld > C), as a plan view may be."""
    from tests.attn_ref import vq_check
    q, k, v = _qkv(2, 384, 256, seed=9, ld=384)
    vq_check("randn", q, k, v, _op(q, k, v, ld=384))


@pytest.mark.gpu
def test_op_peaked_softmax_max_in_last_block(fp32_reference):
    """Scaled scores spanning about -50 .. +50 with every row's maximum in the last 16 keys and its minimum in the first 16:
    the running maximum jumps at the very end, so everything accumulated before is rescaled by ~e^-20."""
    N, T, Cc = 2, 4096, 512
    g = torch.Generator(device="cuda").manual_seed(21)
    u = torch.randn(Cc, device="cuda", generator=g)
    q = (torch.randn(N, T, Cc, device="cuda", generator=g) + 2 * u) * 1.9
    k = torch.randn(N, T, Cc, device="cuda", generator=g) * 1.9
    k[:, -16:] = 0.58 * u + 0.05 * torch.randn(N, 16, Cc, device="cuda", generator=g)
    k[:, :16] = -0.58 * u + 0.05 * torch.randn(N, 16, Cc, device="cuda", generator=g)
    v = torch.randn(N, T, Cc, device="cuda", generator=g)
    q, k, v = q.half(), k.half(), v.half()
    s = torch.bmm(q[:, :512].float(), k.float().transpose(1, 2)) * Cc ** -0.5
    print(f"[vq attention] peaked: scores {s.min().item():.1f} .. {s.max().item():.1f}")
    assert (s.argmax(-1) >= T - 16).all() and (s.argmin(-1) < 16).all()
    assert s.max().item() >= 40 and s.min().item() <= -40
    from tests.attn_ref import vq_check
    vq_check("peaked", q, k, v, _op(q, k, v))


@pytest.mark.gpu
def test_op_default_cli_tile_sampled_rows(fp32_reference):
    """T = 262144 (a 512x512 LQ tile at the f4 bottleneck, the CLI's default chop size), checked on 2048 sampled rows."""
    N, T, Cc = 1, 262144, 512
    q, k, v = (t.contiguous() for t in _qkv(N, T, Cc, seed=5))
    out = _op(q, k, v)
    rows = torch.randperm(T, generator=torch.Generator().manual_seed(6))[:2048].sort().values.cuda()
    ref = _ref_rows(q, k, v, rows, chunk=256)
    assert torch.isfinite(out).all()
    mx, mn = _report("op C=512 T=262144 (2048 rows)", out[:, rows], ref)
    assert mx <= TOL_MAX and mn <= TOL_MEAN


@pytest.mark.gpu
def test_op_rejects_unsupported_shapes():
    from resshift_b200 import _lib
    q = torch.zeros(1, 128, 192, dtype=torch.float16, device="cuda")
    out = torch.empty_like(q)
    with pytest.raises(_lib.RsError, match="C in"):
        _lib.check(_lib.lib.rs_op_vq_attention(q.data_ptr(), q.data_ptr(), q.data_ptr(), 1, 128, 192, 192, out.data_ptr(),
                                               _lib.current_stream()))
    q = torch.zeros(1, 96, 128, dtype=torch.float16, device="cuda")
    with pytest.raises(_lib.RsError, match="multiple of 64"):
        _lib.check(_lib.lib.rs_op_vq_attention(q.data_ptr(), q.data_ptr(), q.data_ptr(), 1, 96, 128, 128, q.data_ptr(),
                                               _lib.current_stream()))


# ------------------------------------------------------------------------------------------------ plans, pipeline

def _vq(name, seed=0):
    from resshift_b200.models.autoencoder import VQModelTorch
    cfg = vq_preset(name)
    m = VQModelTorch(**cfg.to_kwargs())
    m.load_state_dict(random_vq_state_dict(cfg, seed), strict=True)
    return cfg, m.cuda().eval()


def _sd_cuda(cfg, seed=0):
    return {n: t.cuda() for n, t in random_vq_state_dict(cfg, seed).items()}


@pytest.mark.gpu
def test_f4_encode_1024(chunked_oracle):
    """f4 encode of a 1024x1024 image: a 256x256 bottleneck, T = 65536."""
    cfg, m = _vq("f4")
    x = torch.rand(1, 3, 1024, 1024, device="cuda", generator=torch.Generator(device="cuda").manual_seed(11)) * 2 - 1
    got = m.encode(x)
    assert torch.isfinite(got).all()
    mx, mn = _report("f4 encode 1024x1024", got, vo.vq_encode(x, _sd_cuda(cfg), cfg))
    assert mx <= TOL_MAX and mn <= TOL_MEAN


@pytest.mark.gpu
def test_f4_decode_256_latent(chunked_oracle):
    """f4 decode (not quantised) of a 256x256 latent (a 1024x1024 image), T = 65536."""
    cfg, m = _vq("f4")
    z = torch.randn(1, 3, 256, 256, device="cuda", generator=torch.Generator(device="cuda").manual_seed(12)) * 0.6
    got = m.decode(z, force_not_quantize=True)
    assert torch.isfinite(got).all()
    mx, mn = _report("f4 decode 256x256 latent", got, vo.vq_decode(z, _sd_cuda(cfg), cfg, force_not_quantize=True))
    assert mx <= TOL_MAX and mn <= TOL_MEAN


@pytest.mark.gpu
def test_f8_face_encode_1024(chunked_oracle):
    """f8_face encode of a 1024x1024 image: a 128x128 bottleneck, T = 16384."""
    cfg, m = _vq("f8_face")
    x = torch.rand(1, 3, 1024, 1024, device="cuda", generator=torch.Generator(device="cuda").manual_seed(13)) * 2 - 1
    got = m.encode(x)
    mx, mn = _report("f8_face encode 1024x1024", got, vo.vq_encode(x, _sd_cuda(cfg), cfg))
    assert mx <= TOL_MAX and mn <= TOL_MEAN


@pytest.mark.gpu
def test_tiny_non_square_512x768(chunked_oracle):
    """tiny encode / decode at 512x768 (a 128x192 bottleneck, T = 24576, C = 128)."""
    cfg, m = _vq("tiny", seed=2)
    sd = _sd_cuda(cfg, 2)
    g = torch.Generator(device="cuda").manual_seed(14)
    x = torch.rand(2, 3, 512, 768, device="cuda", generator=g) * 2 - 1
    z = torch.randn(2, 3, 128, 192, device="cuda", generator=g) * 0.6
    mx, mn = _report("tiny encode 512x768", m.encode(x), vo.vq_encode(x, sd, cfg))
    assert mx <= TOL_MAX and mn <= TOL_MEAN
    mx, mn = _report("tiny decode 128x192 (not quantised)", m.decode(z, force_not_quantize=True),
                     vo.vq_decode(z, sd, cfg, force_not_quantize=True))
    assert mx <= TOL_MAX and mn <= TOL_MEAN


@pytest.mark.gpu
def test_batch_independence_and_determinism_t16384():
    """Image i of a batch does not depend on its neighbours and runs are bit-reproducible at T = 16384."""
    cfg, m = _vq("tiny")
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.rand(3, 3, 512, 512, device="cuda", generator=g) * 2 - 1
    a = m.encode(x).clone()
    assert torch.equal(a, m.encode(x))
    x2 = torch.rand_like(x) * 2 - 1
    x2[1] = x[1]
    assert torch.equal(m.encode(x2)[1], a[1])
    z = torch.randn(3, 3, 128, 128, device="cuda", generator=g) * 0.6
    d = m.decode(z).clone()
    assert torch.equal(d, m.decode(z))
    z2 = torch.randn_like(z) * 0.6
    z2[2] = z[2]
    assert torch.equal(m.decode(z2)[2], d[2])


@pytest.mark.gpu
def test_plan_takes_fused_kernel_above_8192_only():
    """One fused launch per attention block above 8192 positions; the GEMM + row-softmax program (same launch count as
    before the fused kernel existed) at and below."""
    from resshift_b200 import _lib
    cfg, m = _vq("f4")
    enc, dec = m.plan(0, 1, 256, 256), m.plan(1, 1, 256, 256)
    print(f"[vq attention] f4 256x256 launches: encode {enc.launches} decode {dec.launches}")
    assert enc.launches == F4_256_ENCODE_LAUNCHES and dec.launches == F4_256_DECODE_LAUNCHES
    cfg, m = _vq("tiny")
    x = torch.rand(1, 3, 512, 512, device="cuda") * 2 - 1
    m.encode(x)
    cap, stride = 1024, 160
    ms = (C.c_double * cap)()
    desc = C.create_string_buffer(cap * stride)
    n = C.c_int32()
    _lib.check(_lib.lib.rs_vq_profile_ops(m.plan(0, 1, 512, 512).handle, ms, desc, stride, cap, C.byref(n), _lib.current_stream()))
    rows = [desc.raw[i * stride:(i + 1) * stride].split(b"\0")[0].decode() for i in range(n.value)]
    assert [r for r in rows if r.startswith("vq_attn")] == ["vq_attn T=16384 C=128 N=1"]
    assert not any(r.startswith("softmax") for r in rows)


def _sampler(sf, **kw):
    from resshift_b200.config import preset
    from resshift_b200.sampler import ResShiftSampler, make_configs
    from resshift_b200.weights import random_state_dict
    ucfg, dcfg = preset("tiny")
    dcfg.sf = sf
    vcfg = vq_preset("tiny")
    ae = {"target": "ldm.models.autoencoder.VQModelTorch", "params": vcfg.to_kwargs(), "ckpt_path": random_vq_state_dict(vcfg, 0)}
    configs = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    return ResShiftSampler(configs, sf=sf, use_amp=True, seed=123, **kw)


@pytest.mark.gpu
def test_pipeline_128_lq_tile(chunked_oracle):
    """x4 on a 128x128 LQ tile without tiling (chop_size 512): bicubic x4 -> encode (T = 16384) -> loop on a 128x128
    latent -> decode (T = 16384)."""
    s = _sampler(4, chop_size=512, chop_stride=448, padding_offset=16)
    vcfg = vq_preset("tiny")
    sd_v = _sd_cuda(vcfg, 0)
    g = torch.Generator(device="cuda").manual_seed(31)
    y0 = torch.rand(1, 3, 128, 128, device="cuda", generator=g) * 2 - 1
    out = s.sample_func(y0, noise_repeat=False, mask=None).float()
    assert out.shape == (1, 3, 512, 512) and torch.isfinite(out).all() and out.abs().max().item() <= 1.0
    # z_y after bicubic + encode
    diff, ae = s.base_diffusion, s.autoencoder
    z_y = diff.encode_first_stage(y0, ae, up_sample=True)
    z_y_ref = vo.vq_encode(vo.bicubic_upsample(y0, 4), sd_v, vcfg)
    mx, mn = _report("pipeline 128 LQ: z_y (bicubic x4 + encode)", z_y, z_y_ref)
    assert mx <= TOL_MAX and mn <= TOL_MEAN
    # decoder on the oracle's latent
    img_ref, idx_ref = vo.vq_decode(z_y_ref, sd_v, vcfg, return_indices=True)
    img = ae.decode(z_y_ref)
    flips = (ae.last_indices != idx_ref).float().mean().item()
    mx, mn = _report(f"pipeline 128 LQ: decode(quantise(z_ref)), code flips {flips * 100:.3f} %", img, img_ref)
    assert flips <= 0.002 and mn <= TOL_MEAN
    if flips == 0:
        assert mx <= TOL_MAX
