"""The VQ-GAN bottleneck attention up to 8192 positions (csrc/vq.inc, AttnBlock as three GEMMs on the conv kernel and
softmax_rows_kernel between them) at the sizes it serves: the face-restoration configuration at its native 512x512
(T = 4096, C = 512), small x4 inputs, and both sides of the 8192-position threshold above which the plans switch to the
fused kernel (covered by test_gpu_vq_attention.py).

References run in fp32 with TF32 off.  Operators are compared with fp32 torch on the same fp16 operands, plans with the
oracle on the GPU.  Tolerances are the repository's: max|d| <= 1e-2, mean|d| <= 2e-3 for plans, `_tol` of
test_gpu_ops.py for the GEMMs, fp16 rounding of the result for the softmax.
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import vq_oracle as vo
from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
from tests import plan_ops
from tests.gpu_util import fp32_matmuls

pytestmark = pytest.mark.gpu

TOL_MAX, TOL_MEAN = 1e-2, 2e-3


@pytest.fixture
def fp32_reference():
    with fp32_matmuls():
        yield


def _report(tag, got, ref):
    d = (got.float() - ref.float().to(got.device)).abs()
    print(f"[vq gemm attention] {tag}: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e} ref_std={ref.float().std().item():.3f}")
    return d.max().item(), d.mean().item()


# ------------------------------------------------------------------------------------------------ row softmax operator

def _softmax(s, rows, cols, ld, scale, offset=0):
    """rs_op_softmax_rows in place on the fp16 buffer s, starting `offset` elements in."""
    from resshift_b200 import _lib
    _lib.check(_lib.lib.rs_op_softmax_rows(s.data_ptr() + 2 * offset, rows, cols, ld, scale, _lib.current_stream()))
    torch.cuda.synchronize()


def _scores(rows, cols, scale, seed):
    """fp16 S [rows][cols] whose scaled scores have the shapes a softmax gets wrong: row 0 peaked (about -40 .. +40, the
    maximum in the last 8 columns), row 1 near-uniform, row 2 with its maximum in the first 8 columns, the rest normal
    with standard deviation 3.  A single row is the peaked one."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.randn(rows, cols, device="cuda", generator=g) * 3
    t[0] = torch.rand(cols, device="cuda", generator=g) * 70 - 40
    t[0, -8:] = 36 + 4 * torch.rand(8, device="cuda", generator=g)
    if rows > 1:
        t[1] = 1e-3 * torch.randn(cols, device="cuda", generator=g)
        t[2, :8] = 20 + torch.rand(8, device="cuda", generator=g)
    return (t / scale).half()


SOFTMAX_COLS = [8, 16, 264, 2048, 2880, 4096, 8192]
SOFTMAX_LAYOUTS = [(1, 0), (300, 0), (300, 24)]           # (rows, ld - cols)


@pytest.mark.parametrize("rows,pad", SOFTMAX_LAYOUTS, ids=[f"rows{r}-pad{p}" for r, p in SOFTMAX_LAYOUTS])
@pytest.mark.parametrize("cols", SOFTMAX_COLS)
def test_softmax_rows_vs_fp32(cols, rows, pad):
    scale = 512 ** -0.5
    ld = cols + pad
    s = _scores(rows, cols, scale, seed=cols + rows)
    ref = torch.softmax(s.float() * scale, dim=-1)
    if rows > 1:
        assert ref[0, -8:].sum().item() > 0.99 and ref[2, :8].sum().item() > 0.99
    sentinel = 1234.0
    buf = torch.full((rows, ld), sentinel, dtype=torch.float16, device="cuda")
    buf[:, :cols] = s
    _softmax(buf, rows, cols, ld, scale)
    p = buf[:, :cols].float()
    assert torch.isfinite(p).all()
    assert (buf[:, cols:] == sentinel).all(), "columns beyond cols were written"
    err = (p - ref).abs()
    big = ref >= 1e-4
    rel = (err[big] / ref[big]).max().item()
    small = err[~big].max().item() if (~big).any() else 0.0
    row_sum = (p.sum(-1) - 1).abs().max().item()
    print(f"[vq gemm attention] softmax cols={cols} rows={rows} ld={ld}: max rel {rel:.2e} (ref >= 1e-4), "
          f"max abs {small:.2e} (ref < 1e-4), max |row sum - 1| {row_sum:.2e}")
    assert rel <= 1e-3 and small <= 1e-6 and row_sum <= 2e-3
    # bit-reproducible
    again = torch.full_like(buf, sentinel)
    again[:, :cols] = s
    _softmax(again, rows, cols, ld, scale)
    assert torch.equal(again, buf)


def test_softmax_rows_refuses_what_it_would_get_wrong():
    from resshift_b200 import _lib
    buf = torch.zeros(4, 8224, dtype=torch.float16, device="cuda")
    before = buf.clone()
    bad = [
        (4, 8200, 8224, 0, "cols"),         # beyond the 8192 a row can hold
        (4, 12, 16, 0, "cols"),             # not a multiple of 8
        (4, 0, 16, 0, "cols"),
        (4, 64, 56, 0, "row stride"),       # ld = cols - 8
        (4, 64, 68, 0, "row stride"),       # ld not a multiple of 8
        (0, 64, 64, 0, "rows"),
        (4, 64, 64, 4, "aligned"),          # 8-byte aligned start
    ]
    for rows, cols, ld, offset, what in bad:
        with pytest.raises(_lib.RsError, match=what):
            _softmax(buf, rows, cols, ld, 1.0, offset=offset)
    assert torch.equal(buf, before)


# ----------------------------------------------------------------------------- the three GEMMs on the conv kernel

def _tol(ref):
    return 2e-3 * ref.abs().max().item() + 2e-3


def _gemm(x, ld, rows_hw, w, bias, cout):
    """rs_op_conv2d, ksize 1, as the attention plan runs it: x is [1, H, W, ld] pixels (its first K channels used), the
    "weight" w a dense fp16 [cout][K] tensor (Ipad = K, its row stride).  Returns the fp16 output [1, H, W, cout]."""
    from resshift_b200 import _lib
    H, W = rows_hw
    K = w.shape[1]
    out = torch.full((1, H, W, cout), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(_lib.lib.rs_op_conv2d(x.data_ptr(), 1, H, W, K, ld, w.data_ptr(), K, _lib.ptr(bias), cout, 1, 1, None, 0,
                                     out.data_ptr(), cout, None, 0, 0, _lib.current_stream()))
    torch.cuda.synchronize()
    return out


GEMM_HW = {1024: (32, 32), 2880: (40, 72), 4096: (64, 64), 8192: (64, 128)}
GEMM_CASES = [(t, c) for t in GEMM_HW for c in (128, 512)]


@pytest.mark.parametrize("gemm", ["qk", "pv", "wv"])
@pytest.mark.parametrize("T,Cc", GEMM_CASES, ids=[f"T{t}-C{c}" for t, c in GEMM_CASES])
def test_attention_gemm_shapes(fp32_reference, gemm, T, Cc):
    H, W = GEMM_HW[T]
    g = torch.Generator(device="cuda").manual_seed(T + Cc + len(gemm))
    # activation operands are image 1 of a batch-2 buffer: at a view offset inside a larger tensor, as the plan's are
    if gemm == "qk":                  # S = Q K^T: queries as pixels, keys [T][C] as the weight, Cout = T
        q = torch.randn(2, H, W, Cc, device="cuda", generator=g).half()
        k = torch.randn(2, T, Cc, device="cuda", generator=g).half()
        got = _gemm(q[1], Cc, (H, W), k[1], None, T).reshape(T, T)
        ref = q[1].reshape(T, Cc).float() @ k[1].float().t()
    elif gemm == "pv":                # O = P V + b_v: rows of P as pixels (K = T), V^T [C][T] as the weight, Cout = C
        p = torch.softmax(torch.randn(2, H, W, T, device="cuda", generator=g) * 2, dim=-1).half()
        vt = torch.randn(2, Cc, T, device="cuda", generator=g).half()
        b = torch.randn(Cc, device="cuda", generator=g) * 0.05
        got = _gemm(p[1], T, (H, W), vt[1], b, Cc).reshape(T, Cc)
        ref = p[1].reshape(T, T).float() @ vt[1].float().t() + b
    else:                             # V^T = W_v H_n^T: the rows of W_v as [1, C/64, 64] pixels, tokens [T][C], Cout = T
        wv = (torch.randn(Cc, Cc, device="cuda", generator=g) / Cc ** 0.5).half()
        hn = torch.randn(2, T, Cc, device="cuda", generator=g).half()
        got = _gemm(wv, Cc, (Cc // 64, 64), hn[1], None, T).reshape(Cc, T)
        ref = wv.float() @ hn[1].float().t()
    assert torch.isfinite(got).all()
    mx, mn = _report(f"gemm {gemm} T={T} C={Cc}", got, ref)
    assert mx <= _tol(ref)


# ------------------------------------------------------------------------------------------------------------ plans

def _vq(name, sd):
    from resshift_b200.models.autoencoder import VQModelTorch
    m = VQModelTorch(**vq_preset(name).to_kwargs())
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def _sd_cuda(cfg, seed=0):
    return {n: t.cuda() for n, t in random_vq_state_dict(cfg, seed).items()}


def _inputs(batch, h, w, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(batch, 3, h, w, device="cuda", generator=g) * 2 - 1
    return x, g


def _check_encode(tag, m, sd, cfg, x):
    got = m.encode(x)
    assert torch.isfinite(got).all()
    mx, mn = _report(tag, got, vo.vq_encode(x, sd, cfg))
    assert mx <= TOL_MAX and mn <= TOL_MEAN
    return got


def _check_decode(tag, m, sd, cfg, z):
    got = m.decode(z, force_not_quantize=True)
    assert torch.isfinite(got).all()
    mx, mn = _report(tag, got, vo.vq_decode(z, sd, cfg, force_not_quantize=True))
    assert mx <= TOL_MAX and mn <= TOL_MEAN
    return got


def test_f8_face_512_encode_decode(fp32_reference):
    """The face-restoration configuration at its native size: 512x512 images, a 64x64 bottleneck (T = 4096, C = 512)."""
    cfg = vq_preset("f8_face")
    sd = _sd_cuda(cfg)
    m = _vq("f8_face", sd)
    x, g = _inputs(2, 512, 512, seed=41)
    _check_encode("f8_face encode 512x512 b2 (T=4096 C=512)", m, sd, cfg, x)
    z = torch.randn(2, cfg.embed_dim, 64, 64, device="cuda", generator=g) * 0.6
    _check_decode("f8_face decode 64x64 latent b2 (not quantised)", m, sd, cfg, z)
    assert plan_ops.vq_rows(m.plan(1, 2, 512, 512)).count("softmax 4096") == 2


def test_f4_256_batch3(fp32_reference):
    """f4 encode at 256x256, batch 3 (T = 4096 per image): the per-image GEMM loop runs images 1 and 2 as well."""
    cfg = vq_preset("f4")
    sd = _sd_cuda(cfg)
    x, _ = _inputs(3, 256, 256, seed=42)
    _check_encode("f4 encode 256x256 b3", _vq("f4", sd), sd, cfg, x)


def test_f4_256_batch3_independence_and_determinism():
    """Image 1 of the batch-3 f4 encode is bit-identical when images 0 and 2 change, and runs are bit-reproducible."""
    m = _vq("f4", _sd_cuda(vq_preset("f4")))
    x, g = _inputs(3, 256, 256, seed=42)
    a = m.encode(x).clone()
    assert torch.equal(m.encode(x), a)
    x2 = torch.rand(x.shape, device="cuda", generator=g) * 2 - 1
    x2[1] = x[1]
    b = m.encode(x2)
    assert torch.equal(b[1], a[1])
    assert not torch.equal(b[0], a[0])


def test_tiny_160x288_non_power_of_two(fp32_reference):
    """tiny at 160x288: a 40x72 bottleneck, T = 2880 (not a multiple of 128, width not a power of two), C = 128."""
    cfg = vq_preset("tiny")
    sd = _sd_cuda(cfg, 3)
    m = _vq("tiny", sd)
    x, g = _inputs(2, 160, 288, seed=43)
    _check_encode("tiny encode 160x288 b2 (T=2880 C=128)", m, sd, cfg, x)
    z = torch.randn(2, cfg.embed_dim, 40, 72, device="cuda", generator=g) * 0.6
    _check_decode("tiny decode 40x72 latent b2 (not quantised)", m, sd, cfg, z)


THRESHOLD_CASES = [(512, 2, 8192), (544, 1, 8704)]


@pytest.mark.parametrize("width,batch,T", THRESHOLD_CASES, ids=[f"T{t}" for _, _, t in THRESHOLD_CASES])
def test_f4_both_sides_of_the_8192_threshold(fp32_reference, width, batch, T):
    """f4 at 256x512 (T = 8192, the longest S rows the row softmax takes) and 256x544 (T = 8704, the fused kernel):
    encode and decode against the oracle, and the op list shows which form ran."""
    cfg = vq_preset("f4")
    sd = _sd_cuda(cfg)
    m = _vq("f4", sd)
    x, g = _inputs(batch, 256, width, seed=T)
    _check_encode(f"f4 encode 256x{width} b{batch} (T={T})", m, sd, cfg, x)
    enc_rows = plan_ops.vq_rows(m.plan(0, batch, 256, width))
    z = torch.randn(batch, cfg.embed_dim, 64, width // 4, device="cuda", generator=g) * 0.6
    _check_decode(f"f4 decode 64x{width // 4} latent b{batch} (not quantised)", m, sd, cfg, z)
    dec_rows = plan_ops.vq_rows(m.plan(1, batch, 256, width))
    for rows in (enc_rows, dec_rows):
        softmax = [r for r in rows if r.startswith("softmax")]
        fused = [r for r in rows if r.startswith("vq_attn")]
        if T <= 8192:
            assert softmax == [f"softmax {T}"] * batch and fused == []
        else:
            assert softmax == [] and fused == [f"vq_attn T={T} C=512 N={batch}"]


# ------------------------------------------------------------------------------------------- peaked attention scores

def _attn_block_fp16_scores(record):
    """oracle.vq_oracle.attn_block with the plan's stated roundings: S = q.k rounded to fp16 once, then scaled and
    softmaxed in fp32 (what the reference does under autocast), P rounded to fp16, then P V.  The scaled scores' range
    is appended to `record`."""
    def attn_block(x, sd, p):
        h_ = vo._norm(x, sd, f"{p}.norm")
        q, k, v = (vo._conv(h_, sd, f"{p}.{n}") for n in ("q", "k", "v"))
        b, c, h, w = q.shape
        s = torch.bmm(q.reshape(b, c, h * w).permute(0, 2, 1), k.reshape(b, c, h * w)).half().float() * (int(c) ** (-0.5))
        record.append((s.min().item(), s.max().item()))
        p_ = F.softmax(s, dim=2).half().float()
        h_ = torch.bmm(v.reshape(b, c, h * w), p_.permute(0, 2, 1)).reshape(b, c, h, w)
        return x + vo._conv(h_, sd, f"{p}.proj_out")
    return attn_block


def test_f8_face_512_peaked_scores(fp32_reference, monkeypatch):
    """The q and k weights of encoder.mid.attn_1 scaled so that the scaled scores span about +-30 at 512x512 (softmax
    rows dominated by a few keys).  Held to the oracle with the plan's fp16 S and P (the stated contract); the plain fp32
    oracle's difference is printed for information."""
    cfg = vq_preset("f8_face")
    sd = _sd_cuda(cfg, 1)
    x, _ = _inputs(1, 512, 512, seed=44)
    span = []
    with monkeypatch.context() as mp:
        mp.setattr(vo, "attn_block", _attn_block_fp16_scores(span))
        vo.encoder(x, sd, cfg)
    a = (30.0 / max(abs(span[0][0]), abs(span[0][1]))) ** 0.5
    for n in ("q", "k"):
        for t in ("weight", "bias"):
            sd[f"encoder.mid.attn_1.{n}.{t}"] = sd[f"encoder.mid.attn_1.{n}.{t}"] * a
    m = _vq("f8_face", sd)
    got = m.encode(x)
    assert torch.isfinite(got).all()
    span.clear()
    with monkeypatch.context() as mp:
        mp.setattr(vo, "attn_block", _attn_block_fp16_scores(span))
        ref = vo.vq_encode(x, sd, cfg)
    lo, hi = span[0]
    print(f"[vq gemm attention] peaked: q, k scaled by {a:.3f}; scaled scores {lo:.1f} .. {hi:.1f}")
    assert max(abs(lo), abs(hi)) >= 25
    mx_plain, mn_plain = _report("f8_face encode 512x512 peaked vs plain fp32 oracle (information only)", got,
                                 vo.vq_encode(x, sd, cfg))
    mx, mn = _report("f8_face encode 512x512 peaked vs oracle with fp16 S and P", got, ref)
    assert mx <= TOL_MAX and mn <= TOL_MEAN
