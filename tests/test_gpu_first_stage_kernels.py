"""The first stage's GEMM-form attention (csrc/vq.inc attn_block: V^T = W_v H_n^T, S = Q K^T and O = P V^T + b_v on the
conv kernel, softmax_rows_kernel between them), its row softmax as an operator, and the quantiser's fused
post_quant_conv output, against float64 references with a bound per element.

u16 = 2^-11 (half an fp16 ulp, relative), u32 = 2^-23 (one fp32 operation; tensor-core accumulation may truncate, so a
full ulp), r32 = 2^-24 (one fp32 rounding to nearest), s16 = 2^-25 (half the fp16 subnormal spacing).

a. Row softmax (rs_op_softmax_rows) on fp16 S [rows][cols], against float64 softmax(scale S) on the same fp16 S.  Per
   element, with z = scale s the exact logit, m = max_j z_j and d = z - m <= 0, the kernel's weight e~ = __expf(fl(fl(s
   scale) - mx)) carries a relative error (as a perturbation of the exponent)
       rho = |z| r32          (the fp32 product s * scale)
           + |d| r32          (the subtraction of the row maximum; the maximum itself is one of the rounded logits, a
                               shift common to the row that the normalisation cancels)
           + (2 + 1.173 |d|) u32   (__expf: CUDA's documented 2 + floor(1.173 |x|) ulp)
   and below 2^-126 __expf flushes to zero (absolute 2^-126).  The row sum l adds the e~ of a thread in sequence (at most
   8 ceil(cols / 2048) of them), then 5 shuffle levels and the 8 warp partials in a fixed order: n_l = 8 ceil(cols /
   2048) + 12 roundings of r32 relative to the sum, which itself moves by sum_k p_k rho_k relative.  1 / l and the
   product cost two more.  So
       |p~ - p| <= 1/2 ulp16(p) + p expm1(rho + sum_k p_k rho_k + (n_l + 2) r32) + 2^-126,
   the fp16 store's half ulp taken down to the subnormal spacing.
   Geometry: cols from 8 to 8192, crossing each of the four 16-byte vectors a thread holds (2048 columns each) and the
   last warp's columns of a vector, and every T the plans of b run; rows 1, 300 and cols; a row stride beyond cols whose
   padding must stay untouched; a second run must be bit-identical.
   Input classes, one per row in turn: randn logits (sd 3), near-uniform (1e-3), all equal, peaked (logits in [-40, 30],
   one at +40) and gap (logits in [-55, -45], one at +50: the maximum exceeds every other logit by more than 88, so a
   maximum that misses a warp overflows __expf).  The peaked and gap maxima visit the first and last column and a column
   in the range of every warp of every vector the row reaches.

b. Every GEMM-form attention block of the plans below, the plan's own `<p>.attn` (probed under RS_NO_REUSE=1) against
   float64 attention of its probed fp16 `norm`, `q` and `k`, the fp16-rounded W_v (as pack_conv_weight_kernel rounds it)
   and the fp32 b_v.  For query i and channel c, with p_ij the exact softmax weights, v = n W_v^T the exact values and o
   = p v, the output o + b_v may differ by
       1/2 ulp16                                                      (the stored attention output)
     + sum_j p_ij a_v(j, c)                                           (V^T: its fp16 store, 1/2 ulp16(|v| + acc), plus
                                                                       the accumulation acc = C u32 sum_ci |w_c,ci| |n_j,ci|)
     + e_i exp(2 e_i) dev_ic                                          (S: its fp16 store plus C u32 sum_d |q_id| |k_jd|,
                                                                       times scale, max over j = e_i; pushed through the
                                                                       softmax as test_gpu_attention.py does, dev_ic =
                                                                       sqrt(sum_j p_ij (v_jc - o_ic)^2))
     + sum_j p_ij (rel_ij + u16) |v_jc| + s16 sum_j |v_jc|            (the softmax kernel's allowance rel of a and the
                                                                       fp16 store of P)
     + T u32 sum_j p_ij |v_jc| + u32 (|o_ic| + |b_c|)                 (the fp32 accumulation over T keys, the bias add)
   `<p>` (the block output) is held to float64 x + proj_out(attn) fed the probed `in` and `attn`: 1/2 ulp16 + (C + 2)
   u32 (sum |W_proj| |attn| + |b_proj| + |x|): this pins the residual and the per-image wiring; the conv itself is held
   by test_gpu_conv_instances.py.
   Weight classes of every attention block of a pass: as drawn; q and k scaled so that the scaled logits span about
   +-30 (peaked); q x 1e-3 (near-uniform); b_v replaced by 0.5 randn (bias).

c. The quantiser's output (`quantize`, the decoder's first conv input) against float64 post_quant_conv(codebook[idx])
   with the codes the kernel reported (last_indices), and against post_quant_conv(z) with force_not_quantize: E fmaf
   roundings, 1/2 ulp16 + E r32 (|b| + sum |w| |e|).  decode_code with an index outside [0, n_e) gives NaN at exactly
   that position.

test_coverage prints the worst ratio of each check to its allowance.
"""
import math
from dataclasses import replace

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from tests import gpu_util as G
    from tests import plan_ops
    from tests.first_stage_ref import (FTZ, R32, S16, SM_CLASSES, U16, U32, f32, no_reuse, softmax_allowance, softmax_case,
                                       tokens, w16)

W_CLASSES = ("drawn", "peaked", "uniform", "bias")

RAN = set()          # what ran
OBS = {}             # worst ratio per check


# ------------------------------------------------------------------------------------------------ a. row softmax

SOFTMAX_COLS = sorted({8, 16, 56, 64, 1792, 1800, 2048, 2056, 4096, 6144, 6152, 8184, 8192} |
                      {256, 384, 1024, 2880})          # the last four: the T of plans in b not among the first
SOFTMAX_ROWS = {"1": (lambda c: 1, 0), "300": (lambda c: 300, 24), "T": (lambda c: c, 8)}      # rows, ld - cols


@pytest.mark.parametrize("rows_key", list(SOFTMAX_ROWS))
@pytest.mark.parametrize("cols", SOFTMAX_COLS)
def test_softmax_rows(cols, rows_key):
    nrows, pad = SOFTMAX_ROWS[rows_key]
    for cls, r in softmax_case(nrows(cols), cols, cols + pad)[1].items():
        G.note(OBS, f"softmax {cls}", r)
        RAN.add(("softmax class", cls))
    RAN.add(("softmax cols", cols))


# ------------------------------------------------------------------------------------------------ b. plan attention

def options_config():
    """Attention at every level at C = 64, 192, 384 (a partial W_v tile at 64 and 192, channels not a power of two)."""
    from resshift_b200.vq_arch import vq_preset
    return replace(vq_preset("tiny"), ch=64, ch_mult=(1, 3, 6), attn_resolutions=(64, 32, 16))


def _config(kind, name):
    from resshift_b200.vq_arch import kl_preset, vq_preset
    if kind == "options":
        return options_config()
    return (kl_preset if kind == "kl" else vq_preset)(name)


# name -> (kind, preset, which, batch, image H, image W)
PLANS = {
    "vq_f4_encode_256_b1": ("vq", "f4", 0, 1, 256, 256),
    "vq_f4_encode_256_b3": ("vq", "f4", 0, 3, 256, 256),
    "vq_f4_decode_256_b3": ("vq", "f4", 1, 3, 256, 256),
    "vq_f8_face_decode_512_b1": ("vq", "f8_face", 1, 1, 512, 512),
    "vq_f4_encode_256x512_b2": ("vq", "f4", 0, 2, 256, 512),
    "vq_tiny_decode_160x288_b2": ("vq", "tiny", 1, 2, 160, 288),
    "vq_tiny_encode_32x32_b1": ("vq", "tiny", 0, 1, 32, 32),
    "kl_tiny_encode_64x96_b2": ("kl", "tiny", 0, 2, 64, 96),
    "kl_tiny_decode_64x96_b2": ("kl", "tiny", 1, 2, 64, 96),
    "kl_f8_encode_256_b1": ("kl", "f8", 0, 1, 256, 256),
    "options_encode_64_b2": ("options", None, 0, 2, 64, 64),
    "options_decode_64_b2": ("options", None, 1, 2, 64, 64),
}
# (C, T) of the attention blocks the plans above must reach between them
WANT_CT = {(512, 4096), (512, 8192), (128, 2880), (128, 64), (128, 384), (512, 1024), (64, 4096), (192, 1024), (384, 256)}


def attention_blocks(cfg, which):
    """Parameter prefixes of the attention blocks of a pass, in execution order."""
    if not cfg.has_attn:
        return []
    L = cfg.levels
    if which == 0:
        out = [f"encoder.down.{i}.attn.{j}" for i in range(L) if cfg.enc_attn[i] for j in range(cfg.num_res_blocks[i])]
        return out + ["encoder.mid.attn_1"]
    out = ["decoder.mid.attn_1"]
    return out + [f"decoder.up.{i}.attn.{j}" for i in reversed(range(L)) if cfg.dec_attn[i] for j in range(cfg.num_res_blocks[i] + 1)]


def check_block(tag, m, sd, key, p):
    """The block's attention output and block output against float64 (module docstring, b).  Returns C, T, the span of
    the scaled logits and the worst ratio to the bound of each check."""
    which, B, H, W = key
    pr = {s: m.probe(which, B, H, W, p + s) for s in (".in", ".norm", ".q", ".k", ".attn", "")}
    cc = pr[".q"].shape[1]
    T = pr[".q"].shape[2] * pr[".q"].shape[3]
    x, n, q, k, a, out = (tokens(pr[s]) for s in (".in", ".norm", ".q", ".k", ".attn", ""))
    wv, bv = w16(sd, f"{p}.v.weight", cc), sd[f"{p}.v.bias"].cuda().double()
    wp, bp = w16(sd, f"{p}.proj_out.weight", cc), sd[f"{p}.proj_out.bias"].cuda().double()
    scale = f32(cc ** -0.5)
    worst_a = worst_o = span = 0.0
    step = max(1, (1 << 23) // T)
    for b in range(B):
        v = n[b] @ wv.t()
        acc_v = cc * U32 * (n[b].abs() @ wv.abs().t())
        a_v = 0.5 * G.ulp16(v.abs() + acc_v) + acc_v
        kb = k[b]
        for r0 in range(0, T, step):
            r1 = min(T, r0 + step)
            qb = q[b, r0:r1]
            s = qb @ kb.t()
            acc_s = cc * U32 * (qb.abs() @ kb.abs().t())
            eps = scale * (0.5 * G.ulp16(s.abs() + acc_s) + acc_s).amax(-1, keepdim=True)
            z = scale * s
            span = max(span, z.abs().max().item())
            p_, rel = softmax_allowance(z, T)
            o = p_ @ v
            pv = p_ @ v.abs()
            dev = (p_ @ (v * v) - o * o).clamp(min=0).sqrt()
            allow = (p_ @ a_v + eps * torch.exp(2 * eps) * dev + (p_ * (rel + U16)) @ v.abs() + (S16 + FTZ) * v.abs().sum(0)
                     + T * U32 * pv + U32 * (o.abs() + bv.abs()))
            worst_a = max(worst_a, G.assert_within(f"{tag} {p}.attn image {b} rows {r0}:{r1}", a[b, r0:r1], o + bv, allow, 1.0))
        ref = x[b] + a[b] @ wp.t() + bp
        mag = a[b].abs() @ wp.abs().t() + bp.abs() + x[b].abs()
        worst_o = max(worst_o, G.assert_within(f"{tag} {p} image {b}", out[b], ref, (cc + 2) * U32 * mag, 1.0))
    return cc, T, span, worst_a, worst_o


def _model(kind, cfg, sd):
    from resshift_b200.models.autoencoder import AutoencoderKLTorch, VQModelTorch
    m = (AutoencoderKLTorch if kind == "kl" else VQModelTorch)(**cfg.to_kwargs())
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def _run_pass(m, kind, cfg, which, B, H, W, seed):
    g = G.gen(seed)
    if which == 0:
        x = torch.rand(B, 3, H, W, device="cuda", generator=g) * 2 - 1
        m.encode(x, sample_posterior=False) if kind == "kl" else m.encode(x)
    else:
        f = cfg.downscale
        z = torch.randn(B, cfg.embed_dim, H // f, W // f, device="cuda", generator=g) * 0.6
        m.decode(z) if kind == "kl" else m.decode(z, force_not_quantize=True)
    torch.cuda.synchronize()


def _weight_class(sd, cls, blocks, spans, g):
    """A copy of sd with every attention block of the pass in weight class cls."""
    out = dict(sd)
    for p in blocks:
        if cls == "peaked":
            a = math.sqrt(30.0 / spans[p])
            for n in ("q", "k"):
                for t in ("weight", "bias"):
                    out[f"{p}.{n}.{t}"] = sd[f"{p}.{n}.{t}"] * a
        elif cls == "uniform":
            for t in ("weight", "bias"):
                out[f"{p}.q.{t}"] = sd[f"{p}.q.{t}"] * 1e-3
        elif cls == "bias":
            out[f"{p}.v.bias"] = 0.5 * torch.randn(sd[f"{p}.v.bias"].shape, generator=g)
    return out


@pytest.mark.parametrize("plan", list(PLANS))
def test_plan_attention(plan):
    """Every GEMM-form attention block of the plan, in every weight class: `<p>.attn` and `<p>` within their float64
    bounds; the op list runs one row softmax of T columns per block and image, and no fused attention."""
    from resshift_b200.vq_arch import random_kl_state_dict, random_vq_state_dict
    kind, name, which, B, H, W = PLANS[plan]
    cfg = _config(kind, name)
    sd = (random_kl_state_dict if kind == "kl" else random_vq_state_dict)(cfg, 0)
    blocks = attention_blocks(cfg, which)
    assert blocks
    with no_reuse():
        m = _model(kind, cfg, sd)
        m.plan(which, B, H, W)
    key = (which, B, H, W)
    spans, ts = {}, {}
    g = torch.Generator().manual_seed(len(plan))
    for cls in W_CLASSES:
        sdc = _weight_class(sd, cls, blocks, spans, g)
        m.load_state_dict(sdc, strict=True)
        _run_pass(m, kind, cfg, which, B, H, W, seed=B * H + W)
        for p in blocks:
            cc, T, span, wa, wo = check_block(f"{plan} {cls}", m, sdc, key, p)
            if cls == "drawn":
                spans[p], ts[p] = span, T
            print(f"[plan] {plan} {cls} {p}: C={cc} T={T} scaled logits within +-{span:.1f}")
            if cls == "peaked":
                assert span >= 15, (p, span)
            G.note(OBS, f"attn {cls}", wa)
            G.note(OBS, "block output", wo)
            RAN.add(("ct", cc, T))
            RAN.add(("weight class", cls))
        if cls == "drawn":
            rows = plan_ops.vq_rows(m.plan(which, B, H, W))
            softmax = [r for r in rows if r.startswith("softmax")]
            want = sorted(f"softmax {ts[p]}" for p in blocks for _ in range(B))
            assert sorted(softmax) == want and not [r for r in rows if r.startswith("vq_attn")], (softmax, want)
            for r in softmax:
                RAN.add(("plan softmax", int(r.split()[1])))
    RAN.add(("plan", plan))


# ------------------------------------------------------------------------------------------------ c. quantiser output

def _post_quant_ref(e, sd):
    """float64 post_quant_conv of per-pixel vectors e [N, h, w, E] -> (NCHW output, its accumulation magnitude)."""
    w = sd["post_quant_conv.weight"].cuda()
    cz, E = w.shape[0], w.shape[1]
    w = w.reshape(cz, E).half().double()
    b = sd["post_quant_conv.bias"].cuda().double()
    y = e @ w.t() + b
    mag = e.abs() @ w.abs().t() + b.abs()
    return y.permute(0, 3, 1, 2), mag.permute(0, 3, 1, 2), E


QUANT_CASES = [("tiny", 2, 64, 64), ("f8_face", 1, 128, 128)]


@pytest.mark.parametrize("name,B,H,W", QUANT_CASES, ids=[c[0] for c in QUANT_CASES])
def test_quantize_output(name, B, H, W):
    """`quantize` = post_quant_conv(codebook[idx]) with the reported codes, = post_quant_conv(z) unquantised, and NaN at
    exactly the positions decode_code is given an index outside [0, n_e)."""
    from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
    cfg = vq_preset(name)
    sd = random_vq_state_dict(cfg, 1)
    sd["post_quant_conv.bias"] = 0.5 * torch.randn(sd["post_quant_conv.bias"].shape, generator=torch.Generator().manual_seed(3))
    m = _model("vq", cfg, sd)
    f = cfg.downscale
    g = G.gen(17)
    z = torch.randn(B, cfg.embed_dim, H // f, W // f, device="cuda", generator=g) * 0.6
    book = sd["quantize.embedding.weight"].cuda().double()
    m.decode(z)
    idx = m.last_indices.long()
    assert ((idx >= 0) & (idx < cfg.n_embed)).all()
    ref, mag, E = _post_quant_ref(book[idx], sd)
    got = m.probe(1, B, H, W, "quantize")
    G.note(OBS, "quantize codes", G.assert_within(f"{name} quantize (codes)", got, ref, E * R32 * mag, 1.0))
    m.decode(z, force_not_quantize=True)
    assert (m.last_indices == -1).all()
    ref_z, mag_z, _ = _post_quant_ref(z.double().permute(0, 2, 3, 1), sd)
    G.note(OBS, "quantize z", G.assert_within(f"{name} quantize (force_not_quantize)", m.probe(1, B, H, W, "quantize"),
                                              ref_z, E * R32 * mag_z, 1.0))
    bad = idx.clone()
    hits = [(0, 3, 5, cfg.n_embed), (B - 1, H // f - 2, 1, -1)]
    for n_, y_, x_, v_ in hits:
        bad[n_, y_, x_] = v_
    m.decode_code(bad)
    got = m.probe(1, B, H, W, "quantize")
    nan = torch.isnan(got)
    want = torch.zeros_like(nan)
    for n_, y_, x_, _ in hits:
        want[n_, :, y_, x_] = True
    assert torch.equal(nan, want), "NaN outside exactly the out-of-range positions"
    G.assert_within(f"{name} decode_code in-range positions", got[~want], ref[~want], E * R32 * mag[~want], 1.0)
    RAN.add(("quantize", name))


# ------------------------------------------------------------------------------------------------ d. coverage

def test_coverage():
    """Across the module (run it whole): every softmax T of the plans also ran as an operator case, every (C, T) of the
    plan table ran, and every input class.  Prints the worst ratio of error to allowance per check."""
    if not RAN:
        pytest.skip("run with the rest of the module")
    for check, r in sorted(OBS.items()):
        print(f"[observed] {check:26s} worst ratio {r:.3g}")
    missing = [p for p in PLANS if ("plan", p) not in RAN]
    assert not missing, missing
    plan_t = {r[1] for r in RAN if r[0] == "plan softmax"}
    op_cols = {r[1] for r in RAN if r[0] == "softmax cols"}
    assert plan_t and plan_t <= op_cols, sorted(plan_t - op_cols)
    ct = {r[1:] for r in RAN if r[0] == "ct"}
    assert WANT_CT <= ct, sorted(WANT_CT - ct)
    assert {("softmax class", c) for c in SM_CLASSES} <= RAN
    assert {("weight class", c) for c in W_CLASSES} <= RAN
    assert {("quantize", c[0]) for c in QUANT_CASES} <= RAN
