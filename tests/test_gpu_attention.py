"""Every attention kernel instance, and each attention the shipped plans run on one of them, against float64 references
on the fp16 operands, with a bound per output element.

Kernels: window_attn_kernel<WS, HD> (WS 8 / 16, HD 32 / 64) and the SIMT cross-check (rs_op_window_attention_cfg, with
forced heads per CTA), swin_attn_fused_kernel<E> (rs_op_swin_attn_ex, with forced persistent grids), unet_attn_sm90_kernel
<D> (rs_op_unet_attention) and vq_attn_sm90_kernel<C> (rs_op_vq_attention / _rows).  The first stage's attention over
8192 positions or fewer runs in GEMM form instead (three GEMMs on the conv kernel with softmax_rows_kernel between them,
csrc/vq.inc attn_block); test_gpu_first_stage_kernels.py holds every such block of the first-stage plans and the row
softmax to float64.  test_gpu_cli_tile.py holds vq_attn_sm90_kernel<512> at T = 262144 (the default CLI tile), where
the bound below is too loose to see a lost key block in these classes and a "needle" class is added.

Bound.  For query row i and output channel c, with p_ij the exact (float64) softmax weights, o_ic the exact output and
u16 = 2^-11, u32 = 2^-23 (one fp32 operation; tensor-core accumulation may truncate, so a full ulp):

    |o~ - o| <= 1/2 ulp16 + kP * sum_j p_ij |v_jc| + kS * L_i * dev_ic + s16 * sum_j |v_jc| / l_i

  * The kernels round the unnormalised weights P = exp(s - max) to fp16 for the PV MMA (relative error u16, or an
    absolute 2^-25 below the fp16 normal range: the s16 term, with l_i = sum_j exp(s_ij - max_i) >= 1) while the row sum
    stays fp32.  O and the row sum accumulate in fp32: n_O additions into O (one per k16 MMA step, plus one rescale per
    64-key block for the online kernels) and n_l into the row sum, each relative to the magnitudes summed; the
    normalisation costs two more roundings, ex2.approx a relative 2^-22.  So kP = u16 + (n_O + n_l + 4) u32 + 2^-22:
      - window / fused Swin cores: n_O = T/16, n_l = T/4 + 2 (a lane's 16 or 64 keys, then two shuffles);
      - unet / VQ online softmax: n_O = ceil(T/16) + ceil(T/64), n_l = 18 + 2 ceil(T/64).
    The SIMT cross-check keeps P in fp32 and accumulates with fmaf in round-to-nearest: kP = (2T + 6) 2^-24 + 2^-22, and
    no s16 term.
  * A logit error d_j changes o by sum_j p_ij d_j (v_jc - o_ic), at most max|d| * sum_j p_ij |v_jc - o_ic|; dev_ic =
    sqrt(sum_j p_ij (v_jc - o_ic)^2) bounds that sum from above (Jensen).  The logits accumulate D products in fp32, then
    take the scale, the bias, the mask, the max subtraction and the log2(e) factor of __expf / exp2 (the last two on
    values up to 2 L_i): |d| <= kS L_i with kS = (D + 7) u32 (D + 8 for VQ, which adds two channel halves), where
    L_i = max_j (scale sum_d |q_id| |k_jd| + |bias_ij|) (bias includes the -100 of the shift mask).
  * Equal logits (q = 0, no bias): every P is exactly 1, so only the accumulation part of kP applies.

The fused Swin reference reproduces the unfused path's fp16 stores (norm1 output, qkv, attention output) on float64
values and carries an allowance forward through each stage: the fp16 ulp of the stored intermediate (kernel and
reference may round neighbouring values apart), the stage's own term, and the previous allowance pushed through the
stage in absolute values (|W| * allow for the GEMMs; for attention sum_j p_ij allow(v_jc) plus the logit perturbation
e_i = scale max_j sum_d (a(q) |k| + |q| a(k) + a(q) a(k)) times e^(2 e_i) dev_ic).  norm1 allows a group-mean error of
64 * 2^-24 (|mean| + std) and a relative rstd error of 1024 * 2^-24 on top of the fp32 affine fold.

The worst ratio of each check to its allowance is printed per kernel and input class by test_coverage.
"""
import ctypes as C
import math
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from tests import gpu_util as G
    from resshift_b200 import _lib
    from resshift_b200.arch import relative_position_index, shifted_window_mask

U16, U32, S16 = 2.0 ** -11, 2.0 ** -23, 2.0 ** -25
EX2 = 2.0 ** -22
INSTANCES = [(8, 32), (8, 64), (16, 32), (16, 64)]
CLASSES = ("randn", "peaked", "probe", "equal", "large")
SLOTS = (1, 4, 15, 16, 17, 32, 128, 512)

RAN = set()          # what ran: (kind, feature)
OBS = {}             # worst ratio per (kernel, input class)


def _note(kernel, cls, ratio):
    OBS[(kernel, cls)] = max(OBS.get((kernel, cls), 0.0), ratio)
    RAN.add(("class", kernel, cls))


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ float64 softmax core

def kappas(kind, T, D, exact_p=False):
    """(kP, kS, s16) of the module docstring for a kernel kind at T keys and head width D."""
    if kind == "simt":
        return (2 * T + 6) * 2.0 ** -24 + EX2, (D + 7) * U32, 0.0
    if kind in ("window", "swin"):
        n_o, n_l, ks = T // 16, T // 4 + 2, (D + 7) * U32
    else:
        nb = -(-T // 64)
        n_o, n_l, ks = -(-T // 16) + nb, 18 + 2 * nb, (D + (8 if kind == "vq" else 7)) * U32
    kp = (n_o + n_l + 4) * U32 + EX2
    return (kp, ks, 0.0) if exact_p else (kp + U16, ks, S16)


def softmax_ref(q, k, v, scale, bias=None, err=None):
    """float64 attention on [..., T, D] operands; bias broadcasts to [..., Tq, T].  Returns o and the pieces of the
    bound: pv = sum p|v|, dev, L, sub = sum|v| / l, and with err = (a_q, a_k, a_v) the allowance of the operands pushed
    through the softmax."""
    s = scale * (q @ k.transpose(-1, -2))
    if bias is not None:
        s = s + bias
    m = s.amax(-1, keepdim=True)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    p = e / l
    o = p @ v
    r = {"o": o, "pv": p @ v.abs(), "dev": (p @ (v * v) - o * o).clamp(min=0).sqrt()}
    lg = scale * (q.abs() @ k.abs().transpose(-1, -2))
    if bias is not None:
        lg = lg + bias.abs()
    r["L"] = lg.amax(-1, keepdim=True)
    r["sub"] = v.abs().sum(-2, keepdim=True) / l
    if err is not None:
        aq, ak, av = err
        eps = scale * (aq @ k.abs().transpose(-1, -2) + q.abs() @ ak.transpose(-1, -2) + aq @ ak.transpose(-1, -2)).amax(-1, keepdim=True)
        r["prop"] = p @ av + eps * torch.exp(2 * eps) * r["dev"]
    return r


def allowance(r, kp, ks, s16):
    a = kp * r["pv"] + ks * r["L"] * r["dev"] + s16 * r["sub"]
    return a + r["prop"] if "prop" in r else a


# ------------------------------------------------------------------------------------------------ window layout

def to_windows(t, ws, shift):
    """[N, H, W, C] -> [N * nWy * nWx, ws * ws, C]: the tokens of the shifted partition."""
    N, H, W, Cc = t.shape
    if shift:
        t = torch.roll(t, (-shift, -shift), (1, 2))
    return t.reshape(N, H // ws, ws, W // ws, ws, Cc).permute(0, 1, 3, 2, 4, 5).reshape(-1, ws * ws, Cc)


def from_windows(w, N, H, W, ws, shift):
    Cc = w.shape[-1]
    t = w.reshape(N, H // ws, W // ws, ws, ws, Cc).permute(0, 1, 3, 2, 4, 5).reshape(N, H, W, Cc)
    return torch.roll(t, (shift, shift), (1, 2)) if shift else t


def window_bias(table, heads, ws, N, H, W, shift):
    """[B, heads, T, T] float64: relative_position_bias_table gathered by relative_position_index, + the shift mask."""
    T = ws * ws
    b = table.double()[relative_position_index(ws).reshape(-1).to(table.device)].view(T, T, heads).permute(2, 0, 1)
    nW = (H // ws) * (W // ws)
    if not shift:
        return b[None].expand(N * nW, heads, T, T)
    m = shifted_window_mask(H, W, ws, shift).to(table.device).double()
    return (b[None, None] + m[None, :, None]).expand(N, nW, heads, T, T).reshape(N * nW, heads, T, T)


def _table(cls, heads, ws, g):
    n = (2 * ws - 1) ** 2
    if cls == "equal":
        return torch.zeros(n, heads, device="cuda")
    if cls == "probe":      # distinct entries spanning +-6: a transposed or shifted gather moves every weight
        perm = torch.randperm(n * heads, device="cuda", generator=g).float()
        return (perm / (n * heads - 1) * 12 - 6).view(n, heads)
    return torch.randn(n, heads, device="cuda", generator=g) * 0.5


def _qkv_class(cls, B, T, heads, D, scale, g, targets=None):
    """q, k, v [B, heads, T, D] float32 of an input class; targets[b] = the key every query row of b peaks on."""
    q = torch.randn(B, heads, T, D, device="cuda", generator=g)
    k = torch.randn(B, heads, T, D, device="cuda", generator=g)
    v = torch.randn(B, heads, T, D, device="cuda", generator=g)
    if cls in ("probe", "equal"):
        q.zero_()
    elif cls == "peaked":   # logits in [-40, 15], the target key at +40
        a = 8.0
        b = 40.0 / (scale * a)
        q.zero_()
        q[..., 0] = a
        k.zero_()
        k[..., 0] = b * (torch.rand(B, heads, T, device="cuda", generator=g) * 1.375 - 1)
        k[torch.arange(B, device="cuda"), :, targets, 0] = b
    elif cls == "large":    # |v| near 3e4, logits near +-1e3
        a = math.sqrt(1000.0 / scale)
        q.zero_()
        q[..., 0] = a
        k.zero_()
        k[..., 0] = a * (torch.rand(B, heads, T, device="cuda", generator=g) * 2 - 1)
        sign = torch.where(torch.rand(B, heads, T, D, device="cuda", generator=g) < 0.5, -1.0, 1.0)
        v = 3e4 * (0.8 + 0.2 * torch.rand(B, heads, T, D, device="cuda", generator=g)) * sign
    return q, k, v


# ------------------------------------------------------------------------------------------------ window core

def run_window(qkv, dense, heads, ws, hd, shift, hpc, simt):
    N, H, W, _ = qkv.shape
    out = torch.full((N, H, W, heads * hd), float("nan"), dtype=torch.float16, device="cuda")
    info = (C.c_int32 * 5)()
    _lib.check(_lib.lib.rs_op_window_attention_cfg(qkv.data_ptr(), N, H, W, heads, ws, hd, shift, dense.data_ptr(),
                                                   out.data_ptr(), hpc, int(simt), info, G.stream()))
    torch.cuda.synchronize()
    return out, {"simt": info[0], "hpc": info[1], "grid": (info[2], info[3]), "smem": info[4]}


def default_hpc(heads, windows):
    """The launcher's rule (launch.cuh attn_default_hpc)."""
    hpc = heads
    while hpc > 1 and windows * (heads // hpc) < 4 * _sms() and hpc % 2 == 0:
        hpc //= 2
    if hpc > 1 and windows * (heads // hpc) < 4 * _sms():
        hpc = 1
    return hpc


class WindowCase:
    def __init__(self, cls, N, nwy, nwx, heads, ws, hd, shift, seed):
        self.cls, self.N, self.H, self.W, self.heads, self.ws, self.hd, self.shift = cls, N, nwy * ws, nwx * ws, heads, ws, hd, shift
        g = _gen(seed)
        T, B = ws * ws, N * nwy * nwx
        scale = hd ** -0.5
        # peaked: the target key of a window at its first or last token, or either side of the mask's label boundary
        # (columns ws - shift - 1 and ws - shift of the last token row)
        s = ws // 2
        choices = torch.tensor([0, T - 1, (ws - 1) * ws + ws - s - 1, (ws - 1) * ws + ws - s], device="cuda")
        targets = choices[torch.arange(B, device="cuda") % 4]
        q, k, v = _qkv_class(cls, B, T, heads, hd, scale, g, targets)
        w = torch.stack([q, k, v], 1).permute(0, 3, 1, 2, 4).reshape(B, T, 3 * heads * hd)
        self.qkv = from_windows(w, N, self.H, self.W, ws, shift).half().contiguous()
        self.table = _table(cls, heads, ws, g)
        self.dense = torch.empty(heads * T * T, dtype=torch.float32, device="cuda")
        _lib.check(_lib.lib.rs_op_expand_relpos_ex(self.table.data_ptr(), self.dense.data_ptr(), heads, ws, G.stream()))
        x = to_windows(self.qkv.double(), ws, shift).view(B, T, 3, heads, hd).permute(2, 0, 3, 1, 4)
        self.r = softmax_ref(x[0], x[1], x[2], scale, window_bias(self.table, heads, ws, N, self.H, self.W, shift))
        self.ref = from_windows(self.r["o"].permute(0, 2, 1, 3).reshape(B, T, heads * hd), N, self.H, self.W, ws, shift)

    def check(self, tag, hpc=0, simt=False):
        out, info = run_window(self.qkv, self.dense, self.heads, self.ws, self.hd, self.shift, hpc, simt)
        kind = "simt" if simt else "window"
        kp, ks, s16 = kappas(kind, self.ws * self.ws, self.hd, exact_p=self.cls == "equal")
        B, T = self.r["o"].shape[0], self.ws * self.ws
        a = allowance(self.r, kp, ks, s16).permute(0, 2, 1, 3).reshape(B, T, -1)
        a = from_windows(a, self.N, self.H, self.W, self.ws, self.shift)
        ratio = G.assert_within(tag, out, self.ref, a, 1.0)
        kernel = "window_simt" if simt else f"window<{self.ws},{self.hd}>"
        _note(kernel, self.cls, ratio)
        RAN.add(("instance", kernel))
        if not simt:
            RAN.add(("hpc", kernel, "1" if info["hpc"] == 1 else "all" if info["hpc"] == self.heads else "divisor"))
        return out, info


WINDOW_SHAPES = [(1, 1, 1, False), (3, 3, 5, False), (3, 3, 5, True), (1, 2, 3, True)]


def _divisors(n):
    return [d for d in range(1, n + 1) if n % d == 0]


@pytest.mark.parametrize("shape", WINDOW_SHAPES, ids=lambda s: f"N{s[0]}-{s[1]}x{s[2]}-shift{int(s[3])}")
@pytest.mark.parametrize("ws,hd,heads", [(8, 32, 6), (8, 64, 4), (16, 32, 6), (16, 64, 4), (8, 32, 3), (16, 64, 1)])
def test_window_core_every_hpc(ws, hd, heads, shape):
    """randn operands: every heads-per-CTA count (1, each proper divisor, all heads) and the SIMT kernel agree with
    float64, and the entry reports the launch it was asked for."""
    N, nwy, nwx, shifted = shape
    L = WindowCase("randn", N, nwy, nwx, heads, ws, hd, ws // 2 if shifted else 0, seed=ws * 131 + hd + heads + nwx + shifted)
    outs = []
    for hpc in _divisors(heads):
        out, info = L.check(f"window<{ws},{hd}> heads={heads} {shape} hpc={hpc}", hpc=hpc)
        assert info["hpc"] == hpc and info["grid"] == (N * nwy * nwx, heads // hpc) and info["simt"] == 0, info
        outs.append(out)
    assert all(torch.equal(outs[0], o) for o in outs[1:]), "results depend on the heads per CTA"
    _, info = L.check(f"window simt ws={ws} hd={hd} {shape}", simt=True)
    assert info["simt"] == 1 and info["grid"] == (N * nwy * nwx, heads)


@pytest.mark.parametrize("cls", ["peaked", "probe", "equal", "large"])
@pytest.mark.parametrize("ws,hd,heads", [(8, 32, 6), (8, 64, 4), (16, 32, 6), (16, 64, 4)])
def test_window_core_input_classes(ws, hd, heads, cls):
    """Peaked logits with the maximum at a window's first / last token and on both sides of the mask boundary, the
    bias / mask probe (q = 0, S = bias + mask exactly) on every window position of a shifted map, equal logits and
    large magnitudes, through the instance with all heads per CTA and one, and the SIMT kernel."""
    shift = 0 if cls == "equal" else ws // 2
    L = WindowCase(cls, 3, 3, 5, heads, ws, hd, shift, seed=ws + hd + len(cls))
    a, _ = L.check(f"window<{ws},{hd}> {cls} hpc=all", hpc=heads)
    b, _ = L.check(f"window<{ws},{hd}> {cls} hpc=1", hpc=1)
    assert torch.equal(a, b)
    L.check(f"window simt ws={ws} hd={hd} {cls}", simt=True)


@pytest.mark.parametrize("ws,hd,heads", [(8, 32, 6), (16, 64, 4)])
def test_window_core_launcher_rule_picks_several_heads(ws, hd, heads):
    """At a window count of at least 4 * SMs per head group the launcher itself puts all heads in one CTA."""
    per = math.ceil(4 * _sms() / 12)
    L = WindowCase("peaked", 4, 3, per, heads, ws, hd, ws // 2, seed=3)
    windows = 12 * per
    want = default_hpc(heads, windows)
    assert want > 1
    _, info = L.check(f"window<{ws},{hd}> launcher rule, {windows} windows", hpc=0)
    assert info["hpc"] == want and info["grid"] == (windows, heads // want), info
    RAN.add(("rule_hpc", f"window<{ws},{hd}>"))


def test_window_core_refusals():
    qkv = torch.zeros(1, 16, 16, 3 * 128, dtype=torch.float16, device="cuda")
    dense = torch.zeros(4 * 64 * 64, device="cuda")
    for hpc, simt, match in ((3, 0, "hpc must divide heads"), (-1, 0, "hpc must divide heads"), (2, 1, "SIMT")):
        rc = _lib.lib.rs_op_window_attention_cfg(qkv.data_ptr(), 1, 16, 16, 4, 8, 32, 0, dense.data_ptr(), qkv.data_ptr(),
                                                 hpc, simt, None, G.stream())
        assert rc != 0 and match.encode() in _lib.lib.rs_last_error(), (hpc, simt)


# ------------------------------------------------------------------------------------------------ fused Swin attention half

def _stats_pairs(x, slots):
    """(mean, M2) per (image, equal box of H*W / slots pixels in raster order, channel), float64 -> fp32."""
    N, H, W, E = x.shape
    xs = x.double().reshape(N, slots, H * W // slots, E)
    m = xs.mean(dim=2)
    return torch.stack([m, ((xs - m[:, :, None]) ** 2).sum(dim=2)], dim=-1).float().contiguous()


def _fp16_stage(v, allow):
    """fp16 store of a float64 value that carries an allowance: (rounded value, allowance of the stored value)."""
    r = v.half().double()
    return r, allow + G.ulp16(v.abs() + allow)


class SwinCase:
    def __init__(self, cls, N, H, W, E, shift, slots, seed):
        self.cls, self.N, self.H, self.W, self.E, self.shift, self.slots = cls, N, H, W, E, shift, slots
        self.heads = E // 32
        g = _gen(seed)
        if cls == "largemean":      # group means of +-30 with std 0.5
            sgn = torch.where(torch.rand(N, 1, 1, 32, 1, device="cuda", generator=g) < 0.5, -30.0, 30.0)
            x = torch.randn(N, H, W, 32, E // 32, device="cuda", generator=g) * 0.5 + sgn
            x = x.reshape(N, H, W, E)
        else:                       # each image its own scale and offset: an affine from another image is visible
            s = 1 + torch.rand(N, 1, 1, 1, device="cuda", generator=g)
            o = torch.rand(N, 1, 1, 1, device="cuda", generator=g) * 2 - 1
            x = torch.randn(N, H, W, E, device="cuda", generator=g) * s + o
        self.x = x.half()
        self.gamma = 1 + 0.2 * torch.randn(E, device="cuda", generator=g)
        self.beta = 0.2 * torch.randn(E, device="cuda", generator=g)
        wqkv = torch.randn(3 * E, E, device="cuda", generator=g) / E ** 0.5
        bqkv = torch.randn(3 * E, device="cuda", generator=g) * 0.1
        self.wproj = torch.randn(E, E, device="cuda", generator=g) / E ** 0.5 * 0.5
        self.bproj = torch.randn(E, device="cuda", generator=g) * 0.1
        if cls == "peaked":
            wqkv[:2 * E] *= 2.5
        elif cls in ("probe", "equal"):
            wqkv[:E] = 0
            bqkv[:E] = 0
        elif cls == "large":
            wqkv[:2 * E] *= 30
            bqkv[2 * E:] = 3e4 * (0.8 + 0.2 * torch.rand(E, device="cuda", generator=g)) * torch.sign(torch.randn(E, device="cuda", generator=g))
            wqkv[2 * E:] *= 10
            self.wproj *= 0.25
        self.wqkv, self.bqkv = wqkv, bqkv
        self.table = _table(cls, self.heads, 8, g)
        self.dense = torch.empty(self.heads * 64 * 64, dtype=torch.float32, device="cuda")
        _lib.check(G.L.rs_op_expand_relpos(self.table.data_ptr(), self.dense.data_ptr(), self.heads, G.stream()))
        self.part = _stats_pairs(self.x, slots)
        self.wq_p, _ = G.pack_weight(wqkv)
        self.wp_p, _ = G.pack_weight(self.wproj)
        self.nW = (H // 8) * (W // 8)
        self._reference()

    def _reference(self):
        N, H, W, E, heads = self.N, self.H, self.W, self.E, self.heads
        x = self.x.double()
        xg = x.reshape(N, H * W, 32, E // 32)
        mean = xg.mean(dim=(1, 3))
        std = xg.var(dim=(1, 3), unbiased=False).sqrt()
        rstd = 1 / (std ** 2 + 1e-5).sqrt()
        a = (rstd[:, :, None] * self.gamma.double().view(32, E // 32)).reshape(N, 1, 1, E)
        b = self.beta.double().view(1, 1, 1, E) - (mean[:, :, None].expand(N, 32, E // 32).reshape(N, 1, 1, E)) * a
        n1 = x * a + b
        em = (64 * 2.0 ** -24 * (mean.abs() + std))[:, :, None].expand(N, 32, E // 32).reshape(N, 1, 1, E)
        a1 = (x * a).abs() * 1024 * 2.0 ** -24 + a.abs() * em + 4 * 2.0 ** -24 * ((x * a).abs() + b.abs())
        n1, e1 = _fp16_stage(n1, a1)
        gE = (E + 2) * U32
        w = self.wqkv.half().double()
        qkv = n1 @ w.t() + self.bqkv.double()
        a2 = e1 @ w.abs().t() + gE * (n1.abs() @ w.abs().t() + self.bqkv.double().abs())
        qkv, e2 = _fp16_stage(qkv, a2)
        B = N * self.nW

        def heads_of(t):
            return to_windows(t, 8, self.shift).view(B, 64, 3, heads, 32).permute(2, 0, 3, 1, 4)
        x3, a3 = heads_of(qkv), heads_of(e2)
        r = softmax_ref(x3[0], x3[1], x3[2], 32 ** -0.5, window_bias(self.table, heads, 8, N, H, W, self.shift),
                        err=(a3[0], a3[1], a3[2]))
        kp, ks, s16 = kappas("swin", 64, 32, exact_p=self.cls == "equal")

        def pixels(t):
            return from_windows(t.permute(0, 2, 1, 3).reshape(B, 64, E), N, H, W, 8, self.shift)
        o, e3 = _fp16_stage(pixels(r["o"]), pixels(allowance(r, kp, ks, s16)))
        wp = self.wproj.half().double()
        self.ref = o @ wp.t() + self.bproj.double() + x
        self.allow = e3 @ wp.abs().t() + gE * (o.abs() @ wp.abs().t() + self.bproj.double().abs() + x.abs())

    def run(self, grid=0, inplace=False):
        N, H, W, E = self.N, self.H, self.W, self.E
        src = self.x.clone()
        y = src if inplace else torch.full_like(self.x, float("nan"))
        pout = torch.full((N, self.nW, E, 2), float("nan"), dtype=torch.float32, device="cuda")
        info = (C.c_int32 * 3)()
        _lib.check(G.L.rs_op_swin_attn_ex(src.data_ptr(), N, H, W, E, self.heads, self.shift, self.part.data_ptr(), self.slots,
                                          self.gamma.data_ptr(), self.beta.data_ptr(), self.wq_p.data_ptr(),
                                          self.bqkv.data_ptr(), self.dense.data_ptr(), self.wp_p.data_ptr(),
                                          self.bproj.data_ptr(), y.data_ptr(), pout.data_ptr(), grid, info, G.stream()))
        torch.cuda.synchronize()
        return y, pout, {"grid": info[0], "pairs_per_cta": info[1], "windows": info[2]}

    def check(self, tag, grid=0, inplace=False):
        y, pout, info = self.run(grid, inplace)
        assert info["windows"] == self.nW
        pairs = (self.N * self.nW + 1) // 2
        want_grid = grid or min(pairs, _sms())
        assert info["grid"] == want_grid and info["pairs_per_cta"] == -(-pairs // want_grid), info
        kernel = f"swin<{self.E}>"
        _note(kernel, self.cls, G.assert_within(tag, y, self.ref, self.allow, 1.0))
        self._check_pairs(tag, y, pout)
        RAN.add(("instance", kernel))
        RAN.add(("slots", self.slots))
        if info["pairs_per_cta"] >= 2:
            RAN.add(("swin", "several pairs per CTA"))
        if any((2 * p + 1) % self.nW == 0 for p in range(pairs) if 2 * p + 1 < self.N * self.nW):
            RAN.add(("swin", "pair straddles images"))
        return y, pout

    def _check_pairs(self, tag, y, pout):
        """The window (mean, M2) pairs against float64 statistics of the stored y over the shifted partition."""
        yw = to_windows(y.double(), 8, self.shift).view(self.N, self.nW, 64, self.E)
        m = yw.mean(dim=2)
        m2 = ((yw - m[:, :, None]) ** 2).sum(dim=2)
        sq = (yw * yw).sum(dim=2)
        got = pout.double()
        assert torch.isfinite(got).all(), f"{tag}: missing window pairs"
        dm = (got[..., 0] - m).abs() - 32 * 2.0 ** -24 * yw.abs().amax(dim=2)
        dq = (got[..., 1] - m2).abs() - 128 * 2.0 ** -24 * sq
        assert dm.max().item() <= 0 and dq.max().item() <= 0, f"{tag}: window pairs {dm.max().item():.3g} {dq.max().item():.3g}"


@pytest.mark.parametrize("E", [64, 192])
@pytest.mark.parametrize("shift", [0, 4])
@pytest.mark.parametrize("grid", [1, 2, 3, 7, 0])
def test_swin_forced_grids_odd_windows(grid, shift, E):
    """24x40 maps (15 windows per image) at N = 3: 23 pairs, so pairs straddle images and the last pair has one window;
    grids of 1, 2, 3 and 7 CTAs walk many pairs each.  In place equals out of place bit for bit, and runs repeat."""
    L = SwinCase("randn", 3, 24, 40, E, shift, 16, seed=E + shift + grid)
    y, pout = L.check(f"swin<{E}> shift={shift} grid={grid}", grid=grid)
    y2, pout2, _ = L.run(grid, inplace=True)
    assert torch.equal(G.bits(y), G.bits(y2)) and torch.equal(G.bits(pout), G.bits(pout2)), "in place differs"
    y3, pout3, _ = L.run(grid)
    assert torch.equal(G.bits(y), G.bits(y3)) and torch.equal(G.bits(pout), G.bits(pout3)), "two runs differ"


@pytest.mark.parametrize("E", [64, 192])
@pytest.mark.parametrize("cls", ["peaked", "probe", "equal", "large", "largemean"])
def test_swin_input_classes(cls, E):
    shift = 0 if cls == "equal" else 4
    L = SwinCase(cls, 3, 24, 40, E, shift, 15, seed=len(cls) * 7 + E)
    L.check(f"swin<{E}> {cls}", grid=3)
    L.check(f"swin<{E}> {cls} default grid")


# (slots, H, W): equal boxes of H*W / slots pixels
SLOT_MAPS = {1: (8, 8), 4: (16, 16), 15: (24, 40), 16: (24, 40), 17: (136, 8), 32: (24, 40), 128: (64, 64), 512: (64, 64)}


@pytest.mark.parametrize("cls", ["randn", "largemean"])
@pytest.mark.parametrize("slots", SLOTS)
def test_swin_norm1_slot_counts(slots, cls):
    H, W = SLOT_MAPS[slots]
    E = 192 if slots % 2 == 0 else 64
    L = SwinCase(cls, 3, H, W, E, 4 if H > 8 and W > 8 else 0, slots, seed=slots + len(cls))
    L.check(f"swin<{E}> {cls} slots={slots} {H}x{W}", grid=7 if 3 * L.nW >= 14 else 0)


def test_swin_refusals():
    L = SwinCase("randn", 1, 16, 16, 64, 0, 4, seed=1)
    for grid, match in ((3, "grid must be in"), (-1, "grid must be in")):
        with pytest.raises(_lib.RsError, match=match):
            L.run(grid)
    L.slots = 3
    with pytest.raises(_lib.RsError, match="slots must divide"):
        L.run(0)
    gst = torch.zeros(64, device="cuda")
    with pytest.raises(_lib.RsError, match="gstat_out and counters must be NULL"):
        _lib.check(G.L.rs_op_swin_attn(L.x.data_ptr(), 1, 16, 16, 64, 2, 0, L.part.data_ptr(), 4, L.gamma.data_ptr(),
                                       L.beta.data_ptr(), L.wq_p.data_ptr(), L.bqkv.data_ptr(), L.dense.data_ptr(),
                                       L.wp_p.data_ptr(), L.bproj.data_ptr(), L.x.data_ptr(), None, gst.data_ptr(), None,
                                       G.stream()))


# ------------------------------------------------------------------------------------------------ unet_attn

def _online_targets(T):
    """Per query row group (row % 3) the key it peaks on: in the first block, in the last (partial) block, and in a late
    block after the running maximum sat at +15 (a jump of 25)."""
    late = max(0, (T // 64 - 1) * 64) + 7 if T > 128 else T // 2
    return [min(5, T - 1), T - 1, min(late, T - 1)]


def _online_qkv(cls, N, heads, T, D, g):
    """q, k, v [N, heads, T, D] float32 of an input class for the online-softmax kernels."""
    scale = D ** -0.5
    q = torch.randn(N, heads, T, D, device="cuda", generator=g)
    k = torch.randn(N, heads, T, D, device="cuda", generator=g)
    v = torch.randn(N, heads, T, D, device="cuda", generator=g)
    if cls == "equal":
        q.zero_()
    elif cls == "peaked":
        a = 8.0
        b = 40.0 / (scale * a)
        grp = torch.arange(T, device="cuda") % 3
        q.zero_()
        q[..., torch.arange(T, device="cuda"), grp] = a
        k.zero_()
        k[..., :3] = b * (torch.rand(N, heads, T, 3, device="cuda", generator=g) * 1.375 - 1)
        for c, t in enumerate(_online_targets(T)):
            k[..., t, c] = b
    elif cls == "large":
        q, k, v = _qkv_class("large", N, T, heads, D, scale, g)
    assert q.shape == k.shape == v.shape == (N, heads, T, D)
    return q, k, v


def _row_chunk(batch, T):
    """Query rows per float64 reference chunk: about 2^27 scores at a time."""
    return max(64, min(1024, (1 << 27) // (batch * T)))


def unet_case(cls, N, T, heads, D, new_order, seed, tag=None):
    g = _gen(seed)
    q, k, v = (t.half() for t in _online_qkv(cls, N, heads, T, D, g))
    Cc = heads * D
    if new_order:
        qkv = torch.cat([t.permute(0, 2, 1, 3).reshape(N, T, Cc) for t in (q, k, v)], dim=-1)
    else:
        qkv = torch.stack([q, k, v], dim=3).permute(0, 2, 1, 3, 4).reshape(N, T, 3 * Cc)
    qkv = qkv.contiguous()
    out = torch.full((N, T, Cc), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(_lib.lib.rs_op_unet_attention(qkv.data_ptr(), N, T, heads, D, int(new_order), out.data_ptr(), G.stream()))
    torch.cuda.synchronize()
    kp, ks, s16 = kappas("unet", T, D, exact_p=cls == "equal")
    worst = 0.0
    step = _row_chunk(N * heads, T)
    for r0 in range(0, T, step):
        r1 = min(T, r0 + step)
        r = softmax_ref(q[:, :, r0:r1].double(), k.double(), v.double(), D ** -0.5)
        ref = r["o"].permute(0, 2, 1, 3).reshape(N, r1 - r0, Cc)
        a = allowance(r, kp, ks, s16).permute(0, 2, 1, 3).reshape(N, r1 - r0, Cc)
        worst = max(worst, G.assert_within(tag or f"unet<{D}> {cls} T={T} heads={heads} rows {r0}:{r1}", out[:, r0:r1], ref, a, 1.0))
    _note(f"unet<{D}>", cls, worst)
    RAN.add(("instance", f"unet<{D}>"))
    return out


UNET_T = [2, 127, 128, 129, 191, 193, 4095, 4097]


@pytest.mark.parametrize("T", UNET_T)
@pytest.mark.parametrize("D", [32, 64, 128])
def test_unet_attention_lengths(D, T):
    """The T on either side of the 64-key blocks and the 128-query CTAs that test_gpu_unetmodel.py's head-count matrix
    (T = 1, 15, 63, 64, 65, 1000, 4096, 16384) does not take; three heads, the head order alternating with T, N = 2."""
    unet_case("randn", 2, T, 3, D, UNET_T.index(T) % 2 == 1, seed=D * 1000 + T)


@pytest.mark.parametrize("cls", ["peaked", "equal", "large"])
@pytest.mark.parametrize("T", [63, 129, 4097])
@pytest.mark.parametrize("D", [32, 64, 128])
def test_unet_attention_input_classes(D, T, cls):
    unet_case(cls, 2, T, 3, D, T % 2 == 1, seed=D + T + len(cls))


# ------------------------------------------------------------------------------------------------ vq_attn

def vq_case(cls, N, T, Cc, seed, rows=None):
    g = _gen(seed)
    q, k, v = (t[:, 0].half().contiguous() for t in _online_qkv(cls, N, 1, T, Cc, g))
    out = torch.full((N, T, Cc), float("nan"), dtype=torch.float16, device="cuda")
    rb, re_ = rows or (0, T)
    _lib.check(_lib.lib.rs_op_vq_attention_rows(q.data_ptr(), k.data_ptr(), v.data_ptr(), N, T, Cc, Cc, rb, re_,
                                                out.data_ptr(), G.stream()))
    torch.cuda.synchronize()
    if rows:
        assert torch.isnan(out[:, :rb]).all() and torch.isnan(out[:, re_:]).all(), "rows outside the range written"
    vq_check(cls, q, k, v, out, rows)


def vq_check(cls, q, k, v, out, rows=None):
    """out [N, T, C] of the VQ-GAN attention on fp16 q, k, v [N, T, C] (any row stride) against float64, rows
    [rows[0], rows[1]), the query rows of a 1-D index tensor, or all.  Returns the worst ratio to the bound."""
    N, T, Cc = q.shape
    if torch.is_tensor(rows):
        sel = rows.to(q.device)
    else:
        rb, re_ = rows or (0, T)
        sel = torch.arange(rb, re_, device=q.device)
    kp, ks, s16 = kappas("vq", T, Cc, exact_p=cls == "equal")
    worst = 0.0
    step = _row_chunk(N, T)
    kd, vd = k.double(), v.double()
    for i in range(0, sel.numel(), step):
        r = sel[i:i + step]
        r0, r1 = r[0].item(), r[-1].item() + 1
        ref = softmax_ref(q[:, r].double(), kd, vd, Cc ** -0.5)
        worst = max(worst, G.assert_within(f"vq<{Cc}> {cls} T={T} rows {r0}:{r1}", out[:, r], ref["o"],
                                           allowance(ref, kp, ks, s16), 1.0))
    _note(f"vq<{Cc}>", cls, worst)
    RAN.add(("instance", f"vq<{Cc}>"))
    return worst


# randn at T = 64, 384, 4096, 16384 and 65536 is held by test_gpu_vq_attention.py::test_op_vs_fp32; equal and large
# logits at T <= 4096
VQ_CASES = [(c, t, cls) for c in (128, 256, 512) for t in (64, 128, 4096, 16384) for cls in ("randn", "peaked", "equal", "large")
            if (cls != "randn" or t == 128) and (t < 16384 or cls == "peaked")]


@pytest.mark.parametrize("Cc,T,cls", VQ_CASES, ids=[f"C{c}-T{t}-{cls}" for c, t, cls in VQ_CASES])
def test_vq_attention(Cc, T, cls):
    vq_case(cls, 2, T, Cc, seed=Cc + T + len(cls))


def test_vq_attention_row_range():
    vq_case("peaked", 2, 4096, 256, seed=5, rows=(64, 1216))
    RAN.add(("vq", "rows"))


# ------------------------------------------------------------------------------------------------ plan replay

_ATTN = re.compile(r"attn (\d+)x(\d+) window=(\d+) shift=(\d+) N=(\d+) heads=(\d+) head_dim=(\d+) hpc=(\d+) simt=(\d)")
_SWIN = re.compile(r"swin_attn (\d+)x(\d+) shift=(\d+) grid=(\d+) N=(\d+) E=(\d+) heads=(\d+) slots=(\d+)")
_UNET = re.compile(r"unet_attn T=(\d+) heads=(\d+) D=(\d+) N=(\d+) order=(\w+)")
_VQ = re.compile(r"vq_attn T=(\d+) C=(\d+) N=(\d+)")


def _windows_rows(name, B, H, W):
    from oracle.make_golden_variants import variant_inputs
    from oracle.make_golden_windows import windows_config
    from resshift_b200.models.unet import UNetModelSwin
    from resshift_b200.weights import random_state_dict
    from tests.test_gpu_conv_instances import _desc_rows
    ucfg, _ = windows_config(name)
    m = UNetModelSwin(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 0), strict=True)
    m = m.cuda().eval()
    x, lq, _ = (None if t is None else t.cuda() for t in variant_inputs(ucfg, B, H, W, 6))
    t = torch.full((B,), 3.0, device="cuda")
    m(x, t, lq=lq)
    return _desc_rows(_lib.lib.rs_plan_profile_ops, m.plan(B, H, W).handle, x.data_ptr(), t.data_ptr(), lq.data_ptr(), None)


def _unetmodel_rows(name, H, W):
    from oracle.make_golden_unetmodel import case_config, case_inputs
    from resshift_b200.models.unet import UNetModel
    from resshift_b200.weights import random_state_dict
    from tests.test_gpu_conv_instances import _desc_rows
    ucfg, _, _ = case_config(name)
    m = UNetModel(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 0), strict=True)
    m = m.cuda().eval()
    x, lq = (t.cuda() for t in case_inputs(ucfg, 3, H, W, 5))
    t = torch.tensor([3.0, 1.0, 0.0], device="cuda")
    m(x, t, lq=lq)
    return _desc_rows(_lib.lib.rs_plan_profile_ops, m.plan(3, H, W).handle, x.data_ptr(), t.data_ptr(), lq.data_ptr(), None)


def _plans():
    from oracle.make_golden_unetmodel import CASES
    from tests import test_gpu_conv_instances as T
    plans = {"realsr_denoiser_b16_64x64": T.PLANS["realsr_denoiser_b16_64x64"]}
    for name in ("w16_h32", "w8_h64", "w16_h64"):
        for hw in (64, 128):
            plans[f"{name}_b16_{hw}x{hw}"] = (lambda n=name, s=hw: _windows_rows(n, 16, s, s))
    plans["w16_h64_variant_b16_64x64"] = lambda: _windows_rows("w16_h64_variant", 16, 64, 64)
    for name in CASES:
        plans[f"unetmodel_{name}_b3"] = (lambda n=name: _unetmodel_rows(n, *CASES[n][1:]))
    plans["unetmodel_legacy_b3_64x128"] = lambda: _unetmodel_rows("legacy", 64, 128)
    plans["vq_f4_encode_1024"] = lambda: T._first_stage_rows("vq", "f4", 0, 1, 1024, 1024)
    return plans


def _plan_names():
    from oracle.make_golden_unetmodel import CASES
    return (["realsr_denoiser_b16_64x64"] + [f"{n}_b16_{s}x{s}" for n in ("w16_h32", "w8_h64", "w16_h64") for s in (64, 128)] +
            ["w16_h64_variant_b16_64x64"] + [f"unetmodel_{n}_b3" for n in CASES] +
            ["unetmodel_legacy_b3_64x128", "vq_f4_encode_1024"])


def _distinct(rows, rx):
    return sorted({tuple(rx.match(r).groups()) for r in rows if rx.match(r)})


@pytest.mark.parametrize("plan", _plan_names() if torch.cuda.is_available() else [])
def test_plan_attention(plan):
    """Each distinct attention of a shipped plan (random weights) replayed through the entries with the plan's
    configuration, on randn and peaked operands: the entry reports the plan's heads per CTA or persistent grid, and the
    result is within the float64 bound."""
    rows = _plans()[plan]()
    attn, swin = _distinct(rows, _ATTN), _distinct(rows, _SWIN)
    unet, vq = _distinct(rows, _UNET), _distinct(rows, _VQ)
    print(f"[plan] {plan}: {len(attn)} window, {len(swin)} fused Swin, {len(unet)} unet, {len(vq)} vq attentions")
    assert attn or swin or unet or vq
    for i, d in enumerate(attn):
        H, W, ws, shift, N, heads, hd, hpc, simt = map(int, d)
        assert not simt
        for cls in ("randn", "peaked"):
            L = WindowCase(cls, N, H // ws, W // ws, heads, ws, hd, shift, seed=i)
            _, info = L.check(f"{plan} attn {d} {cls}", hpc=0)
            assert info["hpc"] == hpc, (d, info)
    for i, d in enumerate(swin):
        H, W, shift, grid, N, E, heads, slots = map(int, d)
        for cls in ("randn", "peaked"):
            L = SwinCase(cls, N, H, W, E, shift, slots, seed=i)
            y, pout, info = L.run(0)
            assert info["grid"] == grid, (d, info)
            L.check(f"{plan} swin_attn {d} {cls}")
    for i, d in enumerate(unet):
        T, heads, D, N = map(int, d[:4])
        for cls in ("randn", "peaked"):
            unet_case(cls, N, T, heads, D, d[4] == "new", seed=i, tag=f"{plan} unet_attn {d} {cls}")
    for i, d in enumerate(vq):
        T, Cc, N = map(int, d)
        for cls in ("randn", "peaked"):
            vq_case(cls, N, T, Cc, seed=i)
    RAN.add(("plan", plan))


# ------------------------------------------------------------------------------------------------ coverage

def test_coverage():
    """Across the module (run it whole): every instance ran, each with every input class it takes; heads per CTA of 1,
    a proper divisor and all heads; a CTA with several window pairs and a pair straddling images; every norm1 slot
    count.  Prints the worst observed ratio of error to allowance per kernel and input class."""
    if not RAN:
        pytest.skip("run with the rest of the module")
    for (kernel, cls), r in sorted(OBS.items()):
        print(f"[observed] {kernel:14s} {cls:10s} worst ratio {r:.3g}")
    kernels = [f"window<{ws},{hd}>" for ws, hd in INSTANCES] + ["window_simt", "swin<64>", "swin<192>", "unet<32>", "unet<64>",
                                                                 "unet<128>", "vq<128>", "vq<256>", "vq<512>"]
    missing = [k for k in kernels if ("instance", k) not in RAN]
    assert not missing, missing
    want = {k: (CLASSES if k.startswith("window") else ("randn", "peaked", "equal", "large")) for k in kernels}
    for k in ("swin<64>", "swin<192>"):
        want[k] = CLASSES + ("largemean",)
    gaps = [(k, c) for k, cs in want.items() for c in cs if ("class", k, c) not in RAN]
    assert not gaps, gaps
    gaps = [(ws, hd, h) for ws, hd in INSTANCES for h in ("1", "divisor", "all") if ("hpc", f"window<{ws},{hd}>", h) not in RAN]
    assert not gaps, gaps
    assert ("swin", "several pairs per CTA") in RAN and ("swin", "pair straddles images") in RAN
    assert {("slots", s) for s in SLOTS} <= RAN
