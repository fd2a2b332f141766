"""The attention kernels as the GPU tests drive them (window attention, the fused Swin attention half, unet_attn and
vq_attn), their float64 references and the per-element bound of test_gpu_attention.py's module docstring.  Each check
returns the worst ratio of error to bound it met."""
import ctypes as C
import math

import torch

from resshift_b200 import _lib
from resshift_b200.arch import relative_position_index, shifted_window_mask
from tests import gpu_util as G

U16, U32, S16 = 2.0 ** -11, 2.0 ** -23, 2.0 ** -25
EX2 = 2.0 ** -22


def sms():
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


def bias_table(cls, heads, ws, g):
    n = (2 * ws - 1) ** 2
    if cls == "equal":
        return torch.zeros(n, heads, device="cuda")
    if cls == "probe":      # distinct entries spanning +-6: a transposed or shifted gather moves every weight
        perm = torch.randperm(n * heads, device="cuda", generator=g).float()
        return (perm / (n * heads - 1) * 12 - 6).view(n, heads)
    return torch.randn(n, heads, device="cuda", generator=g) * 0.5


def qkv_class(cls, B, T, heads, D, scale, g, targets=None):
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




class WindowCase:
    def __init__(self, cls, N, nwy, nwx, heads, ws, hd, shift, seed):
        self.cls, self.N, self.H, self.W, self.heads, self.ws, self.hd, self.shift = cls, N, nwy * ws, nwx * ws, heads, ws, hd, shift
        g = G.gen(seed)
        T, B = ws * ws, N * nwy * nwx
        scale = hd ** -0.5
        # peaked: the target key of a window at its first or last token, or either side of the mask's label boundary
        # (columns ws - shift - 1 and ws - shift of the last token row)
        s = ws // 2
        choices = torch.tensor([0, T - 1, (ws - 1) * ws + ws - s - 1, (ws - 1) * ws + ws - s], device="cuda")
        targets = choices[torch.arange(B, device="cuda") % 4]
        q, k, v = qkv_class(cls, B, T, heads, hd, scale, g, targets)
        w = torch.stack([q, k, v], 1).permute(0, 3, 1, 2, 4).reshape(B, T, 3 * heads * hd)
        self.qkv = from_windows(w, N, self.H, self.W, ws, shift).half().contiguous()
        self.table = bias_table(cls, heads, ws, g)
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
        return out, info, G.assert_within(tag, out, self.ref, a, 1.0)




def stats_pairs(x, slots):
    """(mean, M2) per (image, equal box of H*W / slots pixels in raster order, channel), float64 -> fp32."""
    N, H, W, E = x.shape
    xs = x.double().reshape(N, slots, H * W // slots, E)
    m = xs.mean(dim=2)
    return torch.stack([m, ((xs - m[:, :, None]) ** 2).sum(dim=2)], dim=-1).float().contiguous()


def fp16_stage(v, allow):
    """fp16 store of a float64 value that carries an allowance: (rounded value, allowance of the stored value)."""
    r = v.half().double()
    return r, allow + G.ulp16(v.abs() + allow)


class SwinCase:
    def __init__(self, cls, N, H, W, E, shift, slots, seed):
        self.cls, self.N, self.H, self.W, self.E, self.shift, self.slots = cls, N, H, W, E, shift, slots
        self.heads = E // 32
        g = G.gen(seed)
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
        self.table = bias_table(cls, self.heads, 8, g)
        self.dense = torch.empty(self.heads * 64 * 64, dtype=torch.float32, device="cuda")
        _lib.check(G.L.rs_op_expand_relpos(self.table.data_ptr(), self.dense.data_ptr(), self.heads, G.stream()))
        self.part = stats_pairs(self.x, slots)
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
        n1, e1 = fp16_stage(n1, a1)
        gE = (E + 2) * U32
        w = self.wqkv.half().double()
        qkv = n1 @ w.t() + self.bqkv.double()
        a2 = e1 @ w.abs().t() + gE * (n1.abs() @ w.abs().t() + self.bqkv.double().abs())
        qkv, e2 = fp16_stage(qkv, a2)
        B = N * self.nW

        def heads_of(t):
            return to_windows(t, 8, self.shift).view(B, 64, 3, heads, 32).permute(2, 0, 3, 1, 4)
        x3, a3 = heads_of(qkv), heads_of(e2)
        r = softmax_ref(x3[0], x3[1], x3[2], 32 ** -0.5, window_bias(self.table, heads, 8, N, H, W, self.shift),
                        err=(a3[0], a3[1], a3[2]))
        kp, ks, s16 = kappas("swin", 64, 32, exact_p=self.cls == "equal")

        def pixels(t):
            return from_windows(t.permute(0, 2, 1, 3).reshape(B, 64, E), N, H, W, 8, self.shift)
        o, e3 = fp16_stage(pixels(r["o"]), pixels(allowance(r, kp, ks, s16)))
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
        want_grid = grid or min(pairs, sms())
        assert info["grid"] == want_grid and info["pairs_per_cta"] == -(-pairs // want_grid), info
        ratio = G.assert_within(tag, y, self.ref, self.allow, 1.0)
        self._check_pairs(tag, y, pout)
        return y, pout, info, ratio

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




def online_targets(T):
    """Per query row group (row % 3) the key it peaks on: in the first block, in the last (partial) block, and in a late
    block after the running maximum sat at +15 (a jump of 25)."""
    late = max(0, (T // 64 - 1) * 64) + 7 if T > 128 else T // 2
    return [min(5, T - 1), T - 1, min(late, T - 1)]


def online_qkv(cls, N, heads, T, D, g):
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
        for c, t in enumerate(online_targets(T)):
            k[..., t, c] = b
    elif cls == "large":
        q, k, v = qkv_class("large", N, T, heads, D, scale, g)
    assert q.shape == k.shape == v.shape == (N, heads, T, D)
    return q, k, v


def row_chunk(batch, T):
    """Query rows per float64 reference chunk: about 2^27 scores at a time."""
    return max(64, min(1024, (1 << 27) // (batch * T)))


def unet_case(cls, N, T, heads, D, new_order, seed, tag=None):
    g = G.gen(seed)
    q, k, v = (t.half() for t in online_qkv(cls, N, heads, T, D, g))
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
    step = row_chunk(N * heads, T)
    for r0 in range(0, T, step):
        r1 = min(T, r0 + step)
        r = softmax_ref(q[:, :, r0:r1].double(), k.double(), v.double(), D ** -0.5)
        ref = r["o"].permute(0, 2, 1, 3).reshape(N, r1 - r0, Cc)
        a = allowance(r, kp, ks, s16).permute(0, 2, 1, 3).reshape(N, r1 - r0, Cc)
        worst = max(worst, G.assert_within(tag or f"unet<{D}> {cls} T={T} heads={heads} rows {r0}:{r1}", out[:, r0:r1], ref, a, 1.0))
    return out, worst




def vq_case(cls, N, T, Cc, seed, rows=None):
    g = G.gen(seed)
    q, k, v = (t[:, 0].half().contiguous() for t in online_qkv(cls, N, 1, T, Cc, g))
    out = torch.full((N, T, Cc), float("nan"), dtype=torch.float16, device="cuda")
    rb, re_ = rows or (0, T)
    _lib.check(_lib.lib.rs_op_vq_attention_rows(q.data_ptr(), k.data_ptr(), v.data_ptr(), N, T, Cc, Cc, rb, re_,
                                                out.data_ptr(), G.stream()))
    torch.cuda.synchronize()
    if rows:
        assert torch.isnan(out[:, :rb]).all() and torch.isnan(out[:, re_:]).all(), "rows outside the range written"
    return vq_check(cls, q, k, v, out, rows)


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
    step = row_chunk(N, T)
    kd, vd = k.double(), v.double()
    for i in range(0, sel.numel(), step):
        r = sel[i:i + step]
        r0, r1 = r[0].item(), r[-1].item() + 1
        ref = softmax_ref(q[:, r].double(), kd, vd, Cc ** -0.5)
        worst = max(worst, G.assert_within(f"vq<{Cc}> {cls} T={T} rows {r0}:{r1}", out[:, r], ref["o"],
                                           allowance(ref, kp, ks, s16), 1.0))
    return worst


