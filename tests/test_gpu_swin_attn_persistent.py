"""Fused Swin attention half (rs_op_swin_attn) on shapes the per-operator test does not reach: an odd window count split
over several persistent window pairs per CTA (more pairs than SMs, the last pair's second window empty), at E = 64 and
E = 192, and the in-place form (y == x) the denoiser runs, which must equal the out-of-place result bit for bit.
reference: models/swin_transformer.py:246-275,114-145, with the intermediate fp16 roundings of the unfused path."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from tests import gpu_util as G
    from resshift_b200 import _lib


def _reference(x, gamma, beta, wqkv, bqkv, table, wproj, bproj, heads, shift):
    from resshift_b200.arch import relative_position_index, shifted_window_mask
    N, H, W, E = x.shape
    xc = x.float().cpu()
    xn = F.group_norm(xc.permute(0, 3, 1, 2), 32, gamma.cpu(), beta.cpu(), eps=1e-5).half().float()
    qkv = F.conv2d(xn, wqkv.half().float().cpu()[:, :, None, None], bqkv.cpu()).half().float()
    if shift:
        qkv = torch.roll(qkv, (-shift, -shift), (2, 3))
    yw = qkv.reshape(N, 3 * E, H // 8, 8, W // 8, 8).permute(0, 2, 4, 3, 5, 1).reshape(-1, 64, 3, heads, 32)
    qq, kk, vv = (yw[:, :, i].transpose(1, 2) for i in range(3))
    attn = (qq * 32 ** -0.5) @ kk.transpose(-2, -1)
    attn = attn + table.cpu()[relative_position_index(8).reshape(-1)].view(64, 64, heads).permute(2, 0, 1)[None]
    if shift:
        m = shifted_window_mask(H, W, 8, shift)
        attn = (attn.view(-1, m.shape[0], heads, 64, 64) + m[None, :, None]).view(-1, heads, 64, 64)
    o = (attn.softmax(-1) @ vv).transpose(1, 2).reshape(-1, 64, E)
    o = o.view(N, H // 8, W // 8, 8, 8, E).permute(0, 5, 1, 3, 2, 4).reshape(N, E, H, W)
    if shift:
        o = torch.roll(o, (shift, shift), (2, 3))
    o = o.half().float()
    return (F.conv2d(o, wproj.half().float().cpu()[:, :, None, None], bproj.cpu()) + xc.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)


# (N, H, W, shift): 301 and 31 x 9 windows are odd and give 151 / 140 pairs, more than the SMs of an H100 SXM
@pytest.mark.parametrize("E", [64, 192])
@pytest.mark.parametrize("case", [(301, 8, 8, 0), (31, 24, 24, 4)])
def test_swin_attention_half_odd_windows_persistent(case, E):
    N, H, W, shift = case
    heads = E // 32
    g = torch.Generator(device="cuda").manual_seed(N + H + E + shift)
    x = (torch.randn(N, H, W, E, device="cuda", generator=g) * 1.5 + 0.3).half()
    gamma = 1 + 0.2 * torch.randn(E, device="cuda", generator=g)
    beta = 0.2 * torch.randn(E, device="cuda", generator=g)
    wqkv = torch.randn(3 * E, E, device="cuda", generator=g) / E ** 0.5
    bqkv = torch.randn(3 * E, device="cuda", generator=g) * 0.1
    wproj = torch.randn(E, E, device="cuda", generator=g) / E ** 0.5 * 0.5
    bproj = torch.randn(E, device="cuda", generator=g) * 0.1
    table = torch.randn(225, heads, device="cuda", generator=g) * 0.5
    dense = torch.empty(heads * 64 * 64, dtype=torch.float32, device="cuda")
    _lib.check(G.L.rs_op_expand_relpos(table.data_ptr(), dense.data_ptr(), heads, G.stream()))
    rows = 128 if H * W % 128 == 0 else 64
    slots = H * W // rows
    xs = x.float().reshape(N, slots, rows, E)
    mean_s = xs.mean(dim=2)
    part = torch.stack([mean_s, ((xs - mean_s[:, :, None]) ** 2).sum(dim=2)], dim=-1).contiguous()
    wq_p, _ = G.pack_weight(wqkv)
    wp_p, _ = G.pack_weight(wproj)
    nW = (H // 8) * (W // 8)
    assert (N * nW) % 2 == 1 and (N * nW + 1) // 2 > torch.cuda.get_device_properties(0).multi_processor_count

    def run(src, dst):
        pout = torch.full((N, nW, E, 2), float("nan"), dtype=torch.float32, device="cuda")
        _lib.check(G.L.rs_op_swin_attn(src.data_ptr(), N, H, W, E, heads, shift, part.data_ptr(), slots, gamma.data_ptr(),
                                       beta.data_ptr(), wq_p.data_ptr(), bqkv.data_ptr(), dense.data_ptr(), wp_p.data_ptr(),
                                       bproj.data_ptr(), dst.data_ptr(), pout.data_ptr(), None, None, G.stream()))
        torch.cuda.synchronize()
        return pout

    y = torch.full_like(x, float("nan"))
    pout = run(x, y)
    xin = x.clone()
    pout_in = run(xin, xin)
    assert torch.equal(xin, y) and torch.equal(pout_in, pout)

    ref = _reference(x, gamma, beta, wqkv, bqkv, table, wproj, bproj, heads, shift)
    st = G.err_stats(y.cpu(), ref)
    assert st["nan"] == 0 and st["max_abs"] <= 4e-3 * ref.abs().max().item() + 4e-3, st
    yy = y.float().cpu().permute(0, 3, 1, 2)
    if shift:
        yy = torch.roll(yy, (-shift, -shift), (2, 3))
    ywin = yy.reshape(N, E, H // 8, 8, W // 8, 8).permute(0, 2, 4, 1, 3, 5).reshape(N, nW, E, 64)
    m_ref = ywin.mean(dim=3)
    q_ref = ((ywin - m_ref[..., None]) ** 2).sum(dim=3)
    assert not torch.isnan(pout).any()
    assert (pout[..., 0].cpu() - m_ref).abs().max().item() <= 1e-4 * (1 + m_ref.abs().max().item())
    assert ((pout[..., 1].cpu() - q_ref).abs() / (q_ref + 1e-3)).max().item() <= 2e-3
