"""Fused Swin attention half (rs_op_swin_attn_ex) on shapes the per-operator test does not reach: an odd window count
split over several persistent window pairs per CTA (more pairs than SMs, the last pair's second window empty), at E = 64
and E = 192, and the in-place form (y == x) the denoiser runs, which must equal the out-of-place result bit for bit.
Per element against the float64 reference of tests/test_gpu_attention.py (models/swin_transformer.py:246-275,114-145,
with the intermediate fp16 roundings of the unfused path)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from tests import gpu_util as G


# (N, H, W, shift): 301 and 31 x 9 windows are odd and give 151 / 140 pairs, more than the SMs of an H100 SXM
@pytest.mark.parametrize("E", [64, 192])
@pytest.mark.parametrize("case", [(301, 8, 8, 0), (31, 24, 24, 4)])
def test_swin_attention_half_odd_windows_persistent(case, E):
    from tests.attn_ref import SwinCase
    N, H, W, shift = case
    slots = H * W // (128 if H * W % 128 == 0 else 64)
    L = SwinCase("randn", N, H, W, E, shift, slots, seed=N + H + E + shift)
    nW = (H // 8) * (W // 8)
    assert (N * nW) % 2 == 1 and (N * nW + 1) // 2 > torch.cuda.get_device_properties(0).multi_processor_count
    y, pout, _, _ = L.check(f"swin attn persistent E={E} {case}")
    yi, pout_in, _ = L.run(inplace=True)
    assert torch.equal(G.bits(yi), G.bits(y)) and torch.equal(G.bits(pout_in), G.bits(pout))
