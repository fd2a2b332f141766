"""The fused Swin MLP at the benchmark denoiser's own shapes: batch 16, E = 192, hidden 768, at each Swin level
(64x64, 32x32, 16x16 and 8x8), against the float64 bound of test_gpu_mlp_instances.py, with two statistics sinks and
two launches bit-identical.  The maps there have at most 32 tiles; these run up to 512 tiles per launch, with the
residual in place as the Swin block runs it."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from tests import gpu_util as G
    from tests.mlp_ref import KAPPA, reference
    from resshift_b200 import _lib

LEVELS = (64, 32, 16, 8)


@pytest.mark.parametrize("hw", LEVELS, ids=[f"{h}x{h}" for h in LEVELS])
def test_fused_mlp_benchmark_levels(hw):
    N, E, Hd = 16, 192, 768
    g = torch.Generator(device="cuda").manual_seed(hw)
    x = (torch.randn(N, hw, hw, E, device="cuda", generator=g) * 1.5 + 0.3).half()
    res = torch.randn(N, hw, hw, E, device="cuda", generator=g).half()
    w1 = torch.randn(Hd, E, device="cuda", generator=g) / E ** 0.5
    b1 = torch.randn(Hd, device="cuda", generator=g) * 0.5
    w2 = torch.randn(E, Hd, device="cuda", generator=g) / Hd ** 0.5
    b2 = torch.randn(E, device="cuda", generator=g) * 0.5
    w1p, _ = G.pack_weight(w1)
    w2p, _ = G.pack_weight(w2)
    slots = G.box128(hw, hw)[3]
    # two sinks with different channel strides and offsets, as test_fused_mlp_vs_float64 gives them
    specs = [(E + 8, 0), (E + 40, 8)]

    def launch():
        y = res.clone()                                   # in place: out == res
        sk = [torch.full((N * slots * cs * 2 + 64,), float("nan"), device="cuda") for cs, _ in specs]
        parts = (C.c_void_p * 2)(*[s.data_ptr() for s in sk])
        cst = (C.c_int32 * 2)(*[cs for cs, _ in specs])
        cof = (C.c_int32 * 2)(*[co for _, co in specs])
        nslots = C.c_int32()
        _lib.check(_lib.lib.rs_op_mlp_ex(x.data_ptr(), N, hw, hw, E, Hd, w1p.data_ptr(), b1.data_ptr(), w2p.data_ptr(),
                                         b2.data_ptr(), y.data_ptr(), y.data_ptr(), parts, cst, cof, C.byref(nslots),
                                         G.stream()))
        torch.cuda.synchronize()
        assert nslots.value == slots
        return y, sk

    out, sk = launch()
    out2, sk2 = launch()
    assert torch.equal(G.bits(out), G.bits(out2))
    assert all(torch.equal(G.bits(a), G.bits(b)) for a, b in zip(sk, sk2))
    ref, mag, slack = reference(x.reshape(-1, E), res.reshape(-1, E), w1, b1, w2, b2)
    G.assert_within(f"mlp b16 {hw}x{hw}", out.reshape(-1, E), ref, mag, KAPPA, slack=slack)
    for i, (part, (cs, co)) in enumerate(zip(sk, specs)):
        G.check_slot_pairs(f"mlp b16 {hw}x{hw} sink {i}", part, out, cs, co)
