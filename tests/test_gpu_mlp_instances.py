"""The fused Swin MLP (mlp_fused_sm90_kernel<E>, E in {64, 128, 192, 256}) through rs_op_mlp_ex against float64, the
two model-level paths around it (the <256> instance inside a plan, and the unfused fc1 / fc2 fallback of E = 96).  Its
input is either a raw tensor or the output of the GroupNorm apply that runs in front of it (the Swin block's norm2).

The reference is float64 with the kernel's fp16 roundings: of the (normalised) input X, of the hidden activations
H = fp16(GELU(X W1^T + b1)), and of the output fp16(res + b2 + H W2^T).  Per element
|got - ref| <= 1/2 ulp16(ref) + KAPPA * mag2 + slack, with mag2 = |H| |W2|^T + |b2| + |res| and slack = sum_j |W2_ij| e_j
over the hidden values whose float64 value lies so close to an fp16 rounding boundary (closer than the first GEMM's
allowance KAPPA * (|X| |W1|^T + |b1|) x 1.13) that the kernel may have rounded it to the neighbour (e_j = that spacing)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from tests import gpu_util as G
    from tests import plan_ops
    from tests.mlp_ref import KAPPA, mlp, reference
    from resshift_b200 import _lib

# (N, H, W): 8x8 with an odd batch (two images per 128-pixel tile, the second tile half padding), 16x16, 64x64, 32x64
MAPS = {"8x8_n3": (3, 8, 8), "16x16_n2": (2, 16, 16), "64x64_n1": (1, 64, 64), "32x64_n2": (2, 32, 64)}
# input: "none" = the random tensor as is; "gstat" / "pairs" = that tensor normalised by the separate GroupNorm apply the
# Swin block runs in front of the MLP (norm2), from finalised group statistics or from the producers' per-slot pairs
CASES = [(E, r, m, src) for E in (64, 128, 192, 256) for r in (4, 2) for m in MAPS
         for src in (("none", "gstat", "pairs") if r == 4 else ("none",))]


def _group_stats(x, N):
    """float64 per-(image, group) mean and rstd of fp16 x [N, H, W, E] (GroupNorm32, eps 1e-5)."""
    xg = x.double().reshape(N, -1, 32, x.shape[-1] // 32).permute(0, 2, 1, 3).reshape(N, 32, -1)
    mean = xg.mean(dim=2)
    return mean, (xg.var(dim=2, unbiased=False) + 1e-5).rsqrt()


def _slot_pairs(x, bw, bh, slots):
    """(mean, M2) pairs [N][slots][E][2] of x per tile slot, what a producing kernel delivers."""
    N, H, W, E = x.shape
    t = x.float().reshape(N, H // bh, bh, W // bw, bw, E).permute(0, 1, 3, 2, 4, 5).reshape(N, slots, bh * bw, E)
    m = t.mean(dim=2)
    return torch.stack([m, ((t - m[:, :, None]) ** 2).sum(dim=2)], dim=-1).contiguous()


@pytest.mark.parametrize("E,ratio,map_,src", CASES, ids=[f"E{e}-Hd{r}E-{m}-{n}" for e, r, m, n in CASES])
def test_fused_mlp_vs_float64(E, ratio, map_, src):
    """Output against float64, output statistics sinks per slot, two launches bit-identical; with a normalised input, the
    GroupNorm apply (rs_op_groupnorm_apply / _apply_pairs) that produced it against float64 GroupNorm32 as well."""
    N, H, W = MAPS[map_]
    Hd = ratio * E
    seed = E * 7 + ratio * 3 + H + W + len(src)
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(N, H, W, E, device="cuda", generator=g) * 1.5 + 0.3).half()
    res = torch.randn(N, H, W, E, device="cuda", generator=g).half()
    w1 = torch.randn(Hd, E, device="cuda", generator=g) / E ** 0.5
    b1 = torch.randn(Hd, device="cuda", generator=g) * 0.5
    w2 = torch.randn(E, Hd, device="cuda", generator=g) / Hd ** 0.5
    b2 = torch.randn(E, device="cuda", generator=g) * 0.5
    gamma = 1 + 0.2 * torch.randn(E, device="cuda", generator=g)
    beta = 0.2 * torch.randn(E, device="cuda", generator=g)
    w1p, _ = G.pack_weight(w1)
    w2p, _ = G.pack_weight(w2)
    bw, bh, _, slots = G.box128(H, W)
    n_sinks = CASES.index((E, ratio, map_, src)) % 3
    xin = x
    if src != "none":
        mean, rstd = _group_stats(x, N)
        xin = torch.full_like(x, float("nan"))
        if src == "gstat":
            gst = torch.stack([mean, rstd], dim=-1).float().contiguous()
            _lib.check(_lib.lib.rs_op_groupnorm_apply(x.data_ptr(), N, H, W, E, E, gamma.data_ptr(), beta.data_ptr(), None, 0, 0,
                                                      xin.data_ptr(), E, gst.data_ptr(), G.stream()))
        else:
            pairs = _slot_pairs(x, bw, bh, slots)
            _lib.check(_lib.lib.rs_op_groupnorm_apply_pairs(x.data_ptr(), N, H, W, E, E, gamma.data_ptr(), beta.data_ptr(), None, 0,
                                                            0, xin.data_ptr(), E, pairs.data_ptr(), slots, G.stream()))
        torch.cuda.synchronize()
        # the normalisation itself, against float64 GroupNorm32 (fp32 arithmetic, one fp16 rounding)
        xn = (x.double().reshape(N, -1, 32, E // 32) - mean[:, None, :, None]) * rstd[:, None, :, None]
        xn = xn.reshape(N, H, W, E) * gamma.double() + beta.double()
        mag = (x.double().reshape(N, -1, 32, E // 32) * rstd[:, None, :, None]).reshape(N, H, W, E).abs() * gamma.double().abs()
        G.assert_within(f"norm2 {src}", xin, xn, mag + xn.abs(), 2.0 ** -16)

    def sinks():
        return [(torch.full((N * slots * (E + 32 * i + 8) * 2 + 64,), float("nan"), device="cuda"), E + 32 * i + 8, 8 * i)
                for i in range(n_sinks)]
    runs = []
    for _ in range(2):
        sk = sinks()
        out, nslots = mlp(xin, res, w1p, b1, w2p, b2, E, Hd, sinks=sk)
        runs.append((out, sk))
    assert nslots == slots
    (out, sk), (out2, sk2) = runs
    assert torch.equal(G.bits(out), G.bits(out2))
    assert all(torch.equal(G.bits(a[0]), G.bits(b[0])) for a, b in zip(sk, sk2))
    ref, mag, slack = reference(xin.reshape(-1, E), res.reshape(-1, E), w1, b1, w2, b2)
    G.assert_within(f"mlp E={E} Hd={Hd} {map_} {src}", out.reshape(-1, E), ref, mag, KAPPA, slack=slack)
    for i, (part, cstride, coff) in enumerate(sk):
        G.check_slot_pairs(f"mlp sink {i}", part, out, cstride, coff)


def test_mlp_refusals():
    """Widths without an instance and hidden sizes that are not whole 64-column chunks are refused."""
    g = torch.Generator(device="cuda").manual_seed(1)

    def attempt(E, Hd):
        x = torch.randn(2, 16, 16, E, device="cuda", generator=g).half()
        w1p, _ = G.pack_weight(torch.randn(Hd, E, device="cuda", generator=g))
        w2p, _ = G.pack_weight(torch.randn(E, Hd, device="cuda", generator=g))
        b1, b2 = torch.zeros(Hd, device="cuda"), torch.zeros(E, device="cuda")
        with pytest.raises(_lib.RsError, match="fused MLP"):
            mlp(x, None, w1p, b1, w2p, b2, E, Hd)
    attempt(96, 384)
    attempt(64, 4 * 64 + 32)


# ---------------------------------------------------------------------------------------------- model level

def _unet_vs_oracle(ucfg, expect_mlp_e):
    from oracle import unet_variants_oracle as uo
    from resshift_b200.models.unet import UNetModelSwin
    from resshift_b200.weights import random_state_dict
    sd = random_state_dict(ucfg, 0)
    m = UNetModelSwin(**ucfg.to_kwargs())
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, ucfg.in_channels, 64, 64, generator=g)
    lq = torch.rand(2, 3, 64, 64, generator=g) * 2 - 1
    t = torch.tensor([0, 3])
    out = m(x.cuda(), t.cuda(), lq=lq.cuda())
    ref = uo.unet_forward(sd, ucfg, x, t, lq=lq)            # fp32 on the CPU
    d = (out.float().cpu() - ref).abs()
    print(f"[unet] swin_embed_dim={ucfg.swin_embed_dim} mlp_ratio={ucfg.mlp_ratio}: max|d|={d.max():.3e} mean|d|={d.mean():.3e}")
    assert not torch.isnan(out).any()
    assert d.max().item() <= 1e-2 and d.mean().item() <= 2.5e-3          # test_gpu_unet_variants.py's forward bounds
    rows = plan_ops.plan_rows(m.plan(2, 64, 64), x.cuda(), t.float().cuda(), lq.cuda())
    mlps = [r for r in rows if r.startswith("mlp")]
    if expect_mlp_e:
        assert mlps and all(f"E={expect_mlp_e} " in r for r in mlps), mlps
    else:
        assert mlps == [], mlps


def test_unet_swin_embed_256_runs_the_256_instance():
    """A tiny-width UNetModelSwin with swin_embed_dim = 256: the only way a plan reaches mlp_fused_sm90_kernel<256>."""
    import dataclasses
    from resshift_b200.config import preset
    ucfg, _ = preset("tiny")
    _unet_vs_oracle(dataclasses.replace(ucfg, swin_embed_dim=256), 256)


def test_unet_reference_default_swin_width_takes_the_unfused_mlp():
    """The reference constructor's own defaults, swin_embed_dim = 96 and mlp_ratio = 2.0 (hidden 192): no fused MLP
    instance, the fc1 / fc2 convs instead."""
    import dataclasses
    from resshift_b200.config import preset
    ucfg, _ = preset("tiny")
    _unet_vs_oracle(dataclasses.replace(ucfg, swin_embed_dim=96, mlp_ratio=2.0), None)
