"""GPU tests of the reference's global-attention UNetModel on the native kernels: the multi-head attention kernel
(csrc/unet_attn.cuh) per element against float64 on the same fp16 operands over head dims, head counts, sequence
lengths and both head orders, its determinism and per-image independence; every fixture of tests/golden/unetmodel.npz against the
reference and the fp32 oracle; the fused 4-step loop with graph replay; a 64x128 latent; ResShiftSampler end to end
from a ``models.unet.UNetModel`` config, one GPU and a device pool.  Bounds are those of test_gpu_ops.py (kernel) and
test_gpu_unet.py (models)."""

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import unetmodel_oracle as uo
from oracle.make_golden_unetmodel import CASES, OUT_STRIDE, case_config, case_inputs, trajectory_inputs
from resshift_b200.weights import random_state_dict

FWD_MAX, FWD_MEAN = 1e-2, 2.5e-3
LOOP_MAX, LOOP_MEAN = 1e-2, 3e-3


def _lib():
    from resshift_b200 import _lib as L
    return L


def _attn(qkv, N, T, heads, D, new_order):
    L = _lib()
    out = torch.empty(N, T, heads * D, dtype=torch.float16, device="cuda")
    L.check(L.lib.rs_op_unet_attention(qkv.data_ptr(), N, T, heads, D, int(new_order), out.data_ptr(), L.current_stream()))
    return out


@pytest.mark.parametrize("new_order", [False, True])
@pytest.mark.parametrize("T", [1, 15, 63, 64, 65, 1000, 4096, 16384])
@pytest.mark.parametrize("heads", [1, 2, 5, 8])
@pytest.mark.parametrize("D", [32, 64, 128])
def test_unet_attention_vs_fp32(D, heads, T, new_order):
    """Per element against float64 on the fp16 operands (the bound of tests/test_gpu_attention.py)."""
    from tests.attn_ref import unet_case
    unet_case("randn", 3, T, heads, D, new_order, seed=1000 * D + 10 * heads + T % 97)


@pytest.mark.parametrize("D,heads,T", [(32, 5, 4096), (64, 2, 1000), (128, 1, 65)])
def test_unet_attention_deterministic_and_per_image(D, heads, T):
    N = 3
    g = torch.Generator(device="cuda").manual_seed(7)
    qkv = torch.randn(N, T, 3 * heads * D, device="cuda", generator=g).half()
    for new_order in (False, True):
        a = _attn(qkv, N, T, heads, D, new_order)
        b = _attn(qkv, N, T, heads, D, new_order)
        assert torch.equal(a, b)
        alone = _attn(qkv[1:2].contiguous(), 1, T, heads, D, new_order)
        assert torch.equal(alone[0], a[1])


def test_unet_attention_refuses_other_head_dims():
    L = _lib()
    qkv = torch.zeros(1, 64, 3 * 48, dtype=torch.float16, device="cuda")
    out = torch.empty(1, 64, 48, dtype=torch.float16, device="cuda")
    rc = L.lib.rs_op_unet_attention(qkv.data_ptr(), 1, 64, 1, 48, 0, out.data_ptr(), L.current_stream())
    assert rc != 0 and b"32, 64 or 128" in L.lib.rs_last_error()


# ------------------------------------------------------------------------------------------------ models

def _model(ucfg, seed=0):
    from resshift_b200.models.unet import UNetModel
    m = UNetModel(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, seed), strict=True)
    return m.cuda().eval()


def _check(tag, got, ref, bmax=FWD_MAX, bmean=FWD_MEAN):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    print(f"[parity] {tag}: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e}")
    assert not torch.isnan(got).any()
    assert d.max().item() <= bmax and d.mean().item() <= bmean, tag


@pytest.mark.parametrize("name", list(CASES))
def test_forward_vs_reference_golden(golden_dir, name):
    g = np.load(golden_dir / "unetmodel.npz")
    ucfg, _, _ = case_config(name)
    seed, h, w = (int(v) for v in g[f"{name}/seed"])
    x, lq = case_inputs(ucfg, 2, h, w, seed)
    out = _model(ucfg)(x.cuda(), torch.from_numpy(g[f"{name}/t"]).cuda(), lq=lq.cuda())
    _check(f"golden {name}", out.reshape(-1)[::OUT_STRIDE], torch.from_numpy(g[f"{name}/out_sub"]))


@pytest.mark.parametrize("name,hw", [(n, CASES[n][1:]) for n in CASES] + [("legacy", (64, 128))])
def test_forward_vs_oracle_fresh_inputs(name, hw):
    ucfg, _, _ = case_config(name)
    x, lq = case_inputs(ucfg, 2, hw[0], hw[1], 9100)
    t = torch.tensor([0, 3])
    ref = uo.unetmodel_forward(random_state_dict(ucfg, 0), ucfg, x, t, lq=lq)
    _check(f"oracle {name} {hw}", _model(ucfg)(x.cuda(), t.cuda(), lq=lq.cuda()), ref)


def test_fused_loop_vs_reference_trajectory_and_graph_replay(golden_dir):
    from resshift_b200.models.script_util import create_gaussian_diffusion
    g = np.load(golden_dir / "unetmodel.npz")
    ucfg, dcfg, hw = case_config("legacy")
    m = _model(ucfg)
    diff = create_gaussian_diffusion(**dcfg.to_kwargs())
    assert diff._native_ok(m, clip_denoised=False, denoised_fn=None, model_kwargs={"lq": None})
    y, noises = trajectory_inputs(2, dcfg.steps, hw)
    y, noises = y.cuda(), noises.cuda()
    finals = [diff.sample_latent(y, m, {"lq": y}, noises=noises).clone() for _ in range(2)]   # capture, then replay
    eager = diff.sample_latent(y, m, {"lq": y}, noises=noises, use_graph=False)
    assert torch.equal(finals[0], finals[1]) and torch.equal(finals[0], eager)
    _check("loop legacy", finals[0].reshape(-1)[::OUT_STRIDE], torch.from_numpy(g["loop/final_sub"]), LOOP_MAX, LOOP_MEAN)


def test_native_inputs_are_checked():
    from resshift_b200.models.script_util import create_gaussian_diffusion
    ucfg, dcfg, _ = case_config("lq2x")
    m = _model(ucfg)
    diff = create_gaussian_diffusion(**dcfg.to_kwargs())
    z = torch.zeros(1, 3, 32, 32, device="cuda")
    with pytest.raises(ValueError, match="lq must have shape"):
        diff.sample_latent(z, m, {"lq": torch.zeros(1, 3, 32, 32, device="cuda")})
    with pytest.raises(ValueError, match="no mask"):
        diff.sample_latent(z, m, {"lq": torch.zeros(1, 3, 64, 64, device="cuda"), "mask": torch.zeros(1, 1, 64, 64, device="cuda")})


# ------------------------------------------------------------------------------------------------ the whole pipeline

def _sampler(devices=None):
    from resshift_b200.sampler import ResShiftSampler, make_configs
    from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
    ucfg, dcfg, _ = case_config("legacy")
    dcfg.sf = 4
    vcfg = vq_preset("tiny")
    ae = {"target": "ldm.models.autoencoder.VQModelTorch", "params": vcfg.to_kwargs(), "ckpt_path": random_vq_state_dict(vcfg, 0)}
    configs = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    configs.model.target = "models.unet.UNetModel"                       # the reference's yaml target string
    return ResShiftSampler(configs, sf=4, use_amp=True, seed=123, devices=devices, chop_size=64, chop_stride=48,
                           padding_offset=64)


def test_sampler_end_to_end_and_device_pool(tmp_path):
    import cv2
    from resshift_b200.models.unet import UNetModel
    s = _sampler()
    assert isinstance(s.model, UNetModel)
    assert s.base_diffusion._native_ok(s.model, clip_denoised=False, denoised_fn=None, model_kwargs={"lq": None})
    rng = np.random.default_rng(11)
    (tmp_path / "in").mkdir()
    for name, (h, w) in {"a": (90, 70), "b": (61, 47)}.items():     # odd sizes: reflect-padded to padding_offset
        cv2.imwrite(str(tmp_path / "in" / f"{name}.png"), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
    outs = []
    for smp, d in ((s, "ref"), (_sampler("0,0"), "pool")):
        smp.setup_seed()
        smp.inference(tmp_path / "in", tmp_path / d, bs=2)
        outs.append({p.name: p.read_bytes() for p in sorted((tmp_path / d).iterdir())})
    assert len(outs[0]) == 2 and outs[0] == outs[1]
    img = cv2.imread(str(tmp_path / "ref" / "b.png"))
    assert img.shape == (61 * 4, 47 * 4, 3)
