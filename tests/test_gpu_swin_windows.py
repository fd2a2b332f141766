"""GPU parity of the window-attention core's four instances (windows of 8 or 16, heads of 32 or 64) and of UNetModelSwin
built with 16x16 windows and / or 64-wide heads: the core and the SIMT cross-check per element against float64 (the
bounds of tests/test_gpu_attention.py); whole forwards against the reference's goldens (tests/golden/unet_windows.npz) and the fp32 oracle; the
fused 4-step loop; a 128x128 latent; batch independence; graph replay; the sampler's padding.  Bounds are those of
test_gpu_unet.py and test_gpu_ops.py."""
import hashlib
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import unet_variants_oracle as uo
from oracle.make_golden_variants import OUT_STRIDE, trajectory_inputs, variant_inputs
from oracle.make_golden_windows import LOOP_MODEL, WINDOWS, windows_config
from resshift_b200 import _lib
from resshift_b200.weights import random_state_dict

FWD_MAX, FWD_MEAN = 1e-2, 2.5e-3
LOOP_MAX, LOOP_MEAN = 1e-2, 3e-3
INSTANCES = [(8, 32), (8, 64), (16, 32), (16, 64)]

# sha256 of the <8, 32> core's output bytes for _core_inputs(2, 16, 32, 6, 8, 32, seed=11), shift 0 and 4, recorded from
# the build before the kernel became a template (H100, the same inputs from the CPU generator)
PARENT_SHA256 = {0: "89ad004740c316618d3bb3fa3543a141f8495160c20d30d28191d1bc23d00d99", 4: "142a9c51ac9ce16d728a7f59d58e6c9bbc09de61f2c71188b1951c428be87b24"}


# ------------------------------------------------------------------------------------------------ the core kernel

def _core_inputs(N, H, W, heads, ws, hd, seed):
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(N, H, W, 3 * heads * hd, generator=g).half()
    table = torch.randn((2 * ws - 1) ** 2, heads, generator=g) * 0.5
    return qkv.cuda(), table.cuda()


def _core(qkv, table, heads, ws, hd, shift, impl):
    N, H, W, _ = qkv.shape
    T = ws * ws
    dense = torch.empty(heads * T * T, dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.rs_op_expand_relpos_ex(table.data_ptr(), dense.data_ptr(), heads, ws, _lib.current_stream()))
    out = torch.full((N, H, W, heads * hd), float("nan"), dtype=torch.float16, device="cuda")
    os.environ["RS_ATTN_IMPL"] = impl
    try:
        _lib.check(_lib.lib.rs_op_window_attention_ex(qkv.data_ptr(), N, H, W, heads, ws, hd, shift, dense.data_ptr(),
                                                      out.data_ptr(), _lib.current_stream()))
        torch.cuda.synchronize()
    finally:
        os.environ.pop("RS_ATTN_IMPL", None)
    return out


# (windows along H, windows along W): one window, rectangular with odd counts both ways, the last row of windows masked
@pytest.mark.parametrize("shifted", [False, True])
@pytest.mark.parametrize("grid", [(1, 1), (3, 1), (2, 5), (4, 4)])
@pytest.mark.parametrize("heads", [1, 3, 6])
@pytest.mark.parametrize("ws,hd", INSTANCES)
def test_core_instances_vs_fp32_and_simt(ws, hd, heads, grid, shifted):
    """Each instance and the SIMT cross-check per element against float64 (tests/test_gpu_attention.py); the
    RS_ATTN_IMPL-selected rs_op_window_attention_ex gives the same bits as the explicit launch."""
    from tests.attn_ref import WindowCase
    if shifted and grid == (1, 1):
        pytest.skip("no shifted windows at a single-window resolution")
    shift = ws // 2 if shifted else 0
    L = WindowCase("randn", 3, grid[0], grid[1], heads, ws, hd, shift, seed=ws * 100 + hd + heads + grid[0] * ws + shift)
    for impl in ("mma", "simt"):
        out, _, _ = L.check(f"core {impl} ws={ws} hd={hd} heads={heads} grid={grid} shift={shift}", simt=impl == "simt")
        assert torch.equal(out, _core(L.qkv, L.table, heads, ws, hd, shift, impl)), impl


@pytest.mark.parametrize("shift", [0, 4])
def test_instance_8_32_is_bit_identical_to_the_untemplated_kernel(shift):
    qkv, table = _core_inputs(2, 16, 32, 6, 8, 32, seed=11)
    out = _core(qkv, table, 6, 8, 32, shift, "mma")
    dense = torch.empty(6 * 64 * 64, dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.rs_op_expand_relpos(table.data_ptr(), dense.data_ptr(), 6, _lib.current_stream()))
    old_entry = torch.empty_like(out)
    _lib.check(_lib.lib.rs_op_window_attention(qkv.data_ptr(), 2, 16, 32, 6, shift, dense.data_ptr(), old_entry.data_ptr(),
                                               _lib.current_stream()))
    torch.cuda.synchronize()
    assert torch.equal(out, old_entry)
    assert hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest() == PARENT_SHA256[shift]


def test_core_refuses_other_windows_heads_and_shifts():
    qkv, table = _core_inputs(1, 32, 32, 2, 16, 64, seed=1)
    for ws, hd, shift, H, why in ((4, 64, 0, 32, "window_size"), (16, 48, 0, 32, "head_dim"), (16, 64, 4, 32, "shift"),
                                  (16, 64, 0, 24, "multiples")):
        rc = _lib.lib.rs_op_window_attention_ex(qkv.data_ptr(), 1, H, 32, 2, ws, hd, shift, table.data_ptr(), qkv.data_ptr(),
                                                _lib.current_stream())
        assert rc < 0 and why.encode() in _lib.lib.rs_last_error(), (ws, hd, shift, H)


# ------------------------------------------------------------------------------------------------ whole models

def _model(ucfg, seed=0):
    from resshift_b200.models.unet import UNetModelSwin
    m = UNetModelSwin(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, seed), strict=True)
    return m.cuda().eval()


def _check(tag, got, ref, bmax=FWD_MAX, bmean=FWD_MEAN):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    print(f"[parity] {tag}: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e}")
    assert not torch.isnan(got).any()
    assert d.max().item() <= bmax and d.mean().item() <= bmean, tag


def _cuda(*ts):
    return [None if t is None else t.cuda() for t in ts]


@pytest.mark.parametrize("tag", list(WINDOWS) + [f"{LOOP_MODEL}_64x128"])
def test_forward_vs_reference_golden(golden_dir, tag):
    g = np.load(golden_dir / "unet_windows.npz")
    ucfg, _ = windows_config(tag.split("_64x128")[0])
    seed, h, w = (int(v) for v in g[f"{tag}/seed"])
    x, lq, mask = _cuda(*variant_inputs(ucfg, 2, h, w, seed))
    out = _model(ucfg)(x, torch.from_numpy(g[f"{tag}/t"]).cuda(), lq=lq, mask=mask)
    _check(f"golden {tag}", out.reshape(-1)[::OUT_STRIDE], torch.from_numpy(g[f"{tag}/out_sub"]))


@pytest.mark.parametrize("name", list(WINDOWS))
def test_forward_vs_oracle_fresh_inputs(name):
    ucfg, _ = windows_config(name)
    x, lq, mask = variant_inputs(ucfg, 2, 64, 64, 9300)
    t = torch.tensor([0, 3])
    ref = uo.unet_forward(random_state_dict(ucfg, 0), ucfg, x, t, lq=lq, mask=mask)
    x, lq, mask, t = _cuda(x, lq, mask, t)
    _check(f"oracle {name}", _model(ucfg)(x, t, lq=lq, mask=mask), ref)


def test_forward_with_the_simt_cross_check_agrees_with_the_tensor_core_path(monkeypatch):
    ucfg, _ = windows_config(LOOP_MODEL)
    x, lq, _ = _cuda(*variant_inputs(ucfg, 2, 64, 64, 9301))
    t = torch.tensor([2, 1], device="cuda")
    a = _model(ucfg)(x, t, lq=lq).clone()
    monkeypatch.setenv("RS_ATTN_IMPL", "simt")
    _check("simt vs tensor core", _model(ucfg)(x, t, lq=lq), a)      # (the cross-check keeps P in fp32, the instances round it to fp16)


def test_fused_loop_vs_reference_trajectory_and_graph_replay(golden_dir):
    from resshift_b200.models.script_util import create_gaussian_diffusion
    g = np.load(golden_dir / "unet_windows.npz")
    ucfg, dcfg = windows_config(LOOP_MODEL)
    m = _model(ucfg)
    diff = create_gaussian_diffusion(**dcfg.to_kwargs())
    assert diff._native_ok(m, clip_denoised=False, denoised_fn=None, model_kwargs={"lq": None})
    y, noises = _cuda(*trajectory_inputs(2, dcfg.steps))
    finals = [diff.sample_latent(y, m, {"lq": y}, noises=noises).clone() for _ in range(2)]   # capture, then replay
    assert torch.equal(finals[0], finals[1])
    _check("loop w16_h64", finals[0].reshape(-1)[::OUT_STRIDE], torch.from_numpy(g["loop/final_sub"]), LOOP_MAX, LOOP_MEAN)


def test_graph_replay_equals_eager_enqueue():
    ucfg, _ = windows_config(LOOP_MODEL)
    m = _model(ucfg)
    x, lq, _ = _cuda(*variant_inputs(ucfg, 2, 64, 64, 9302))
    t = torch.tensor([3, 0], device="cuda")
    eager = m(x, t, lq=lq).clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m(x, t, lq=lq)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = m(x, t, lq=lq)
    for _ in range(2):
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager)


def test_128x128_latent_vs_oracle_on_gpu():
    """Twice the constructor's size: 8x8 windows of 16 at the first level, and the 8x8 level of the constructor (one
    window of 8) becomes a 16x16 map of four."""
    ucfg, _ = windows_config(LOOP_MODEL)
    sd = random_state_dict(ucfg, 0)
    x, lq, _ = _cuda(*variant_inputs(ucfg, 1, 128, 128, 9303))
    t = torch.tensor([2], device="cuda")
    tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        ref = uo.unet_forward({k: v.cuda() for k, v in sd.items()}, ucfg, x, t, lq=lq)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    _check("128x128 w16_h64", _model(ucfg)(x, t, lq=lq), ref)


def test_images_of_a_batch_are_independent():
    ucfg, _ = windows_config(LOOP_MODEL)
    m = _model(ucfg)
    x, lq, _ = _cuda(*variant_inputs(ucfg, 3, 64, 64, 9304))
    t = torch.tensor([3, 1, 2], device="cuda")
    full = m(x, t, lq=lq).clone()
    x2, lq2, t2 = torch.randn_like(x), torch.rand_like(lq) * 2 - 1, torch.tensor([0, 1, 0], device="cuda")
    x2[1], lq2[1] = x[1], lq[1]
    other = m(x2, t2, lq=lq2)
    assert torch.equal(other[1], full[1]) and not torch.equal(other[0], full[0])


def test_indivisible_latent_names_the_required_multiple():
    ucfg, _ = windows_config(LOOP_MODEL)
    m = _model(ucfg)
    x, lq, _ = _cuda(*variant_inputs(ucfg, 1, 96, 64, 1))
    with pytest.raises(ValueError, match="multiples of 64"):
        m(x, torch.tensor([1], device="cuda"), lq=lq)
    import ctypes as C
    h = C.c_void_p()
    assert _lib.lib.rs_plan_create(m._ensure_engine(x.device), 1, 96, 64, C.byref(h)) < 0
    assert b"multiples of 64" in _lib.lib.rs_last_error()


def test_sampler_pads_a_96x80_input_to_the_models_multiple():
    from resshift_b200.sampler import ResShiftSampler, make_configs
    from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
    ucfg, dcfg = windows_config(LOOP_MODEL)
    dcfg.sf = 4
    vcfg = vq_preset("tiny")
    ae = {"target": "ldm.models.autoencoder.VQModelTorch", "params": vcfg.to_kwargs(), "ckpt_path": random_vq_state_dict(vcfg, 0)}
    configs = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    s = ResShiftSampler(configs, sf=4, use_amp=True, seed=123, chop_size=512, chop_stride=448, padding_offset=64)
    gen = torch.Generator(device="cuda").manual_seed(9)
    y0 = torch.rand(1, 3, 96, 80, device="cuda", generator=gen) * 2 - 1
    outs = [s.sample_func(y0, noise_repeat=True).clone() for _ in range(2)]
    assert tuple(outs[0].shape) == (1, 3, 384, 320) and not torch.isnan(outs[0]).any()
    assert torch.equal(outs[0], outs[1])
    assert outs[0].abs().max().item() <= 1.0 and outs[0].std().item() > 1e-3
