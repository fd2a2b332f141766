"""Pins the oracle, the parameter inventory and the shift mask to the reference for UNetModelSwin built with 16x16 windows
and / or 64-wide heads.  The fixtures were recorded from the unmodified reference by oracle/make_golden_windows.py.
CPU only."""
import json

import numpy as np
import pytest
import torch

from oracle import diffusion_oracle as do
from oracle import unet_variants_oracle as uo
from oracle.make_golden_variants import OUT_STRIDE, PROBE_STRIDE, trajectory_inputs, variant_inputs
from oracle.make_golden_windows import LOOP_MODEL, WINDOWS, windows_config
from resshift_b200.arch import shifted_window_mask, unet_param_spec
from resshift_b200.weights import random_state_dict

TOL = 2e-4   # fp32 CPU vs fp32 CPU, different op order


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(golden_dir / "unet_windows.npz")


@pytest.mark.parametrize("tag", list(WINDOWS) + [f"{LOOP_MODEL}_64x128"])
def test_oracle_forward_matches_reference(gold, tag):
    ucfg, _ = windows_config(tag.split("_64x128")[0])
    sd = random_state_dict(ucfg, 0)
    seed, h, w = (int(v) for v in gold[f"{tag}/seed"])
    x, lq, mask = variant_inputs(ucfg, 2, h, w, seed)
    probes = {}
    out = uo.unet_forward(sd, ucfg, x, torch.from_numpy(gold[f"{tag}/t"]), lq=lq, mask=mask, probes=probes)
    assert np.abs(out.reshape(-1)[::OUT_STRIDE].numpy() - gold[f"{tag}/out_sub"]).max() < TOL
    keys = [k for k in gold.files if k.startswith(f"{tag}/probe_sub/")]
    assert len(keys) == len(probes)
    for k in keys:
        got = probes[k.split("/probe_sub/")[1]].reshape(-1)[::PROBE_STRIDE].numpy()
        assert np.abs(got - gold[k]).max() < TOL * max(1.0, np.abs(gold[k]).max()), k


def test_oracle_loop_matches_reference(gold):
    ucfg, dcfg = windows_config(LOOP_MODEL)
    sd = random_state_dict(ucfg, 0)
    y, noises = trajectory_inputs(2, dcfg.steps)
    tabs = do.schedule_tables(do.eta_schedule(dcfg.steps, dcfg.min_noise_level, dcfg.etas_end, dcfg.kappa,
                                              dcfg.schedule_kwargs["power"]), dcfg.kappa)
    final = do.p_sample_loop(lambda xx, tt: uo.unet_forward(sd, ucfg, xx, tt, lq=y), y, list(noises), tabs, dcfg.kappa)
    assert np.abs(final.reshape(-1)[::OUT_STRIDE].numpy() - gold["loop/final_sub"]).max() < TOL


@pytest.mark.parametrize("name", list(WINDOWS))
def test_param_spec_matches_reference_inventory(golden_dir, name):
    ref = json.loads((golden_dir / "unet_keys_windows.json").read_text())[name]
    ucfg, _ = windows_config(name)
    mine = {n: list(s) for n, s, _ in unet_param_spec(ucfg)}
    assert mine == ref
    tables = {tuple(s) for n, s in mine.items() if n.endswith("relative_position_bias_table")}
    heads = ucfg.swin_heads
    assert tables == ({(961, heads), (225, heads)} if ucfg.window_size == 16 else {(225, heads)})


@pytest.mark.parametrize("hw", [(64, 64), (32, 32), (64, 128)])
def test_shift_mask_of_16x16_windows_equals_the_reference(gold, hw):
    ref = gold[f"mask/{hw[0]}x{hw[1]}"]
    mine = shifted_window_mask(hw[0], hw[1], 16, 8)
    assert tuple(mine.shape) == ref.shape
    assert set(mine.unique().tolist()) <= {0.0, -100.0}
    assert np.array_equal((mine != 0).numpy().astype(np.int8), ref)
    assert ref.any() and not ref[: -(hw[1] // 16)].any()        # only the last row of windows is masked


@pytest.mark.parametrize("window,head", [(8, 32), (8, 64), (16, 32), (16, 64)])
def test_constructor_accepts_the_four_instances(window, head):
    from resshift_b200.models.unet import UNetModelSwin
    ucfg, _ = windows_config("w16_h64")
    m = UNetModelSwin(**{**ucfg.to_kwargs(), "window_size": window, "num_head_channels": head})
    assert m.cfg.swin_heads == 128 // head
    assert set(m.state_dict()) == {n for n, _, _ in unet_param_spec(m.cfg)}


@pytest.mark.parametrize("kwargs,why", [
    (dict(window_size=4), "window_size"),
    (dict(window_size=7), "window_size"),
    (dict(num_head_channels=16), "head dim"),
    (dict(swin_embed_dim=96, num_head_channels=48), "head dim"),
])
def test_constructor_refuses_other_windows_and_heads(kwargs, why):
    from resshift_b200.models.unet import UNetModelSwin
    ucfg, _ = windows_config("w16_h64")
    with pytest.raises(ValueError, match=why):
        UNetModelSwin(**{**ucfg.to_kwargs(), **kwargs})


def test_library_refuses_other_windows_and_heads():
    import ctypes as C
    from resshift_b200 import _lib
    ucfg, _ = windows_config("w16_h64")
    for field, value, word in (("window_size", 4, b"window_size"), ("window_size", 32, b"window_size"),
                               ("swin_heads", 8, b"head_dim"), ("swin_heads", 1, b"head_dim")):
        cfgc, optc, h = _lib.make_config(ucfg), _lib.make_options(ucfg), C.c_void_p()
        setattr(cfgc, field, value)
        assert _lib.lib.rs_unet_create_ex(C.byref(cfgc), C.byref(optc), C.byref(h)) < 0
        assert word in _lib.lib.rs_last_error()
    cfgc, optc, h = _lib.make_config(ucfg), _lib.make_options(ucfg), C.c_void_p()
    _lib.check(_lib.lib.rs_unet_create_ex(C.byref(cfgc), C.byref(optc), C.byref(h)))
    names, buf, shape, nd, isb = {}, C.create_string_buffer(256), (C.c_int32 * 4)(), C.c_int32(), C.c_int32()
    for i in range(_lib.lib.rs_unet_param_count(h)):
        _lib.check(_lib.lib.rs_unet_param_info(h, i, buf, 256, shape, C.byref(nd), C.byref(isb)))
        names[buf.value.decode()] = tuple(shape[: nd.value])
    _lib.lib.rs_unet_destroy(h)
    assert names == {n: tuple(s) for n, s, _ in unet_param_spec(ucfg)}
