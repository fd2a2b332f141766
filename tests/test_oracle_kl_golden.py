"""Pins the KL first-stage oracle (oracle/kl_oracle.py) against outputs of the reference's own AutoencoderKLTorch
(oracle/make_golden_kl.py -> tests/golden/kl_*.npz, kl_keys.json), checks that the native classes and engine list the
reference's state_dict, and that the KL entry points of the C ABI refuse what they cannot run (no GPU needed)."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from oracle import kl_oracle as ko
from resshift_b200 import _lib
from resshift_b200.vq_arch import kl_param_spec, kl_preset, random_kl_state_dict, vq_preset

TOL = 2e-4
FIXTURES = [("tiny", "kl_tiny.npz"), ("f8", "kl_f8.npz")]


@pytest.mark.parametrize("name", ["tiny", "f8"])
def test_kl_param_inventory_matches_reference(golden_dir, name):
    gold = json.loads((golden_dir / "kl_keys.json").read_text())[name]
    assert [(k, list(s)) for k, s, _ in kl_param_spec(kl_preset(name))] == [(k, s) for k, s in gold]


@pytest.mark.parametrize("name", ["tiny", "f8"])
def test_native_classes_state_dict_match_reference(golden_dir, name):
    from resshift_b200.models.autoencoder import AutoencoderKLTorch, EncoderKLTorch
    gold = json.loads((golden_dir / "kl_keys.json").read_text())[name]
    cfg = kl_preset(name)
    m = AutoencoderKLTorch(**cfg.to_kwargs())
    assert [(k, list(v.shape)) for k, v in m.state_dict().items()] == [(k, s) for k, s in gold]
    m.load_state_dict(random_kl_state_dict(cfg, 1), strict=True)
    enc = EncoderKLTorch(**cfg.to_kwargs())
    assert [(k, list(v.shape)) for k, v in enc.state_dict().items()] == \
        [(k, s) for k, s in gold if k.startswith(("encoder.", "quant_conv."))]
    with pytest.raises(AssertionError):              # the reference asserts double_z for the KL classes
        AutoencoderKLTorch(**{**cfg.to_kwargs(), "ddconfig": {**cfg.ddconfig(), "double_z": False}})


@pytest.mark.parametrize("name", ["tiny", "f8"])
def test_kl_engine_inventory_matches_reference(golden_dir, name):
    gold = json.loads((golden_dir / "kl_keys.json").read_text())[name]
    h = C.c_void_p()
    cfgc = _lib.make_vq_config(kl_preset(name))
    cfgc.n_embed = 123                               # ignored by a KL engine
    _lib.check(_lib.lib.rs_kl_create(C.byref(cfgc), C.byref(h)))
    try:
        buf, shape, nd, isb = C.create_string_buffer(256), (C.c_int32 * 4)(), C.c_int32(), C.c_int32()
        mine = []
        for i in range(_lib.lib.rs_unet_param_count(h)):
            _lib.check(_lib.lib.rs_unet_param_info(h, i, buf, 256, shape, C.byref(nd), C.byref(isb)))
            mine.append([buf.value.decode(), [shape[j] for j in range(nd.value)]])
        assert mine == gold
    finally:
        _lib.lib.rs_unet_destroy(h)


@pytest.mark.parametrize("name,fname", FIXTURES)
def test_kl_encode_decode(golden_dir, name, fname):
    g = np.load(golden_dir / fname)
    cfg = kl_preset(name)
    sd = random_kl_state_dict(cfg, 0)
    x = torch.from_numpy(g["x"])
    z, m = ko.kl_encode(x, sd, cfg, return_moments=True)
    assert np.abs(m.numpy() - g["moments"]).max() < TOL
    assert np.abs(z.numpy() - g["mode"]).max() < TOL
    noise = torch.randn(z.shape, generator=torch.Generator().manual_seed(int(g["sample_seed"])))
    assert np.abs(ko.kl_encode(x, sd, cfg, noise=noise).numpy() - g["sample"]).max() < TOL
    assert np.abs(ko.kl_decode(torch.from_numpy(g["mode"]), sd, cfg).numpy() - g["dec"]).max() < TOL


def _engine(create, cfg):
    h = C.c_void_p()
    cfgc = _lib.make_vq_config(cfg)
    _lib.check(getattr(_lib.lib, create)(C.byref(cfgc), C.byref(h)))
    return h


def test_kl_entry_points_refuse_null_and_foreign_plans():
    L = _lib.lib
    nul = None
    calls = {
        "rs_kl_encode": lambda p: L.rs_kl_encode(p, nul, nul, nul, nul, nul),
        "rs_kl_encode_begin": lambda p: L.rs_kl_encode_begin(p, nul, nul),
        "rs_kl_encode_end": lambda p: L.rs_kl_encode_end(p, nul, nul, nul, nul),
        "rs_kl_decode": lambda p: L.rs_kl_decode(p, nul, nul, nul),
        "rs_kl_decode_begin": lambda p: L.rs_kl_decode_begin(p, nul, nul),
        "rs_kl_decode_end": lambda p: L.rs_kl_decode_end(p, nul, nul),
        "rs_vq_decode_code": lambda p: L.rs_vq_decode_code(p, nul, nul, nul),
    }
    for name, call in calls.items():
        assert call(None) < 0 and b"not a first-stage" in L.rs_last_error(), name
    assert L.rs_kl_create(None, None) < 0 and b"null argument" in L.rs_last_error()
    # a denoiser engine is neither
    from resshift_b200.config import preset
    h = C.c_void_p()
    ucfg = _lib.make_config(preset("tiny")[0])
    _lib.check(L.rs_unet_create(C.byref(ucfg), C.byref(h)))
    try:
        assert L.rs_vq_plan_create(h, 1, 64, 64, 0, C.byref(C.c_void_p())) < 0 and b"not a VQ-GAN or KL engine" in L.rs_last_error()
    finally:
        L.rs_unet_destroy(h)
    cfg = kl_preset("tiny")
    cfgc = _lib.make_vq_config(cfg)
    cfgc.z_channels = 9
    assert L.rs_kl_create(C.byref(cfgc), C.byref(C.c_void_p())) < 0 and b"z_channels" in L.rs_last_error()


def test_vq_and_kl_calls_refuse_each_others_plans():
    """A plan's engine kind is checked before anything else of the call (unbound plans: no device needed)."""
    L = _lib.lib
    made = []
    try:
        plans = {}
        for kind, create, cfg in (("vq", "rs_vq_create", vq_preset("tiny")), ("kl", "rs_kl_create", kl_preset("tiny"))):
            e = _engine(create, cfg)
            made.append((L.rs_unet_destroy, e))
            for which in (0, 1):
                p = C.c_void_p()
                _lib.check(L.rs_vq_plan_create(e, 1, 64, 64, which, C.byref(p)))
                made.append((L.rs_plan_destroy, p))
                plans[kind, which] = p
        nul = None
        kl_calls = [(0, lambda p: L.rs_kl_encode(p, nul, nul, nul, nul, nul)), (0, lambda p: L.rs_kl_encode_begin(p, nul, nul)),
                    (0, lambda p: L.rs_kl_encode_end(p, nul, nul, nul, nul)), (1, lambda p: L.rs_kl_decode(p, nul, nul, nul)),
                    (1, lambda p: L.rs_kl_decode_begin(p, nul, nul)), (1, lambda p: L.rs_kl_decode_end(p, nul, nul))]
        vq_calls = [(0, lambda p: L.rs_vq_encode(p, nul, nul, nul)), (0, lambda p: L.rs_vq_encode_begin(p, nul, nul)),
                    (0, lambda p: L.rs_vq_encode_end(p, nul, nul)), (1, lambda p: L.rs_vq_decode(p, nul, nul, nul, 0, nul)),
                    (1, lambda p: L.rs_vq_decode_begin(p, nul, nul, 0, nul)), (1, lambda p: L.rs_vq_decode_end(p, nul, nul)),
                    (1, lambda p: L.rs_vq_decode_code(p, nul, nul, nul))]
        for which, call in kl_calls:
            assert call(plans["vq", which]) < 0 and b"not a KL plan" in L.rs_last_error()
            assert call(plans["kl", which]) < 0 and b"not bound" in L.rs_last_error()
        for which, call in vq_calls:
            assert call(plans["kl", which]) < 0 and b"not a VQ-GAN plan" in L.rs_last_error()
            assert call(plans["vq", which]) < 0 and b"not bound" in L.rs_last_error()
        # the attention-row control takes both kinds (this 16x16 bottleneck has no fused attention)
        for kind in ("vq", "kl"):
            assert L.rs_vq_set_attention_rows(plans[kind, 0], 0, 64) < 0 and b"no fused attention" in L.rs_last_error()
    finally:
        for destroy, h in reversed(made):
            destroy(h)
