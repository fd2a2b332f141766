"""Pins the first-stage oracle of the Encoder / Decoder options (oracle/vq_options_oracle.py) — level attention,
attn_type none, pooled resampling, tanh_out, dropout — against outputs of the reference's own VQModelTorch /
AutoencoderKLTorch (oracle/make_golden_vq_options.py -> tests/golden/vq_opt_*.npz, vq_keys_options.json); checks that
vq_arch, the native classes and the engine list the reference's state_dict for them, and that what stays refused is
refused with its reason (no GPU needed)."""
import ctypes as C
import json
from dataclasses import replace

import numpy as np
import pytest
import torch

from oracle import vq_options_oracle as oo
from oracle import vq_oracle as vo
from oracle.make_golden_vq_options import RUNS, configs, inputs
from resshift_b200 import _lib
from resshift_b200.vq_arch import (VQConfig, kl_param_spec, ldm_vq_preset, random_kl_state_dict, random_vq_state_dict,
                                   vq_param_spec, vq_preset)

TOL = 2e-4
CASES = list(configs())
RUN_IDS = [(name, r) for name, runs in RUNS.items() for r in range(len(runs))]


def _spec(cfg):
    return kl_param_spec(cfg) if cfg.kl else vq_param_spec(cfg)


def _model(cfg):
    from resshift_b200.models.autoencoder import AutoencoderKLTorch, VQModelTorch
    return (AutoencoderKLTorch if cfg.kl else VQModelTorch)(**cfg.to_kwargs())


@pytest.mark.parametrize("name,r", RUN_IDS)
def test_oracle_matches_reference(golden_dir, name, r):
    cfg = configs()[name]
    gold = np.load(golden_dir / RUNS[name][r][3])
    x, z = inputs(name, r)
    if cfg.kl:
        sd = random_kl_state_dict(cfg, 0)
        m = oo.kl_moments(x, sd, cfg)
        assert np.abs(m.numpy() - gold["moments"]).max() < TOL
        mode = torch.from_numpy(gold["moments"][:, :cfg.embed_dim])
        assert np.abs(oo.kl_decode(mode, sd, cfg).numpy() - gold["dec"]).max() < TOL
        return
    sd = random_vq_state_dict(cfg, 0)
    assert np.abs(oo.vq_encode(x, sd, cfg).numpy() - gold["enc"]).max() < TOL
    _, idx = oo.vq_decode(z, sd, cfg, return_indices=True)
    assert np.array_equal(idx.numpy(), gold["idx"])
    assert np.abs(oo.vq_decode(z, sd, cfg, force_not_quantize=True).numpy() - gold["dec_nq"]).max() < TOL
    if cfg.tanh_out:
        assert np.abs(gold["dec_nq"]).max() < 1


@pytest.mark.parametrize("name", ["tiny", "f4"])
def test_options_oracle_equals_shipped_oracle_without_options(name):
    """With the shipped options the options oracle computes what oracle/vq_oracle.py does, and chunked attention rows
    change nothing."""
    cfg = vq_preset(name)
    sd = random_vq_state_dict(cfg, 0)
    g = torch.Generator().manual_seed(9)
    x = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1
    ref = vo.vq_encode(x, sd, cfg)
    assert torch.equal(oo.vq_encode(x, sd, cfg), ref)
    assert torch.allclose(oo.vq_encode(x, sd, cfg, chunk=64), ref, atol=1e-5, rtol=0)
    z = torch.randn(1, cfg.embed_dim, 16, 16, generator=g) * 0.6
    assert torch.equal(oo.vq_decode(z, sd, cfg), vo.vq_decode(z, sd, cfg))


def test_attention_levels_follow_the_reference():
    """The encoder halves resolution level by level, the decoder doubles resolution // 2^(L-1): at resolution 90 the
    encoder's level 1 (45) has attention and no decoder level does (it sees 22, 44, 88)."""
    c = configs()
    assert c["res90"].enc_attn == (False, True, False) and c["res90"].dec_attn == (False, False, False)
    assert c["levels"].enc_attn == c["levels"].dec_attn == (False, True, True)
    assert c["ldm_f8"].enc_attn == c["ldm_f8"].dec_attn == (False, False, False, True)
    assert c["noattn_pool_tanh"].enc_attn == (False,) * 3 and not c["noattn_pool_tanh"].has_attn


@pytest.mark.parametrize("name", CASES)
def test_param_inventory_matches_reference(golden_dir, name):
    gold = json.loads((golden_dir / "vq_keys_options.json").read_text())[name]
    assert [(k, list(s)) for k, s, _ in _spec(configs()[name])] == [(k, s) for k, s in gold]


@pytest.mark.parametrize("name", CASES)
def test_native_class_and_engine_inventory_match_reference(golden_dir, name):
    gold = json.loads((golden_dir / "vq_keys_options.json").read_text())[name]
    cfg = configs()[name]
    m = _model(cfg)
    assert [(k, list(v.shape)) for k, v in m.state_dict().items()] == [(k, s) for k, s in gold]
    m.load_state_dict((random_kl_state_dict if cfg.kl else random_vq_state_dict)(cfg, 1), strict=True)
    h = C.c_void_p()
    cfgc, optc = _lib.make_vq_config(cfg), _lib.make_vq_options(cfg)
    _lib.check(getattr(_lib.lib, "rs_kl_create_ex" if cfg.kl else "rs_vq_create_ex")(C.byref(cfgc), C.byref(optc), C.byref(h)))
    try:
        buf, shape, nd, isb = C.create_string_buffer(256), (C.c_int32 * 4)(), C.c_int32(), C.c_int32()
        mine = []
        for i in range(_lib.lib.rs_unet_param_count(h)):
            _lib.check(_lib.lib.rs_unet_param_info(h, i, buf, 256, shape, C.byref(nd), C.byref(isb)))
            mine.append([buf.value.decode(), [shape[j] for j in range(nd.value)]])
        assert sorted(mine) == sorted(gold)
    finally:
        _lib.lib.rs_unet_destroy(h)


def test_ddconfig_options_reach_the_config():
    from resshift_b200.models.autoencoder import VQModelTorch
    cfg = configs()["noattn_pool_tanh"]
    m = VQModelTorch(**cfg.to_kwargs())
    assert (m.cfg.attn_type, m.cfg.resamp_with_conv, m.cfg.tanh_out) == ("none", False, True)
    # vanilla-xformers is AttnBlock's math with AttnBlock's parameters
    x = replace(vq_preset("tiny"), attn_resolutions=(16,), attn_type="vanilla-xformers")
    assert vq_param_spec(x) == vq_param_spec(replace(x, attn_type="vanilla"))
    # dropout is identity at inference and has no parameters
    assert vq_param_spec(replace(vq_preset("tiny"), dropout=0.3)) == vq_param_spec(vq_preset("tiny"))
    # the shipped presets keep their inventory and options
    for cfg in (vq_preset("f4"), vq_preset("f8_face")):
        o = _lib.make_vq_options(cfg)
        assert (o.mid_attn, o.resamp_with_conv, o.tanh_out) == (1, 1, 0) and not any(o.enc_attn) and not any(o.dec_attn)


@pytest.mark.parametrize("key,value,reason", [
    ("attn_type", "linear", "NotImplementedError"),
    ("attn_type", "memory-efficient-cross-attn", "NotImplementedError"),
    ("use_linear_attn", True, "NotImplementedError"),
    ("give_pre_end", True, "pre-norm features"),
    ("attn_resolutions", [64], "multiple of 64"),              # level 0 of the tiny topology has 32 channels
])
def test_refused_options_raise_value_error(key, value, reason):
    from resshift_b200.models.autoencoder import AutoencoderKLTorch, VQModelTorch
    from resshift_b200.vq_arch import kl_preset
    for cfg, cls in ((vq_preset("tiny"), VQModelTorch), (kl_preset("tiny"), AutoencoderKLTorch)):
        kw = cfg.to_kwargs()
        kw["ddconfig"] = {**kw["ddconfig"], key: value}
        with pytest.raises(ValueError, match=reason):
            cls(**kw)


def test_create_ex_refuses_bad_flags():
    L = _lib.lib
    cfg = vq_preset("tiny")
    cfgc = _lib.make_vq_config(cfg)
    for create in (L.rs_vq_create_ex, L.rs_kl_create_ex):
        c = _lib.make_vq_config(replace(cfg, double_z=True, kl=True)) if create is L.rs_kl_create_ex else cfgc
        assert create(C.byref(c), None, C.byref(C.c_void_p())) < 0 and b"null argument" in L.rs_last_error()
        for field, idx in (("enc_attn", 1), ("dec_attn", 2), ("mid_attn", None), ("resamp_with_conv", None), ("tanh_out", None)):
            for bad in (2, -1):
                o = _lib.make_vq_options(cfg)
                if idx is None:
                    setattr(o, field, bad)
                else:
                    getattr(o, field)[idx] = bad
                assert create(C.byref(c), C.byref(o), C.byref(C.c_void_p())) < 0, (field, bad)
                assert b"rs_vq_options fields are 0 or 1" in L.rs_last_error()
        o = _lib.make_vq_options(cfg)
        o.enc_attn[0] = 1                                   # 32 channels
        assert create(C.byref(c), C.byref(o), C.byref(C.c_void_p())) < 0 and b"not a multiple of 64" in L.rs_last_error()


def test_plan_refuses_fused_form_at_64_channels_naming_the_block():
    """tiny with attention at level 1 (64 channels): a 192x192 image puts 96x96 = 9216 positions there, more than the
    GEMM form holds, and the fused kernel covers 128, 256 and 512 channels."""
    L = _lib.lib
    cfg = replace(vq_preset("tiny"), attn_resolutions=(32,))
    assert cfg.enc_attn == (False, True, False)
    h = C.c_void_p()
    cfgc, optc = _lib.make_vq_config(cfg), _lib.make_vq_options(cfg)
    _lib.check(L.rs_vq_create_ex(C.byref(cfgc), C.byref(optc), C.byref(h)))
    try:
        p = C.c_void_p()
        assert L.rs_vq_plan_create(h, 1, 192, 192, 0, C.byref(p)) < 0
        err = L.rs_last_error()
        assert b"encoder.down.1.attn.0" in err and b"{128, 256, 512}" in err, err
        assert L.rs_vq_plan_create(h, 1, 192, 192, 1, C.byref(p)) < 0 and b"decoder.up.1.attn.0" in L.rs_last_error()
        _lib.check(L.rs_vq_plan_create(h, 1, 128, 128, 0, C.byref(p)))       # 64x64 = 4096 positions: the GEMM form
        try:
            n = C.c_int32(-1)
            _lib.check(L.rs_vq_attention_count(p, C.byref(n)))
            assert n.value == 0
            assert L.rs_vq_run_between(p, 1, None) < 0 and b"not bound" in L.rs_last_error()
        finally:
            L.rs_plan_destroy(p)
    finally:
        L.rs_unet_destroy(h)


def test_attention_count_of_a_plan_with_several_fused_attentions():
    """f4 with attention at 128 and 64 (levels 1 and 2: 256 and 512 channels) on a 512x512 image: 256x256 and 128x128
    positions at those levels and the mid block, 2 + 2 + 1 fused attentions in the encoder, 3 + 3 + 1 in the decoder."""
    L = _lib.lib
    cfg = replace(vq_preset("f4"), attn_resolutions=(128, 64))
    h = C.c_void_p()
    cfgc, optc = _lib.make_vq_config(cfg), _lib.make_vq_options(cfg)
    _lib.check(L.rs_vq_create_ex(C.byref(cfgc), C.byref(optc), C.byref(h)))
    try:
        for which, want in ((0, 5), (1, 7)):
            p = C.c_void_p()
            _lib.check(L.rs_vq_plan_create(h, 1, 512, 512, which, C.byref(p)))
            try:
                n = C.c_int32()
                _lib.check(L.rs_vq_attention_count(p, C.byref(n)))
                assert n.value == want
                assert L.rs_vq_set_attention_rows_at(p, want, 0, 64) < 0 and b"outside [0, %d)" % want in L.rs_last_error()
                _lib.check(L.rs_vq_set_attention_rows_at(p, want - 1, 0, 64))
                _lib.check(L.rs_vq_set_attention_rows_at(p, want - 1, 0, 128 * 128))
            finally:
                L.rs_plan_destroy(p)
    finally:
        L.rs_unet_destroy(h)


def test_ldm_presets_build():
    for name in ("vq-f8", "vq-f8-n256", "vq-f16", "vq-f4-noattn"):
        cfg = ldm_vq_preset(name)
        assert isinstance(cfg, VQConfig) and vq_param_spec(cfg)
