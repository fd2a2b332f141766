"""First stages with 16- to 64-channel latents without a GPU: the oracle (oracle/kl_oracle.py, oracle/vq_oracle.py)
against outputs of the reference's own AutoencoderKLTorch / VQModelTorch on the "tiny" topology with 16- and 64-channel
latents (oracle/make_golden_wide_latents.py -> tests/golden/wide_latents.npz, wide_latents_keys.json), the parameter
inventories of those and of LDM's kl-f16 / kl-f32 in the Python spec, the native classes and the engine, the latent
width rule of VQConfig and of the engine constructors, and the wide kernels' register use (no spills, from ptxas)."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import kl_oracle as ko
from oracle import vq_oracle as vo
from resshift_b200 import _lib
from resshift_b200.vq_arch import (VQConfig, kl_param_spec, kl_preset, random_kl_state_dict, random_vq_state_dict,
                                   vq_param_spec, wide_vq_preset)

TOL = 2e-4                      # as tests/test_oracle_kl_golden.py
KL_NAMES = ["tiny16", "tiny64", "f16", "f32"]
VQ_NAMES = ["tiny16", "tiny64"]
INVENTORIES = [("kl", n) for n in KL_NAMES] + [("vq", n) for n in VQ_NAMES]


def _cfg(kind, name):
    return kl_preset(name) if kind == "kl" else wide_vq_preset(name)


def _gold_keys(golden_dir, kind, name):
    return json.loads((golden_dir / "wide_latents_keys.json").read_text())[f"{kind}_{name}"]


@pytest.mark.parametrize("kind,name", INVENTORIES)
def test_param_inventory_matches_reference(golden_dir, kind, name):
    cfg = _cfg(kind, name)
    spec = kl_param_spec(cfg) if kind == "kl" else vq_param_spec(cfg)
    assert [(k, list(s)) for k, s, _ in spec] == [(k, s) for k, s in _gold_keys(golden_dir, kind, name)]


@pytest.mark.parametrize("kind,name", [("kl", "tiny16"), ("kl", "tiny64"), ("vq", "tiny16"), ("vq", "tiny64")])
def test_native_classes_state_dict_match_reference(golden_dir, kind, name):
    from resshift_b200.models.autoencoder import AutoencoderKLTorch, VQModelTorch
    cfg = _cfg(kind, name)
    m = (AutoencoderKLTorch if kind == "kl" else VQModelTorch)(**cfg.to_kwargs())
    assert [(k, list(v.shape)) for k, v in m.state_dict().items()] == [(k, s) for k, s in _gold_keys(golden_dir, kind, name)]
    m.load_state_dict((random_kl_state_dict if kind == "kl" else random_vq_state_dict)(cfg, 1), strict=True)


def _engine(kind, cfg):
    h = C.c_void_p()
    cfgc, optc = _lib.make_vq_config(cfg), _lib.make_vq_options(cfg)
    create = _lib.lib.rs_kl_create_ex if kind == "kl" else _lib.lib.rs_vq_create_ex
    _lib.check(create(C.byref(cfgc), C.byref(optc), C.byref(h)))
    return h


@pytest.mark.parametrize("kind,name", INVENTORIES)
def test_engine_inventory_matches_reference(golden_dir, kind, name):
    h = _engine(kind, _cfg(kind, name))
    try:
        buf, shape, nd, isb = C.create_string_buffer(256), (C.c_int32 * 4)(), C.c_int32(), C.c_int32()
        mine = []
        for i in range(_lib.lib.rs_unet_param_count(h)):
            _lib.check(_lib.lib.rs_unet_param_info(h, i, buf, 256, shape, C.byref(nd), C.byref(isb)))
            mine.append([buf.value.decode(), [shape[j] for j in range(nd.value)]])
        assert mine == _gold_keys(golden_dir, kind, name)
    finally:
        _lib.lib.rs_unet_destroy(h)


@pytest.mark.parametrize("name", ["tiny16", "tiny64"])
def test_kl_oracle_against_reference(golden_dir, name):
    g = np.load(golden_dir / "wide_latents.npz")
    cfg = kl_preset(name)
    sd = random_kl_state_dict(cfg, 0)
    x = torch.from_numpy(g[f"kl_{name}_x"])
    z, m = ko.kl_encode(x, sd, cfg, return_moments=True)
    assert np.abs(m.numpy() - g[f"kl_{name}_moments"]).max() < TOL
    assert np.abs(z.numpy() - g[f"kl_{name}_mode"]).max() < TOL
    noise = torch.randn(z.shape, generator=torch.Generator().manual_seed(int(g["sample_seed"])))
    assert np.abs(ko.kl_encode(x, sd, cfg, noise=noise).numpy() - g[f"kl_{name}_sample"]).max() < TOL
    assert np.abs(ko.kl_decode(torch.from_numpy(g[f"kl_{name}_mode"]), sd, cfg).numpy() - g[f"kl_{name}_dec"]).max() < TOL


@pytest.mark.parametrize("name", ["tiny16", "tiny64"])
def test_vq_oracle_against_reference(golden_dir, name):
    g = np.load(golden_dir / "wide_latents.npz")
    cfg = wide_vq_preset(name)
    sd = random_vq_state_dict(cfg, 0)
    x, z = torch.from_numpy(g[f"vq_{name}_x"]), torch.from_numpy(g[f"vq_{name}_z"])
    assert np.abs(vo.vq_encode(x, sd, cfg).numpy() - g[f"vq_{name}_enc"]).max() < TOL
    _, idx = vo.quantize(z, sd)
    assert np.array_equal(idx.numpy(), g[f"vq_{name}_idx"])
    assert np.abs(vo.vq_decode(z, sd, cfg).numpy() - g[f"vq_{name}_dec"]).max() < TOL
    assert np.abs(vo.vq_decode(z, sd, cfg, force_not_quantize=True).numpy() - g[f"vq_{name}_dec_nq"]).max() < TOL


ACCEPTED, REFUSED = [16, 24, 64], [9, 12, 72]


@pytest.mark.parametrize("field", ["z_channels", "embed_dim"])
def test_vqconfig_latent_width_rule(field):
    for kl in (False, True):
        for c in ACCEPTED + [1, 8]:
            VQConfig(**{field: c}, double_z=kl, kl=kl)
        for c in REFUSED + [0, 65, 128, 256]:
            with pytest.raises(ValueError, match=f"{field} must be 1..8 or a multiple of 8 from 16 to 64"):
                VQConfig(**{field: c}, double_z=kl, kl=kl)


@pytest.mark.parametrize("kind", ["kl", "vq"])
@pytest.mark.parametrize("field", ["z_channels", "embed_dim"])
def test_engine_latent_width_rule(kind, field):
    """rs_kl_create / rs_vq_create take the widths VQConfig takes and name the rule for the others (taming's 256-dim
    VQGANs among them); plans of every accepted width build (no device needed)."""
    L = _lib.lib
    base = kl_preset("tiny") if kind == "kl" else wide_vq_preset("tiny16")
    create = L.rs_kl_create if kind == "kl" else L.rs_vq_create
    for c in ACCEPTED:
        cfgc = _lib.make_vq_config(base)
        setattr(cfgc, field, c)
        h = C.c_void_p()
        _lib.check(create(C.byref(cfgc), C.byref(h)))
        try:
            for which in (0, 1):
                p = C.c_void_p()
                _lib.check(L.rs_vq_plan_create(h, 1, 64, 96, which, C.byref(p)))
                L.rs_plan_destroy(p)
        finally:
            L.rs_unet_destroy(h)
    for c in REFUSED + [256]:
        cfgc = _lib.make_vq_config(base)
        setattr(cfgc, field, c)
        assert create(C.byref(cfgc), C.byref(C.c_void_p())) < 0
        msg = L.rs_last_error().decode()
        assert f"{field} must be 1..8 or a multiple of 8 from 16 to 64, got {c}" in msg, msg


@pytest.mark.parametrize("name", ["f16", "f32"])
def test_ldm_kl_plans_build(name):
    """LDM's kl-f16 / kl-f32 plans at 512x512 and 1024x1024 (no device needed)."""
    L = _lib.lib
    h = _engine("kl", kl_preset(name))
    try:
        for size in (512, 1024):
            for which in (0, 1):
                p = C.c_void_p()
                _lib.check(L.rs_vq_plan_create(h, 1, size, size, which, C.byref(p)))
                L.rs_plan_destroy(p)
    finally:
        L.rs_unet_destroy(h)


_NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
_WIDE_KERNELS = ["pointwise_conv_wide_kernel", "kl_posterior_wide_kernel"] + \
    [f"vq_quantize_wide_kernel<{e}>" for e in range(16, 65, 8)]


@pytest.mark.skipif(shutil.which(_NVCC) is None, reason="nvcc not available")
def test_wide_kernels_do_not_spill(tmp_path):
    """Every wide first-stage kernel instance compiles for sm_90a with no local-memory stack and no spills."""
    csrc = Path(__file__).resolve().parent.parent / "resshift_b200" / "csrc"
    src = tmp_path / "wide.cu"
    src.write_text(f'#include "{csrc / "vq_kernels.cuh"}"\n' + "".join(
        f"template __global__ void rs::vq_quantize_wide_kernel<{e}>(const rs::QuantizeParams);\n" for e in range(16, 65, 8)))
    r = subprocess.run([_NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
                        str(src), "-o", str(tmp_path / "wide.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    names = subprocess.run(["c++filt"], input=r.stderr, capture_output=True, text=True).stdout \
        if shutil.which("c++filt") else r.stderr
    found = {}
    cur = None
    for line in names.splitlines():
        m = re.search(r"Compiling entry function '(.+)' for 'sm_90a'", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            found[cur] = tuple(int(v) for v in m.groups())
    for k in _WIDE_KERNELS:
        mangled = re.sub(r"<(\d+)>", r"ILi\1E", k)                  # the name when c++filt is not there
        hits = [v for name, v in found.items() if k in name or mangled in name]
        assert hits, f"{k}: not in the ptxas report"
        assert hits[0] == (0, 0, 0), f"{k}: stack frame / spill stores / spill loads {hits[0]}"
