"""Pins the UNetModelConv oracle to the reference (the constructor defaults; scale-shift with ResBlockConv down / up and
pooled resampling; lq at twice the latent size; uneven num_res_blocks on a non-square latent; a T = 4 trajectory), the
package's inventory to the reference's ``state_dict``, the constructor's refusals and the overlay's
``models.unet.UNetModelConv``.  The fixtures were recorded from the unmodified reference by
oracle/make_golden_unetconv.py.  CPU only."""
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import diffusion_oracle as do
from oracle import unetconv_oracle as uo
from oracle.make_golden_unetconv import CASES, OUT_STRIDE, PROBE_STRIDE, case_config, case_inputs, trajectory_inputs
from resshift_b200.arch import latent_multiple, unetconv_param_spec
from resshift_b200.config import UNetModelConvConfig
from resshift_b200.weights import random_state_dict

ROOT = Path(__file__).resolve().parents[1]
TOL = 2e-4   # fp32 CPU vs fp32 CPU, different op order


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(golden_dir / "unetconv.npz")


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_forward_matches_reference(gold, name):
    ucfg, _, _ = case_config(name)
    sd = random_state_dict(ucfg, 0)
    seed, h, w = (int(v) for v in gold[f"{name}/seed"])
    x, lq = case_inputs(ucfg, 2, h, w, seed)
    probes = {}
    out = uo.unetconv_forward(sd, ucfg, x, torch.from_numpy(gold[f"{name}/t"]), lq=lq, probes=probes)
    assert np.abs(out.reshape(-1)[::OUT_STRIDE].numpy() - gold[f"{name}/out_sub"]).max() < TOL
    keys = [k for k in gold.files if k.startswith(f"{name}/probe_sub/")]
    assert len(keys) == len(probes)
    for k in keys:
        got = probes[k.split("/probe_sub/")[1]].reshape(-1)[::PROBE_STRIDE].numpy()
        assert np.abs(got - gold[k]).max() < TOL * max(1.0, np.abs(gold[k]).max()), k


def test_oracle_loop_matches_reference(gold):
    ucfg, dcfg, hw = case_config("defaults")
    sd = random_state_dict(ucfg, 0)
    y, noises = trajectory_inputs(2, dcfg.steps, hw)
    tabs = do.schedule_tables(do.eta_schedule(dcfg.steps, dcfg.min_noise_level, dcfg.etas_end, dcfg.kappa,
                                              dcfg.schedule_kwargs["power"]), dcfg.kappa)
    final = do.p_sample_loop(lambda xx, tt: uo.unetconv_forward(sd, ucfg, xx, tt, lq=y), y, list(noises), tabs, dcfg.kappa)
    assert np.abs(final.reshape(-1)[::OUT_STRIDE].numpy() - gold["loop/final_sub"]).max() < TOL


@pytest.mark.parametrize("name", list(CASES))
def test_param_spec_matches_reference_inventory(golden_dir, name):
    ref = json.loads((golden_dir / "unet_keys_unetconv.json").read_text())[name]
    ucfg, _, _ = case_config(name)
    mine = {n: list(s) for n, s, _ in unetconv_param_spec(ucfg)}
    assert mine == ref
    assert not any(".in_layers.0." in n or n.startswith("out.0.") for n in mine)      # no GroupNorm parameters
    assert latent_multiple(ucfg) == 2 ** (len(ucfg.channel_mult) - 1)


@pytest.mark.parametrize("kwargs,why", [
    (dict(cond_lq=False), "cond_lq"),
    (dict(dims=1), "dims"),
    (dict(in_channels=7), "in_channels"),
    (dict(model_channels=36), "multiple of 8"),
    (dict(channel_mult=(1, 2, 2), num_res_blocks=(1, 1)), "same length"),
])
def test_constructor_refuses_uncovered_options(kwargs, why):
    from resshift_b200.models.unet import UNetModelConv
    ucfg, _, _ = case_config("defaults")
    args = {**ucfg.to_kwargs(), **kwargs}
    with pytest.raises(ValueError, match=why):
        UNetModelConv(**args)
    with pytest.raises(ValueError, match=why):
        UNetModelConvConfig(**args)


def test_forward_has_the_reference_signature():
    """forward(x, timesteps, lq=None): no mask= (as the reference's), lq required, x with out_channels channels."""
    from resshift_b200.models.unet import UNetModelConv
    ucfg, _, _ = case_config("defaults")
    m = UNetModelConv(**ucfg.to_kwargs())
    with pytest.raises(TypeError):
        m(torch.zeros(1, 3, 32, 32), torch.zeros(1), lq=torch.zeros(1, 3, 32, 32), mask=torch.zeros(1, 1, 32, 32))
    with pytest.raises(ValueError, match="pass lq="):
        m(torch.zeros(1, 3, 32, 32), torch.zeros(1))
    with pytest.raises(ValueError, match="out_channels"):
        m(torch.zeros(1, 6, 32, 32), torch.zeros(1), lq=torch.zeros(1, 3, 32, 32))
    assert {n for n, _ in m.state_dict().items()} == {n for n, _, _ in unetconv_param_spec(ucfg)}
    # zero_module (reference models/unet.py:964-967)
    assert all(float(v.abs().sum()) == 0 for n, v in m.state_dict().items() if ".out_layers.1." in n)


def test_make_configs_targets_unetconv():
    from resshift_b200.sampler import make_configs
    ucfg, dcfg, _ = case_config("ss_updown")
    cfg = make_configs(ucfg, dcfg)
    assert cfg.model.target == "resshift_b200.models.unet.UNetModelConv"
    assert UNetModelConvConfig(**dict(cfg.model.params)) == ucfg


def test_overlay_resolves_unetconv_to_this_package(tmp_path):
    """Under `python -m resshift_b200.launch`, the reference's `models.unet.UNetModelConv` (a yaml `model.target`) is this
    package's class, and the sampler maps the target string to it."""
    ref_root = tmp_path / "reference"
    (ref_root / "models").mkdir(parents=True)
    probe = tmp_path / "probe_entry.py"
    probe.write_text(
        "import models.unet\n"
        "from resshift_b200.sampler import _NATIVE_TARGETS\n"
        "print('unet=' + models.unet.UNetModelConv.__module__)\n"
        "print('target=' + _NATIVE_TARGETS['models.unet.UNetModelConv'])\n")
    env = dict(**__import__("os").environ, PYTHONPATH=str(ref_root) + ":" + str(ROOT / "oracle" / "_shims"))
    out = subprocess.run([sys.executable, "-m", "resshift_b200.launch", str(probe)], cwd=str(ROOT), env=env,
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    got = dict(line.split("=", 1) for line in out.stdout.strip().splitlines() if "=" in line)
    assert got["unet"] == "resshift_b200.models.unet"
    assert got["target"] == "resshift_b200.models.unet.UNetModelConv"
