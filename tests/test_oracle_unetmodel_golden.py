"""Pins the UNetModel oracle to the reference (both attention head orders, lq at the latent size and at twice it, a
non-square latent whose lowest level attends over 15 positions, a T = 4 trajectory), the package's inventory to the
reference's ``state_dict``, the constructor's refusals and the overlay's ``models.unet.UNetModel``.  The fixtures were
recorded from the unmodified reference by oracle/make_golden_unetmodel.py.  CPU only."""
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import diffusion_oracle as do
from oracle import unetmodel_oracle as uo
from oracle.make_golden_unetmodel import CASES, OUT_STRIDE, PROBE_STRIDE, case_config, case_inputs, trajectory_inputs
from resshift_b200.arch import latent_multiple, unetmodel_param_spec
from resshift_b200.config import UNetModelConfig
from resshift_b200.weights import random_state_dict

ROOT = Path(__file__).resolve().parents[1]
TOL = 2e-4   # fp32 CPU vs fp32 CPU, different op order


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(golden_dir / "unetmodel.npz")


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_forward_matches_reference(gold, name):
    ucfg, _, _ = case_config(name)
    sd = random_state_dict(ucfg, 0)
    seed, h, w = (int(v) for v in gold[f"{name}/seed"])
    x, lq = case_inputs(ucfg, 2, h, w, seed)
    probes = {}
    out = uo.unetmodel_forward(sd, ucfg, x, torch.from_numpy(gold[f"{name}/t"]), lq=lq, probes=probes)
    assert np.abs(out.reshape(-1)[::OUT_STRIDE].numpy() - gold[f"{name}/out_sub"]).max() < TOL
    keys = [k for k in gold.files if k.startswith(f"{name}/probe_sub/")]
    assert len(keys) == len(probes)
    for k in keys:
        got = probes[k.split("/probe_sub/")[1]].reshape(-1)[::PROBE_STRIDE].numpy()
        assert np.abs(got - gold[k]).max() < TOL * max(1.0, np.abs(gold[k]).max()), k


def test_oracle_loop_matches_reference(gold):
    ucfg, dcfg, hw = case_config("legacy")
    sd = random_state_dict(ucfg, 0)
    y, noises = trajectory_inputs(2, dcfg.steps, hw)
    tabs = do.schedule_tables(do.eta_schedule(dcfg.steps, dcfg.min_noise_level, dcfg.etas_end, dcfg.kappa,
                                              dcfg.schedule_kwargs["power"]), dcfg.kappa)
    final = do.p_sample_loop(lambda xx, tt: uo.unetmodel_forward(sd, ucfg, xx, tt, lq=y), y, list(noises), tabs, dcfg.kappa)
    assert np.abs(final.reshape(-1)[::OUT_STRIDE].numpy() - gold["loop/final_sub"]).max() < TOL


@pytest.mark.parametrize("name", list(CASES))
def test_param_spec_matches_reference_inventory(golden_dir, name):
    ref = json.loads((golden_dir / "unet_keys_unetmodel.json").read_text())[name]
    ucfg, _, _ = case_config(name)
    mine = {n: list(s) for n, s, _ in unetmodel_param_spec(ucfg)}
    assert mine == ref


def test_output_blocks_are_single_head_without_num_head_channels():
    """The reference builds output-block AttentionBlocks without num_heads (models/unet.py:517-523)."""
    ucfg, _, _ = case_config("new_order")
    heads = {(c, o): ucfg.heads(c, o) for c, o in ucfg.attention_layers()}
    assert all(h == 1 for (c, o), h in heads.items() if o)
    assert all(h == 2 for (c, o), h in heads.items() if not o)
    assert latent_multiple(ucfg) == 8


@pytest.mark.parametrize("kwargs,why", [
    (dict(num_classes=10), "num_classes"),
    (dict(cond_lq=False), "cond_lq"),
    (dict(dims=1), "dims"),
    (dict(num_head_channels=16), "head dims 32, 64 and 128"),
    (dict(num_head_channels=-1, num_heads=1), "head dims 32, 64 and 128"),      # the constructor's default: one 256-wide head
    (dict(in_channels=7), "in_channels"),
    (dict(model_channels=48), "GroupNorm32"),
])
def test_constructor_refuses_uncovered_options(kwargs, why):
    from resshift_b200.models.unet import UNetModel
    ucfg, _, _ = case_config("legacy")
    args = {**ucfg.to_kwargs(), **kwargs}
    with pytest.raises(ValueError, match=why):
        UNetModel(**args)
    with pytest.raises(ValueError, match=why):
        UNetModelConfig(**args)


def test_forward_refuses_labels_without_cuda():
    from resshift_b200.models.unet import UNetModel
    ucfg, _, _ = case_config("legacy")
    m = UNetModel(**ucfg.to_kwargs())
    with pytest.raises(ValueError, match="class-conditional"):
        m(torch.zeros(1, 3, 32, 32), torch.zeros(1), y=torch.zeros(1), lq=torch.zeros(1, 3, 32, 32))
    assert {n for n, _ in m.state_dict().items()} == {n for n, _, _ in unetmodel_param_spec(ucfg)}


def test_overlay_resolves_unetmodel_to_this_package(tmp_path):
    """Under `python -m resshift_b200.launch`, the reference's `models.unet.UNetModel` (a yaml `model.target`) is this
    package's class, and the sampler maps the target string to it."""
    ref_root = tmp_path / "reference"
    (ref_root / "models").mkdir(parents=True)
    probe = tmp_path / "probe_entry.py"
    probe.write_text(
        "import models.unet\n"
        "from resshift_b200.sampler import _NATIVE_TARGETS\n"
        "print('unet=' + models.unet.UNetModel.__module__)\n"
        "print('target=' + _NATIVE_TARGETS['models.unet.UNetModel'])\n")
    env = dict(**__import__("os").environ, PYTHONPATH=str(ref_root) + ":" + str(ROOT / "oracle" / "_shims"))
    out = subprocess.run([sys.executable, "-m", "resshift_b200.launch", str(probe)], cwd=str(ROOT), env=env,
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    got = dict(line.split("=", 1) for line in out.stdout.strip().splitlines() if "=" in line)
    assert got["unet"] == "resshift_b200.models.unet"
    assert got["target"] == "resshift_b200.models.unet.UNetModel"
