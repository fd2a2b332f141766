"""Pins the DDPM / DDIM process to the reference: the port's and the oracle's float64 tables (respaced to 8 and 80 and
not respaced), the public signatures, the oracle's ancestral and DDIM trajectories for the three UNet families, the
port's torch route (learned-range variance, and every fused-route case with the oracle as the model) and the launcher's
``models.script_util``.  The fixtures were recorded from the unmodified reference by oracle/make_golden_ddpm.py.
CPU only."""
import inspect
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as do
from oracle import unet_oracle, unetconv_oracle, unetmodel_oracle
from oracle.make_golden_ddpm import (BETA_END, BETA_START, CASES, E_STEPS, FUSED, OUT_STRIDE, RESPACINGS, STEPS, TABLES,
                                     case_inputs, diffusion_kwargs, learned_range_model, model_config)
from resshift_b200.models import gaussian_diffusion as gd
from resshift_b200.models.script_util import create_gaussian_diffusion_ddpm
from resshift_b200.weights import random_state_dict

ROOT = Path(__file__).resolve().parents[1]
TOL = 2e-4   # fp32 CPU vs fp32 CPU, different op order; relative to the fixture's largest magnitude


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(golden_dir / "ddpm.npz")


def _key(r):
    return str(r or STEPS)


@pytest.mark.parametrize("respacing", RESPACINGS)
def test_port_tables_equal_reference(gold, respacing):
    diff = create_gaussian_diffusion_ddpm(beta_start=BETA_START, beta_end=BETA_END, steps=STEPS,
                                          timestep_respacing=respacing)
    k = _key(respacing)
    assert diff.timestep_map == gold[f"tab/{k}/timestep_map"].tolist()
    assert diff.num_timesteps == len(diff.timestep_map) == (respacing or STEPS)
    assert diff.original_num_steps == STEPS
    for name in TABLES:
        np.testing.assert_array_equal(getattr(diff, name), gold[f"tab/{k}/{name}"], err_msg=name)
    # the rows handed to rs_ddpm_sampler_create: the reference's own tables, and FIXED_LARGE's log variance (:791-794)
    tabs = diff.ddpm_tables()
    np.testing.assert_array_equal(tabs[4], np.log(np.append(gold[f"tab/{k}/posterior_variance"][1],
                                                            gold[f"tab/{k}/betas"][1:])))
    np.testing.assert_array_equal(tabs[5], gold[f"tab/{k}/posterior_log_variance_clipped"])


@pytest.mark.parametrize("respacing", RESPACINGS)
def test_oracle_tables_equal_reference(gold, respacing):
    tabs = do.schedule(STEPS, BETA_START, BETA_END, respacing)
    k = _key(respacing)
    np.testing.assert_array_equal(tabs["timestep_map"], gold[f"tab/{k}/timestep_map"])
    for name in set(TABLES) & set(tabs):
        np.testing.assert_array_equal(tabs[name], gold[f"tab/{k}/{name}"], err_msg=name)


def test_signatures_match_reference(gold):
    ours = {"create_gaussian_diffusion_ddpm": create_gaussian_diffusion_ddpm,
            "p_sample_loop": gd.SpacedDiffusionDDPM.p_sample_loop,
            "ddim_sample_loop": gd.SpacedDiffusionDDPM.ddim_sample_loop}
    for name, fn in ours.items():
        assert str(inspect.signature(fn)) == str(gold[f"sig/{name}"]), name


def test_factory_options_and_refusals():
    kw = dict(beta_start=BETA_START, beta_end=BETA_END, timestep_respacing=8)
    V, M = gd.ModelVarTypeDDPM, gd.ModelMeanType
    assert create_gaussian_diffusion_ddpm(**kw).model_var_type == V.FIXED_LARGE
    assert create_gaussian_diffusion_ddpm(**kw).model_mean_type == M.EPSILON
    assert create_gaussian_diffusion_ddpm(sigma_small=True, **kw).model_var_type == V.FIXED_SMALL
    assert create_gaussian_diffusion_ddpm(learn_sigma=True, **kw).model_var_type == V.LEARNED_RANGE
    assert create_gaussian_diffusion_ddpm(predict_xstart=True, **kw).model_mean_type == M.START_X
    assert create_gaussian_diffusion_ddpm(**kw).scale_factor == 1.0
    with pytest.raises(NotImplementedError, match="unknown beta schedule"):
        create_gaussian_diffusion_ddpm(noise_schedule="cosine", **kw)
    with pytest.raises(AssertionError):
        create_gaussian_diffusion_ddpm(beta_start=BETA_START, beta_end=BETA_END, timestep_respacing=8.0)
    with pytest.raises(NotImplementedError):
        create_gaussian_diffusion_ddpm(**kw).training_losses(None, None, None)
    x = torch.randn(2, 3, 4, 4)
    assert create_gaussian_diffusion_ddpm(**kw)._scale_input(x, torch.tensor([1, 2])) is x


def _oracle_model(case, lq):
    family, _ = CASES[case][:2]
    ucfg, _ = model_config(case)
    sd = random_state_dict(ucfg, 0)
    fwd = {"unetmodel": unetmodel_oracle.unetmodel_forward, "unetconv": unetconv_oracle.unetconv_forward,
           "swin": unet_oracle.unet_forward}[family]
    return lambda x, t: fwd(sd, ucfg, x, t, lq=lq)


def _inputs(case):
    if CASES[case][0] == "callable":
        return case_inputs(case, hw=(16, 16))
    return case_inputs(case, hw=model_config(case)[1])


def _close(got, ref, what):
    err = np.abs(np.asarray(got) - ref).max()
    assert err < TOL * max(1.0, np.abs(ref).max()), f"{what}: max|d| {err:.3e} at max|ref| {np.abs(ref).max():.3e}"


def _check_record(gold, case, rec, final):
    _close(final.numpy(), gold[f"{case}/final"], f"{case} final")
    for k in (E_STEPS if case == "e" else range(len(rec))):
        _close(rec[k][0].reshape(-1)[::OUT_STRIDE].numpy(), gold[f"{case}/sample/{k}"], f"{case} sample {k}")
        _close(rec[k][1].reshape(-1)[::OUT_STRIDE].numpy(), gold[f"{case}/pred_xstart/{k}"], f"{case} pred_xstart {k}")


@pytest.mark.parametrize("case", FUSED + ("e",))
def test_oracle_trajectory_matches_reference(gold, case):
    _, _, respacing, loop, kw, clip, eta, _ = CASES[case]
    lq, noises = _inputs(case)
    tabs = do.schedule(STEPS, BETA_START, BETA_END, respacing)
    rec = []
    final = do.sample_loop(_oracle_model(case, lq), list(noises), tabs, loop, eps=not kw.get("predict_xstart", False),
                           clip=clip, small=kw.get("sigma_small", False), eta=eta, record=rec)
    _check_record(gold, case, rec, final)


def _port_progressive(case, model, lq, noises, monkeypatch):
    """the port's torch route, its randn_like draws fed from the case's noises"""
    _, _, _, loop, _, clip, eta, _ = CASES[case]
    diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs(case))
    queue = list(noises[1:])
    monkeypatch.setattr(torch, "randn_like", lambda ref: queue.pop(0))
    kw = dict(noise=noises[0], clip_denoised=clip, model_kwargs={"lq": lq}, device="cpu")
    if loop == "ddim":
        rec = list(diff.ddim_sample_loop_progressive(model, tuple(noises[0].shape), eta=eta, **kw))
    else:
        rec = list(diff.p_sample_loop_progressive(model, tuple(noises[0].shape), **kw))
    assert not queue
    return rec


@pytest.mark.parametrize("case", FUSED)
def test_port_torch_route_matches_reference(gold, case, monkeypatch):
    """SpacedDiffusionDDPM's torch route, with the oracle UNet as the model (timesteps mapped by the port)"""
    lq, noises = _inputs(case)
    fwd = _oracle_model(case, lq)
    rec = _port_progressive(case, lambda x, t, lq=None: fwd(x, t), lq, noises, monkeypatch)
    _check_record(gold, case, [(r["sample"], r["pred_xstart"]) for r in rec], rec[-1]["sample"])


def test_port_learned_range_matches_reference_exactly(gold, monkeypatch):
    """Case f: LEARNED_RANGE (the model's second half interpolates the log variance, :779-786) on the torch route is
    the reference's arithmetic, bit for bit."""
    lq, noises = _inputs("f")
    rec = _port_progressive("f", learned_range_model, lq, noises, monkeypatch)
    assert len(rec) == 8
    for k, r in enumerate(rec):
        np.testing.assert_array_equal(r["sample"].reshape(-1).numpy(), gold[f"f/sample/{k}"])
        np.testing.assert_array_equal(r["pred_xstart"].reshape(-1).numpy(), gold[f"f/pred_xstart/{k}"])
    np.testing.assert_array_equal(rec[-1]["sample"].numpy(), gold["f/final"])


def test_port_loop_returns_decoded_final(gold, monkeypatch):
    """p_sample_loop / ddim_sample_loop return decode_first_stage of the last sample; without a first stage that is
    the sample itself, and decode divides by scale_factor first (:1216-1225)."""
    lq, noises = _inputs("f")
    diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs("f"))
    queue = list(noises[1:])
    monkeypatch.setattr(torch, "randn_like", lambda ref: queue.pop(0))
    out = diff.p_sample_loop(learned_range_model, tuple(noises[0].shape), noise=noises[0], clip_denoised=False,
                             model_kwargs={"lq": lq}, device="cpu")
    np.testing.assert_array_equal(out.numpy(), gold["f/final"])

    class Halver(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.p = torch.nn.Parameter(torch.zeros(1))

        def decode(self, z):
            return z * 0.5

    diff.scale_factor = 0.25
    z = torch.randn(2, 3, 4, 4)
    torch.testing.assert_close(diff.decode_first_stage(z, Halver()), (1 / 0.25 * z) * 0.5, rtol=0, atol=0)


def test_launcher_resolves_ddpm_factory_to_this_package(tmp_path):
    """Under `python -m resshift_b200.launch`, the reference's `models.script_util.create_gaussian_diffusion_ddpm` (a
    script call or a yaml `diffusion.target`) is this package's factory."""
    ref_root = tmp_path / "reference"
    (ref_root / "models").mkdir(parents=True)
    probe = tmp_path / "probe_entry.py"
    probe.write_text(
        "import models.script_util as su\n"
        "f = su.create_gaussian_diffusion_ddpm\n"
        "print('factory=' + f.__module__)\n"
        "d = f(beta_start=0.0015, beta_end=0.0155, timestep_respacing=8)\n"
        "print('process=' + type(d).__module__ + '.' + type(d).__name__)\n"
        "print('resshift=' + su.create_gaussian_diffusion.__module__)\n")
    env = dict(**__import__("os").environ, PYTHONPATH=str(ref_root) + ":" + str(ROOT / "oracle" / "_shims"))
    out = subprocess.run([sys.executable, "-m", "resshift_b200.launch", str(probe)], cwd=str(ROOT), env=env,
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    got = dict(line.split("=", 1) for line in out.stdout.strip().splitlines() if "=" in line)
    assert got["factory"] == "resshift_b200.models.script_util"
    assert got["process"] == "resshift_b200.models.gaussian_diffusion.SpacedDiffusionDDPM"
    assert got["resshift"] == "resshift_b200.models.script_util"
