"""Pins DDIM inversion (SpacedDiffusionDDPM.ddim_reverse_sample and the t = 0 .. T-1 loop around it) to the reference:
the signature, the alphas_cumprod_next row, the oracle's reverse trajectories for the three UNet families, the port's
torch route (learned-range variance bit for bit, and every fused-route case with the oracle as the model) and the
eta refusal.  The fixtures were recorded from the unmodified reference by oracle/make_golden_ddim_reverse.py.
CPU only."""
import inspect

import numpy as np
import pytest
import torch

from oracle import ddim_reverse_oracle as ro
from oracle import unet_oracle, unetconv_oracle, unetmodel_oracle
from oracle.make_golden_ddim_reverse import (CASES, FUSED, OUT_STRIDE, RESPACING, case_inputs, diffusion_kwargs,
                                             model_config)
from oracle.make_golden_ddpm import BETA_END, BETA_START, STEPS, learned_range_model
from resshift_b200 import _lib
from resshift_b200.models import gaussian_diffusion as gd
from resshift_b200.models.script_util import create_gaussian_diffusion_ddpm
from resshift_b200.weights import random_state_dict

TOL = 2e-4   # fp32 CPU vs fp32 CPU, different op order; relative to the fixture's largest magnitude


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(golden_dir / "ddim_reverse.npz")


@pytest.fixture(scope="module")
def ddpm_gold(golden_dir):
    return np.load(golden_dir / "ddpm.npz")


def test_signature_matches_reference(gold):
    assert str(inspect.signature(gd.SpacedDiffusionDDPM.ddim_reverse_sample)) == str(gold["sig/ddim_reverse_sample"])


def test_acp_next_row(ddpm_gold):
    """alphas_cumprod_next is the reference's table (0 at T - 1), and the last row handed to
    rs_ddim_reverse_sampler_create; the eight rows before it are rs_ddpm_sampler_create's."""
    diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs("a"))
    ref = ddpm_gold[f"tab/{RESPACING}/alphas_cumprod_next"]
    np.testing.assert_array_equal(diff.alphas_cumprod_next, ref)
    assert diff.alphas_cumprod_next[-1] == 0.0
    np.testing.assert_array_equal(ro.schedule(STEPS, BETA_START, BETA_END, RESPACING)["alphas_cumprod_next"], ref)
    tabs = diff.ddim_reverse_tables()
    assert tabs.shape == (len(_lib.DDPM_TABLE_ROWS) + 1, RESPACING) and tabs.flags["C_CONTIGUOUS"]
    np.testing.assert_array_equal(tabs[:len(_lib.DDPM_TABLE_ROWS)], diff.ddpm_tables())
    np.testing.assert_array_equal(tabs[len(_lib.DDPM_TABLE_ROWS)], ref)


def test_eta_other_than_zero_is_refused():
    """ddim_reverse_sample asserts eta == 0 before it calls the model, as the reference does (:1043)"""
    diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs("e"))
    x = torch.zeros(1, 3, 4, 4)

    def never(*a, **k):
        raise RuntimeError("the model must not be called")

    with pytest.raises(AssertionError, match="Reverse ODE only for deterministic path"):
        diff.ddim_reverse_sample(never, x, torch.tensor([0]), eta=0.5)


def _oracle_model(case, lq):
    family, _ = CASES[case][:2]
    ucfg, _ = model_config(case)
    sd = random_state_dict(ucfg, 0)
    fwd = {"unetmodel": unetmodel_oracle.unetmodel_forward, "unetconv": unetconv_oracle.unetconv_forward,
           "swin": unet_oracle.unet_forward}[family]
    return lambda x, t: fwd(sd, ucfg, x, t, lq=lq)


def _close(got, ref, what):
    err = np.abs(np.asarray(got) - ref).max()
    assert err < TOL * max(1.0, np.abs(ref).max()), f"{what}: max|d| {err:.3e} at max|ref| {np.abs(ref).max():.3e}"


def _check_record(gold, case, rec, final):
    _close(final.numpy(), gold[f"{case}/final"], f"{case} final")
    for k in range(len(rec)):
        _close(rec[k][0].reshape(-1)[::OUT_STRIDE].numpy(), gold[f"{case}/sample/{k}"], f"{case} sample {k}")
        _close(rec[k][1].reshape(-1)[::OUT_STRIDE].numpy(), gold[f"{case}/pred_xstart/{k}"], f"{case} pred_xstart {k}")


@pytest.mark.parametrize("case", FUSED)
def test_oracle_reverse_loop_matches_reference(gold, case):
    kw, clip = CASES[case][2], CASES[case][3]
    lq, x_start = case_inputs(case)
    tabs = ro.schedule(STEPS, BETA_START, BETA_END, RESPACING)
    rec = []
    final = ro.reverse_loop(_oracle_model(case, lq), x_start, tabs, eps=not kw.get("predict_xstart", False), clip=clip,
                            record=rec)
    assert len(rec) == RESPACING
    _check_record(gold, case, rec, final)


@pytest.mark.parametrize("case", FUSED)
def test_port_torch_route_matches_reference(gold, case):
    """SpacedDiffusionDDPM's torch route, with the oracle UNet as the model (timesteps mapped by the port)"""
    lq, x_start = case_inputs(case)
    fwd = _oracle_model(case, lq)
    diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs(case))
    model = lambda x, t, lq=None: fwd(x, t)                                        # noqa: E731
    rec = list(diff.ddim_reverse_sample_loop_progressive(model, x_start, clip_denoised=CASES[case][3],
                                                         model_kwargs={"lq": lq}))
    assert len(rec) == RESPACING
    _check_record(gold, case, [(r["sample"], r["pred_xstart"]) for r in rec], rec[-1]["sample"])


def test_port_oracle_step_is_port_step():
    """the oracle's reverse step and the port's ddim_reverse_sample are the same fp32 expression, bit for bit"""
    tabs = ro.schedule(STEPS, BETA_START, BETA_END, RESPACING)
    g = torch.Generator().manual_seed(3)
    for kw in (dict(), dict(predict_xstart=True)):
        diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs("a"), **kw)
        for clip in (False, True):
            for i in (0, RESPACING // 2, RESPACING - 1):
                x = torch.randn(2, 3, 5, 7, generator=g) * 1.5
                out = torch.randn(2, 3, 5, 7, generator=g)
                got = diff.ddim_reverse_sample(lambda xx, tt, **k: out, x, torch.tensor([i, i]), clip_denoised=clip)
                ref_s, ref_x = ro.reverse_step(tabs, i, x, out, eps=not kw, clip=clip)
                assert torch.equal(got["pred_xstart"], ref_x) and torch.equal(got["sample"], ref_s), (kw, clip, i)


def test_port_learned_range_matches_reference_exactly(gold):
    """Case e: LEARNED_RANGE (the model's second half only sets the variance, which the ODE ignores) on the torch
    route is the reference's arithmetic, bit for bit; the loop returns the last sample."""
    lq, x_start = case_inputs("e")
    diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs("e"))
    assert diff.model_var_type == gd.ModelVarTypeDDPM.LEARNED_RANGE
    assert not diff._native_ok(learned_range_model, None, {"lq": lq})
    rec = list(diff.ddim_reverse_sample_loop_progressive(learned_range_model, x_start, clip_denoised=False,
                                                         model_kwargs={"lq": lq}))
    assert len(rec) == RESPACING
    for k, r in enumerate(rec):
        np.testing.assert_array_equal(r["sample"].reshape(-1).numpy(), gold[f"e/sample/{k}"])
        np.testing.assert_array_equal(r["pred_xstart"].reshape(-1).numpy(), gold[f"e/pred_xstart/{k}"])
    out = diff.ddim_reverse_sample_loop(learned_range_model, x_start, clip_denoised=False, model_kwargs={"lq": lq})
    np.testing.assert_array_equal(out.numpy(), gold["e/final"])


def test_reverse_loop_with_denoised_fn_walks_upward():
    """denoised_fn is applied to x0 before the clamp, and the loop visits t = 0 .. T-1 at the mapped timesteps"""
    diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs("a"))
    seen = []

    def model(x, t, **k):
        seen.append(t.tolist())
        return 0.1 * x

    x = torch.rand(2, 3, 4, 4) * 2 - 1
    rec = list(diff.ddim_reverse_sample_loop_progressive(model, x, clip_denoised=True, denoised_fn=lambda v: 3 * v))
    assert seen == [[m, m] for m in diff.timestep_map]
    xt = x
    for i, r in enumerate(rec):
        t = torch.tensor([i, i])
        x0 = (3 * diff._predict_xstart_from_eps(xt, t, 0.1 * xt)).clamp(-1, 1)
        assert torch.equal(r["pred_xstart"], x0)
        xt = r["sample"]
