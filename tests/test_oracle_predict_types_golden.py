"""Pins the predict_type / input-scaling oracle (oracle/predict_types_oracle.py) to the reference's own
``p_sample_loop_progressive`` trajectories (tests/golden/loop_predict_types.npz, recorded by
oracle/make_golden_predict_types.py), and the library's host tables of those configurations (rs_schedule_tables_ex) to
the reference's fp32 expressions.  CPU only.

Bound of the trajectories: fp32 CPU against fp32 CPU in a different op order (the repo's 2e-4), relative to the
magnitude of the fixture where that exceeds 1: the epsilon cases reach |x| ~ 13, where 2e-4 absolute would ask for
under 4 ulp of the largest values after a 4-step loop.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import diffusion_oracle as do
from oracle import predict_types_oracle as po
from oracle.make_golden_predict_types import CASES, STRIDE, case_config, trajectory_inputs
from resshift_b200 import _lib
from resshift_b200.weights import random_state_dict

TOL = 2e-4


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(golden_dir / "loop_predict_types.npz")


def _oracle_model(name):
    ucfg, _, _ = case_config(name)
    sd = random_state_dict(ucfg, 0)
    if CASES[name][0] == "swin":
        from oracle import unet_oracle as uo
        return lambda lq: (lambda x, t: uo.unet_forward(sd, ucfg, x, t, lq=lq))
    from oracle import unetmodel_oracle as umo
    return lambda lq: (lambda x, t: umo.unetmodel_forward(sd, ucfg, x, t, lq=lq))


def _tables(dcfg):
    return do.schedule_tables(do.eta_schedule(dcfg.steps, dcfg.min_noise_level, dcfg.etas_end, dcfg.kappa,
                                              dcfg.schedule_kwargs["power"]), dcfg.kappa)


def _close(tag, got, ref):
    d = np.abs(got.reshape(-1)[::STRIDE].numpy() - ref)
    bound = TOL * max(1.0, float(np.abs(ref).max()))
    print(f"[parity] {tag}: max|d|={d.max():.3e} (bound {bound:.3e})")
    assert d.max() < bound, tag


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_loop_matches_reference(gold, name):
    _, dcfg, _ = case_config(name)
    y, noises = trajectory_inputs(name)
    rec = []
    final = po.p_sample_loop(_oracle_model(name)(y), y, list(noises), _tables(dcfg), dcfg.kappa,
                             mean_type=dcfg.predict_type, normalize_input=dcfg.normalize_input,
                             latent_flag=dcfg.latent_flag, record=rec)
    _close(f"{name} final", final, gold[f"{name}/final_sub"])
    for k, r in enumerate(rec):
        _close(f"{name} pred_xstart {k}", r["pred_xstart"], gold[f"{name}/pred_xstart/{k}"])
        _close(f"{name} sample {k}", r["sample"], gold[f"{name}/sample/{k}"])


def test_xstart_oracle_is_the_shipped_oracle():
    """For xstart with both scalings on, the loop is diffusion_oracle.p_sample_loop, bit for bit."""
    _, dcfg, _ = case_config("swin_residual")
    g = torch.Generator().manual_seed(5)
    y = torch.rand(2, 3, 8, 8, generator=g) * 2 - 1
    noises = list(torch.randn(dcfg.steps + 1, 2, 3, 8, 8, generator=g))
    model = lambda x, t: torch.tanh(x * 0.7 + t[:, None, None, None] * 0.1) - 0.2 * y
    tabs = _tables(dcfg)
    a, b = [], []
    fa = do.p_sample_loop(model, y, noises, tabs, dcfg.kappa, record=a)
    fb = po.p_sample_loop(model, y, noises, tabs, dcfg.kappa, record=b)
    assert torch.equal(fa, fb)
    for ra, rb in zip(a, b):
        for k in ("sample", "pred_xstart", "mean"):
            assert torch.equal(ra[k], rb[k]), k


# ------------------------------------------------------------------------------------------------ host tables

def _tables_ex(diff, mean_type, normalize_input, latent_flag):
    T = diff.num_timesteps
    opt = _lib.SamplerOptionsC(_lib.MEAN_TYPES[mean_type], normalize_input, latent_flag)
    dst = (C.c_float * (8 * T + 1))()
    rc = _lib.lib.rs_schedule_tables_ex(T, (C.c_double * T)(*diff.sqrt_etas.tolist()), float(diff.kappa),
                                        (C.c_int32 * T)(*diff.timestep_map), C.byref(opt), dst)
    return rc, np.frombuffer(dst, dtype=np.float32).copy()


def _diffusion(**over):
    from resshift_b200.config import DiffusionConfig
    from resshift_b200.models.script_util import create_gaussian_diffusion
    return create_gaussian_diffusion(**{**DiffusionConfig(steps=15, min_noise_level=0.04, sf=1).to_kwargs(), **over})


@pytest.mark.parametrize("normalize_input,latent_flag", [(1, 1), (1, 0), (0, 1), (0, 0)])
@pytest.mark.parametrize("mean_type", list(po.MEAN_TYPES))
def test_schedule_tables_ex_are_the_reference_fp32_values(mean_type, normalize_input, latent_flag):
    diff = _diffusion(predict_type=mean_type, normalize_input=bool(normalize_input), latent_flag=bool(latent_flag))
    T = diff.num_timesteps
    rc, a = _tables_ex(diff, mean_type, normalize_input, latent_flag)
    assert rc == 0, _lib.lib.rs_last_error()
    # the first 5 T + 1 values are rs_schedule_tables' layout; only in_scale depends on the scaling
    base = diff.step_tables()
    for j, k in enumerate(("coef1", "coef2", "std", "in_scale", "tsteps")):
        if k != "in_scale":
            assert np.array_equal(a[j * T:(j + 1) * T].view(np.int32), base[k].view(np.int32)), k
    assert a[5 * T] == base["prior_coef"]
    t = torch.arange(T)
    one = torch.ones(T)
    sqrt_etas32 = torch.from_numpy(diff.sqrt_etas)[t].float()
    if not normalize_input:
        in_scale = one
    elif latent_flag:
        in_scale = base["in_scale"]
    else:   # 1 / (fp32(sqrt_eta) * kappa * 3 + 1), every operation in fp32 as the reference's _scale_input rounds it
        in_scale = one / (sqrt_etas32 * diff.kappa * 3 + 1)
    assert np.array_equal(a[3 * T:4 * T].view(np.int32), np.asarray(in_scale, dtype=np.float32).view(np.int32))
    rows = a[5 * T + 1:].reshape(3, T)
    assert np.array_equal(rows[0].view(np.int32), (sqrt_etas32 * diff.kappa).numpy().view(np.int32))
    assert np.array_equal(rows[1].view(np.int32), torch.from_numpy(diff.etas)[t].float().numpy().view(np.int32))
    assert np.array_equal(rows[2].view(np.int32), torch.from_numpy(1 - diff.etas)[t].float().numpy().view(np.int32))


def test_schedule_tables_ex_refusals():
    diff = _diffusion()
    T = diff.num_timesteps
    se, tm = (C.c_double * T)(*diff.sqrt_etas.tolist()), (C.c_int32 * T)(*diff.timestep_map)
    dst = (C.c_float * (8 * T + 1))()
    for opt, what in (((4, 1, 1), "unknown mean type 4"), ((-1, 1, 1), "unknown mean type -1"),
                      ((0, 2, 1), "must be 0 or 1"), ((1, 1, -1), "must be 0 or 1")):
        o = _lib.SamplerOptionsC(*opt)
        assert _lib.lib.rs_schedule_tables_ex(T, se, float(diff.kappa), tm, C.byref(o), dst) != 0
        assert what in _lib.lib.rs_last_error().decode()
    assert _lib.lib.rs_schedule_tables_ex(T, se, float(diff.kappa), tm, None, dst) != 0
