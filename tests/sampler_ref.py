"""Step references and trajectory comparisons shared by the sampler GPU tests (the ResShift step of
test_gpu_sampler_kernels.py, the DDPM / DDIM bounds of test_gpu_ddpm.py)."""
import numpy as np
import torch

from resshift_b200.weights import random_state_dict
from tests import gpu_util as G

U = 2.0 ** -24


def step_bound(x, x0, nz, t, ref64):
    """The step bound of test_gpu_sampler_kernels.py's module docstring for step t (x, x0, nz fp32 tensors)."""
    c1, c2 = float(ref64["coef1"][t]), float(ref64["coef2"][t])
    a, b = (c1 * x.double()).abs(), (c2 * x0.double()).abs()
    if t == 0:
        return 4 * U * (a + b)
    sn = (float(ref64["std"][t]) * nz.double()).abs()
    return 4 * U * (a + b) + 3 * U * sn + (2 + 0.5 * abs(float(ref64["log_var"][t]))) * U * sn


def step_ref(x, x0, nz, t, ref64):
    v = float(ref64["coef1"][t]) * x.double() + float(ref64["coef2"][t]) * x0.double()
    return v + float(ref64["std"][t]) * nz.double() if t != 0 else v


def dev32(a):
    """_extract_into_tensor's fp32 rounding of a float64 table, on the device"""
    return torch.from_numpy(np.asarray(a, dtype=np.float64)).float().cuda()


def ulps(a, b):
    ia, ib = G.bits(a).long(), G.bits(b).long()
    ia = torch.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return int((ia - ib).abs().max())


def _model(family, name):
    from resshift_b200.config import preset
    from resshift_b200.models.unet import UNetModel, UNetModelConv, UNetModelSwin
    if family == "unetmodel":
        from oracle.make_golden_unetmodel import case_config
        ucfg, _, hw = case_config(name)
        cls = UNetModel
    elif family == "unetconv":
        from oracle.make_golden_unetconv import case_config
        ucfg, _, hw = case_config(name)
        cls = UNetModelConv
    else:
        ucfg, _ = preset(name)
        hw, cls = (64, 64), UNetModelSwin
    m = cls(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 0), strict=True)
    return m.cuda().eval(), hw


_MODELS = {}


def cached_model(family, name):
    if (family, name) not in _MODELS:
        _MODELS[(family, name)] = _model(family, name)
    return _MODELS[(family, name)]


def bound(ref, factor=1.0):
    """test_gpu_unetmodel's bounds on a denoiser output (1e-2 max, 3e-3 mean), scaled by what carries that error into the
    step's results: the trajectory's magnitude (unclipped eps trajectories reach |x| ~ 85, and the denoiser's error is
    relative), and for eps prediction the x0 conversion's factor sqrt(1 / acp_t - 1) (``factor``, at most 15.9 on the
    1000 -> 8 schedule), which multiplies the model output's error in pred_xstart and in the step built on it"""
    s = max(1.0, float(np.abs(ref).max())) * max(1.0, factor)
    return 1e-2 * s, 3e-3 * s


def compare(tag, got, ref, bounds=None):
    got = np.asarray(got, dtype=np.float64)
    d = np.abs(got - ref)
    mx, mn = bounds or bound(ref)
    print(f"{tag}: max|d| {d.max():.3e} (bound {mx:.3e}) mean|d| {d.mean():.3e} (bound {mn:.3e}) max|ref| {np.abs(ref).max():.3e}")
    assert d.max() < mx and d.mean() < mn, tag
