"""ORACLE (test infrastructure): the ``p_sample`` residual-shift loop of ``oracle/diffusion_oracle.py`` for every
``predict_type`` of the reference ('xstart', 'epsilon', 'epsilon_scale', 'residual') and every input scaling
(``normalize_input``, ``latent_flag``).  Every function cites the reference file:line it follows; pinned against the
trajectories of ``oracle/make_golden_predict_types.py`` (-> ``tests/golden/loop_predict_types.npz``).  For 'xstart' with
both scalings on, ``p_sample_loop`` computes exactly what ``diffusion_oracle.p_sample_loop`` does.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional

import numpy as np
import torch

MEAN_TYPES = ("xstart", "epsilon", "epsilon_scale", "residual")


def _f32(a: np.ndarray, i: int) -> torch.Tensor:
    """_extract_into_tensor (reference models/gaussian_diffusion.py:92-105): float64 table value -> fp32."""
    return torch.tensor(float(np.float32(a[i])))


def scale_input(x: torch.Tensor, tabs: Dict[str, np.ndarray], i: int, kappa: float, normalize_input: bool = True,
                latent_flag: bool = True) -> torch.Tensor:
    """_scale_input — reference models/gaussian_diffusion.py:598-609."""
    if not normalize_input:
        return x
    if latent_flag:
        return x / torch.sqrt(_f32(tabs["etas"], i) * kappa ** 2 + 1)
    return x / (_f32(tabs["sqrt_etas"], i) * kappa * 3 + 1)


def predict_xstart(mean_type: str, out: torch.Tensor, x_t: torch.Tensor, y: torch.Tensor, tabs: Dict[str, np.ndarray],
                   i: int, kappa: float) -> torch.Tensor:
    """The model output as x0 — reference models/gaussian_diffusion.py:277-292 (p_mean_variance) with
    _predict_xstart_from_eps / _eps_scale / _residual :308-324, op by op in fp32."""
    if mean_type == "xstart":
        return out
    if mean_type == "residual":
        return y - out
    if mean_type == "epsilon":
        return (x_t - _f32(tabs["sqrt_etas"], i) * kappa * out - _f32(tabs["etas"], i) * y) / _f32(1 - tabs["etas"], i)
    if mean_type == "epsilon_scale":
        return (x_t - out - _f32(tabs["etas"], i) * y) / _f32(1 - tabs["etas"], i)
    raise ValueError(f"unknown mean type {mean_type!r}")


def p_sample_loop(model: Callable, z_y: torch.Tensor, noises: List[torch.Tensor], tabs: Dict[str, np.ndarray],
                  kappa: float, mean_type: str = "xstart", normalize_input: bool = True, latent_flag: bool = True,
                  record: Optional[list] = None) -> torch.Tensor:
    """reference models/gaussian_diffusion.py:421-472 (+ p_sample :332-365, p_mean_variance :234-307,
    prior_sample :517-529), no clipping.  ``model(x_in, t)`` returns the model output; ``noises`` holds T+1 tensors in
    draw order (prior first, then one per step including the unused one at t == 0); ``tabs`` is
    ``diffusion_oracle.schedule_tables``."""
    T = len(tabs["etas"])
    x = z_y + _f32(kappa * tabs["sqrt_etas"], T - 1) * noises[0]
    for k, i in enumerate(range(T - 1, -1, -1)):
        t = torch.full((z_y.shape[0],), i, dtype=torch.long, device=z_y.device)
        out = model(scale_input(x, tabs, i, kappa, normalize_input, latent_flag), t).float()
        pred = predict_xstart(mean_type, out, x, z_y, tabs, i, kappa)
        mean = _f32(tabs["coef1"], i) * x + _f32(tabs["coef2"], i) * pred
        nonzero = 0.0 if i == 0 else 1.0
        sample = mean + nonzero * torch.exp(0.5 * _f32(tabs["log_var"], i)) * noises[k + 1]
        if record is not None:
            record.append({"sample": sample, "pred_xstart": pred, "mean": mean})
        x = sample
    return x
