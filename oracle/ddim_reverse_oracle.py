"""ORACLE (test infrastructure): CPU fp32 restatement of DDIM inversion in the reference's DDPM process
(``GaussianDiffusionDDPM.ddim_reverse_sample``, reference models/gaussian_diffusion.py:1030-1066) for eps and x0
prediction, and the t = 0 .. T-1 loop around it.  Builds on ``oracle/ddpm_oracle.py`` (schedule, x0); pinned against
trajectories produced by the imported reference (``oracle/make_golden_ddim_reverse.py`` ->
``tests/golden/ddim_reverse.npz``).
"""
from __future__ import annotations

from typing import Callable, Dict, Optional

import numpy as np
import torch

from oracle.ddpm_oracle import _f32, pred_xstart
from oracle.ddpm_oracle import schedule as _ddpm_schedule


def schedule(steps: int, beta_start: float, beta_end: float, respacing: Optional[int] = None) -> Dict[str, np.ndarray]:
    """ddpm_oracle.schedule plus alphas_cumprod_next = append(acp[1:], 0) (reference models/gaussian_diffusion.py:653)"""
    tabs = _ddpm_schedule(steps, beta_start, beta_end, respacing)
    tabs["alphas_cumprod_next"] = np.append(tabs["alphas_cumprod"][1:], 0.0)
    return tabs


def reverse_step(tabs, i: int, x, out, eps: bool, clip: bool):
    """ddim_reverse_sample (reference models/gaussian_diffusion.py:1043-1066): eps re-derived from x0 (:1054-1057), then
    x_{t+1} = x0 sqrt(acp_next) + sqrt(1 - acp_next) eps (:1058-1064).  Returns (sample, pred_xstart)."""
    x0 = pred_xstart(tabs, i, x, out, eps, clip)
    e = (_f32(tabs["sqrt_recip_alphas_cumprod"], i) * x - x0) / _f32(tabs["sqrt_recipm1_alphas_cumprod"], i)
    an = _f32(tabs["alphas_cumprod_next"], i)
    return x0 * torch.sqrt(an) + torch.sqrt(1 - an) * e, x0


def reverse_loop(model: Callable, x_start: torch.Tensor, tabs: Dict[str, np.ndarray], eps: bool, clip: bool,
                 record: Optional[list] = None) -> torch.Tensor:
    """x = x_start, then for t = 0 .. T-1 the model on x at the mapped timestep (models/respace.py:60-63) and the
    reverse step.  ``model(x, t_model)``; ``record`` receives (sample, pred_xstart) per step."""
    T = len(tabs["betas"])
    x = x_start
    for i in range(T):
        t = torch.full((x.shape[0],), int(tabs["timestep_map"][i]), dtype=torch.long)
        x, x0 = reverse_step(tabs, i, x, model(x, t).float(), eps, clip)
        if record is not None:
            record.append((x, x0))
    return x
