"""ORACLE (test infrastructure): CPU fp32 restatement of the reference's DDPM / DDIM process
(``GaussianDiffusionDDPM`` / ``SpacedDiffusionDDPM``): its respaced float64 schedule, the ancestral step and the DDIM
step for eps and x0 prediction with the fixed variances, and the two loops.  Every function cites the reference
file:line it follows; pinned against tables and trajectories produced by the imported reference
(``oracle/make_golden_ddpm.py`` -> ``tests/golden/ddpm.npz``).
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional

import numpy as np
import torch


def schedule(steps: int, beta_start: float, beta_end: float, respacing: Optional[int] = None) -> Dict[str, np.ndarray]:
    """float64 tables of the respaced process.  Betas: "linear" schedule (reference models/gaussian_diffusion.py:25-28);
    kept steps: space_timesteps (models/respace.py:17-18); respaced betas 1 - acp_i / acp_last (respace.py:79-88);
    tables: models/gaussian_diffusion.py:642-680 and FIXED_LARGE's variance :791-794."""
    base = np.linspace(beta_start ** 0.5, beta_end ** 0.5, steps, dtype=np.float64) ** 2
    n = steps if respacing is None else respacing
    keep = {int((steps / n) * x) for x in range(n)}
    tmap, betas, last = [], [], 1.0
    for i, acp in enumerate(np.cumprod(1.0 - base)):
        if i in keep:
            betas.append(1 - acp / last)
            last = acp
            tmap.append(i)
    b = np.array(betas, dtype=np.float64)
    acp = np.cumprod(1.0 - b)
    acp_prev = np.append(1.0, acp[:-1])
    pv = b * (1.0 - acp_prev) / (1.0 - acp)
    return {
        "timestep_map": np.array(tmap, dtype=np.int64),
        "betas": b,
        "alphas_cumprod": acp,
        "alphas_cumprod_prev": acp_prev,
        "sqrt_recip_alphas_cumprod": np.sqrt(1.0 / acp),
        "sqrt_recipm1_alphas_cumprod": np.sqrt(1.0 / acp - 1),
        "posterior_variance": pv,
        "posterior_log_variance_clipped": np.log(np.append(pv[1], pv[1:])),
        "posterior_mean_coef1": b * np.sqrt(acp_prev) / (1.0 - acp),
        "posterior_mean_coef2": (1.0 - acp_prev) * np.sqrt(1.0 - b) / (1.0 - acp),
        "log_variance_fixed_large": np.log(np.append(pv[1], b[1:])),
    }


def _f32(tab: np.ndarray, i: int) -> torch.Tensor:
    """_extract_into_tensor: the float64 value cast to fp32 (reference models/gaussian_diffusion.py:92-105)"""
    return torch.tensor(float(np.float32(tab[i])))


def pred_xstart(tabs, i: int, x: torch.Tensor, out: torch.Tensor, eps: bool, clip: bool) -> torch.Tensor:
    """p_mean_variance's x0 (reference models/gaussian_diffusion.py:803-824, _predict_xstart_from_eps :838-843)"""
    x0 = _f32(tabs["sqrt_recip_alphas_cumprod"], i) * x - _f32(tabs["sqrt_recipm1_alphas_cumprod"], i) * out if eps else out
    return x0.clamp(-1, 1) if clip else x0


def ancestral_step(tabs, i: int, x, out, noise, eps: bool, clip: bool, small: bool):
    """p_sample (reference models/gaussian_diffusion.py:879-892) with q_posterior_mean_variance (:726-729); the
    log variance of FIXED_SMALL or FIXED_LARGE (:788-801).  Returns (sample, pred_xstart)."""
    x0 = pred_xstart(tabs, i, x, out, eps, clip)
    mean = _f32(tabs["posterior_mean_coef1"], i) * x0 + _f32(tabs["posterior_mean_coef2"], i) * x
    lv = _f32(tabs["posterior_log_variance_clipped" if small else "log_variance_fixed_large"], i)
    nonzero = torch.tensor(0.0 if i == 0 else 1.0)
    return mean + nonzero * torch.exp(0.5 * lv) * noise, x0


def ddim_step(tabs, i: int, x, out, noise, eps: bool, clip: bool, eta: float):
    """ddim_sample (reference models/gaussian_diffusion.py:1000-1028, _predict_eps_from_xstart :855-859).
    Returns (sample, pred_xstart)."""
    x0 = pred_xstart(tabs, i, x, out, eps, clip)
    e = (_f32(tabs["sqrt_recip_alphas_cumprod"], i) * x - x0) / _f32(tabs["sqrt_recipm1_alphas_cumprod"], i)
    ab, abp = _f32(tabs["alphas_cumprod"], i), _f32(tabs["alphas_cumprod_prev"], i)
    sigma = eta * torch.sqrt((1 - abp) / (1 - ab)) * torch.sqrt(1 - ab / abp)
    mean = x0 * torch.sqrt(abp) + torch.sqrt(1 - abp - sigma ** 2) * e
    nonzero = torch.tensor(0.0 if i == 0 else 1.0)
    return mean + nonzero * sigma * noise, x0


def sample_loop(model: Callable, noises: List[torch.Tensor], tabs: Dict[str, np.ndarray], kind: str, eps: bool,
                clip: bool, small: bool = False, eta: float = 0.0, record: Optional[list] = None) -> torch.Tensor:
    """p_sample_loop_progressive (reference models/gaussian_diffusion.py:937-983) or ddim_sample_loop_progressive
    (:1101-1147): x_T = noises[0], then per step the model on x_t at the mapped timestep (models/respace.py:60-63)
    and the step with noises[k + 1].  ``model(x, t_model)``; ``record`` receives (sample, pred_xstart) per step."""
    T = len(tabs["betas"])
    x = noises[0]
    for k, i in enumerate(range(T - 1, -1, -1)):
        t = torch.full((x.shape[0],), int(tabs["timestep_map"][i]), dtype=torch.long)
        out = model(x, t).float()
        if kind == "ddim":
            x, x0 = ddim_step(tabs, i, x, out, noises[k + 1], eps, clip, eta)
        else:
            x, x0 = ancestral_step(tabs, i, x, out, noises[k + 1], eps, clip, small)
        if record is not None:
            record.append((x, x0))
    return x
