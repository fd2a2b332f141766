"""Golden trajectories of the reference's other ``predict_type``s and input scalings, recorded by running the UNMODIFIED
reference's ``p_sample_loop_progressive`` (like ``oracle/make_golden_variants.py``; needs the reference tree):

    python -m oracle.make_golden_predict_types

Writes ``tests/golden/loop_predict_types.npz``: per case (``CASES``), the trajectory at T = 4, batch 2, with the
identity first stage and ``clip_denoised=False`` (y and the T + 1 noises re-drawn from the stored seed by
``trajectory_inputs``), sub-sampled with stride ``STRIDE``: every step's pred_xstart and sample, and the final sample.
The weights are ``resshift_b200.weights.random_state_dict``, loaded strictly.  Re-running reproduces the file bit for
bit (CPU, fixed seeds).

The epsilon cases end their schedule at sqrt_eta = ``EPS_ETAS_END`` instead of the shipped 0.99.  An epsilon model's
output enters x0 multiplied by kappa sqrt_eta_t / (1 - eta_t) (epsilon) or 1 / (1 - eta_t) (epsilon_scale): about 100 at
the first step of the shipped schedule (kappa 2), where a random-weight model, which has not learnt to predict the
noise, would throw x0 to |x| ~ 100 and make the trajectory say nothing.  At 0.5 both factors are at most 4/3
(2 * 0.5 / 0.75 and 1 / 0.75), and the recorded trajectories stay O(1): final std 2.0 to 2.5 and max |x| under 14,
against 0.6 to 0.9 and 6.6 for the xstart and residual cases (the generator prints both).
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.make_golden import GOLD, _import_reference
from oracle.make_golden_variants import _IdentityAE

EPS_ETAS_END = 0.5
STRIDE = 11
# name -> (model family, DiffusionConfig overrides)
CASES = {
    "swin_epsilon": ("swin", dict(predict_type="epsilon", etas_end=EPS_ETAS_END)),
    "swin_epsilon_scale": ("swin", dict(predict_type="epsilon_scale", etas_end=EPS_ETAS_END)),
    "swin_residual": ("swin", dict(predict_type="residual")),
    "swin_xstart_latent_flag_off": ("swin", dict(latent_flag=False)),
    "swin_xstart_normalize_off": ("swin", dict(normalize_input=False)),
    "unetmodel_epsilon": ("unetmodel", dict(predict_type="epsilon", etas_end=EPS_ETAS_END)),
}
SEEDS = {name: 900 + i for i, name in enumerate(CASES)}


def case_config(name: str):
    """(model config, DiffusionConfig, latent (H, W)) of a case: the tiny-width UNetModelSwin or the ``legacy``
    UNetModel of oracle/make_golden_unetmodel.py, T = 4, sf = 1."""
    from resshift_b200.config import DiffusionConfig, UNetConfig
    family, over = CASES[name]
    dcfg = DiffusionConfig(steps=4, min_noise_level=0.2, sf=1, **over)
    if family == "swin":
        return UNetConfig(model_channels=32, swin_embed_dim=64), dcfg, (64, 64)
    from oracle.make_golden_unetmodel import case_config as um_config
    ucfg, _, hw = um_config("legacy")
    return ucfg, dcfg, hw


def trajectory_inputs(name: str, batch: int = 2):
    """y and the T + 1 loop noises of a case, drawn on the CPU generator."""
    _, dcfg, hw = case_config(name)
    g = torch.Generator().manual_seed(SEEDS[name])
    y = torch.rand(batch, 3, *hw, generator=g) * 2 - 1
    noises = torch.stack([torch.randn(batch, 3, *hw, generator=g) for _ in range(dcfg.steps + 1)])
    return y, noises


def main():
    from resshift_b200.weights import random_state_dict

    UNetModelSwin, create_gaussian_diffusion, gd = _import_reference()
    from models.unet import UNetModel                            # noqa: E402  (reference)
    torch.set_grad_enabled(False)
    arrays = {}
    for name, (family, _) in CASES.items():
        ucfg, dcfg, _ = case_config(name)
        model = (UNetModelSwin if family == "swin" else UNetModel)(**ucfg.to_kwargs()).eval()
        model.load_state_dict(random_state_dict(ucfg, 0), strict=True)
        diff = create_gaussian_diffusion(**dcfg.to_kwargs())
        T = diff.num_timesteps
        y, noises = trajectory_inputs(name)
        queue = list(noises[1:])
        orig = gd.th.randn_like
        gd.th.randn_like = lambda ref: queue.pop(0)
        try:
            rec = list(diff.p_sample_loop_progressive(
                y, model, first_stage_model=_IdentityAE(), noise=noises[0], noise_repeat=False,
                clip_denoised=False, denoised_fn=None, model_kwargs={"lq": y}, device="cpu"))
        finally:
            gd.th.randn_like = orig
        assert not queue
        arrays[f"{name}/final_sub"] = rec[-1]["sample"].reshape(-1)[::STRIDE].numpy().copy()
        for k in range(T):
            arrays[f"{name}/pred_xstart/{k}"] = rec[k]["pred_xstart"].reshape(-1)[::STRIDE].numpy().copy()
            arrays[f"{name}/sample/{k}"] = rec[k]["sample"].reshape(-1)[::STRIDE].numpy().copy()
        amax = max(max(r["sample"].abs().max().item(), r["pred_xstart"].abs().max().item()) for r in rec)
        print(f"{name}: T={T} final std {rec[-1]['sample'].std().item():.4f} max |x| {amax:.3f}")
    np.savez_compressed(GOLD / "loop_predict_types.npz", **arrays)


if __name__ == "__main__":
    main()
