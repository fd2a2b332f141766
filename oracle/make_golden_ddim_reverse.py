"""Golden fixtures of DDIM inversion in the reference's DDPM process (``create_gaussian_diffusion_ddpm`` ->
``SpacedDiffusionDDPM.ddim_reverse_sample``), recorded by running the UNMODIFIED reference (needs the reference tree):

    python -m oracle.make_golden_ddim_reverse

The reference has the step only (models/gaussian_diffusion.py:1030-1066); this script walks it t = 0 .. T-1, each step
fed the previous step's ``sample``, the loop ``SpacedDiffusionDDPM.ddim_reverse_sample_loop`` of this package runs.
Writes ``tests/golden/ddim_reverse.npz``:
  * ``sig/ddim_reverse_sample``: ``inspect.signature`` of the reference's method;
  * per case, steps=1000, beta_start=0.0015, beta_end=0.0155 respaced to 8, batch 2, x_start and lq drawn from the
    case's seed (``case_inputs``): ``<case>/final`` (the whole x_T), ``<case>/sample/<k>`` and
    ``<case>/pred_xstart/<k>`` (every step, sub-sampled by OUT_STRIDE):
      a  eps, no clip, UNetModel ``legacy``
      b  x0, clip, UNetModelSwin ``tiny``
      c  eps, clip, UNetModelConv ``defaults``
      d  x0, no clip, UNetModel ``legacy``
      e  learn_sigma=True (LEARNED_RANGE) with make_golden_ddpm's ``learned_range_model``, eps, no clip: the torch
         route only (the native UNets refuse a 2 C head); every step whole
The weights are ``random_state_dict`` (seed 0), loaded strictly.  Re-running reproduces the file bit for bit (CPU,
fixed seeds).
"""
from __future__ import annotations

import inspect

import numpy as np
import torch

from oracle.make_golden import GOLD, _import_reference
from oracle.make_golden_ddpm import BETA_END, BETA_START, STEPS, learned_range_model

RESPACING = 8
OUT_STRIDE = 7
# case -> (model family, model case, diffusion kwargs, clip, seed)
CASES = {
    "a": ("unetmodel", "legacy", dict(), False, 910),
    "b": ("swin", "tiny", dict(predict_xstart=True), True, 911),
    "c": ("unetconv", "defaults", dict(), True, 912),
    "d": ("unetmodel", "legacy", dict(predict_xstart=True), False, 913),
    "e": ("callable", None, dict(learn_sigma=True), False, 914),
}
FUSED = ("a", "b", "c", "d")


def diffusion_kwargs(case: str) -> dict:
    return dict(beta_start=BETA_START, beta_end=BETA_END, steps=STEPS, timestep_respacing=RESPACING, **CASES[case][2])


def model_config(case: str):
    """(config, latent H, W) of a case's denoiser"""
    family, name = CASES[case][:2]
    if family == "unetmodel":
        from oracle.make_golden_unetmodel import case_config
        ucfg, _, hw = case_config(name)
    elif family == "unetconv":
        from oracle.make_golden_unetconv import case_config
        ucfg, _, hw = case_config(name)
    else:
        from resshift_b200.config import preset
        ucfg, _ = preset(name)
        hw = (64, 64)
    return ucfg, hw


def case_hw(case: str):
    return (16, 16) if CASES[case][0] == "callable" else model_config(case)[1]


def case_inputs(case: str, batch: int = 2, channels: int = 3):
    """lq and x_start (a clean latent in [-1, 1]) of a case, drawn on the CPU generator from its seed."""
    hw = case_hw(case)
    g = torch.Generator().manual_seed(CASES[case][4])
    lq = torch.rand(batch, 3, *hw, generator=g) * 2 - 1
    x_start = torch.rand(batch, channels, *hw, generator=g) * 2 - 1
    return lq, x_start


def main():
    from resshift_b200.weights import random_state_dict

    _import_reference()
    from models.script_util import create_gaussian_diffusion_ddpm   # noqa: E402  (reference)
    from models.respace import SpacedDiffusionDDPM                  # noqa: E402  (reference)
    from models.unet import UNetModel, UNetModelConv, UNetModelSwin  # noqa: E402  (reference)
    torch.set_grad_enabled(False)
    arrays = {"sig/ddim_reverse_sample": np.array(str(inspect.signature(SpacedDiffusionDDPM.ddim_reverse_sample)))}
    classes = {"unetmodel": UNetModel, "unetconv": UNetModelConv, "swin": UNetModelSwin}
    for case, (family, _, _, clip, _) in CASES.items():
        diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs(case))
        T = diff.num_timesteps
        if family == "callable":
            model = learned_range_model
        else:
            ucfg, _ = model_config(case)
            model = classes[family](**ucfg.to_kwargs()).eval()
            model.load_state_dict(random_state_dict(ucfg, 0), strict=True)
        lq, x = case_inputs(case)
        rec = []
        for i in range(T):
            t = torch.tensor([i] * x.shape[0])
            out = diff.ddim_reverse_sample(model, x, t, clip_denoised=clip, denoised_fn=None, model_kwargs={"lq": lq})
            rec.append(out)
            x = out["sample"]
        arrays[f"{case}/final"] = rec[-1]["sample"].numpy().copy()
        stride = 1 if family == "callable" else OUT_STRIDE
        for k in range(T):
            arrays[f"{case}/sample/{k}"] = rec[k]["sample"].reshape(-1)[::stride].numpy().copy()
            arrays[f"{case}/pred_xstart/{k}"] = rec[k]["pred_xstart"].reshape(-1)[::stride].numpy().copy()
        print(case, "T=%d x_T std %.4f max %.4f" % (T, rec[-1]["sample"].std().item(),
                                                  rec[-1]["sample"].abs().max().item()))
    np.savez_compressed(GOLD / "ddim_reverse.npz", **arrays)


if __name__ == "__main__":
    main()
