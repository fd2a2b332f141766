"""Golden fixtures of the reference's DDPM / DDIM process (``create_gaussian_diffusion_ddpm`` ->
``SpacedDiffusionDDPM``), recorded by running the UNMODIFIED reference (needs the reference tree):

    python -m oracle.make_golden_ddpm

Writes ``tests/golden/ddpm.npz``:
  * ``tab/<respacing>/<name>``: every float64 table and ``timestep_map`` of steps=1000, beta_start=0.0015,
    beta_end=0.0155, respaced to 8 and 80 and not respaced ("1000");
  * ``sig/<name>``: ``inspect.signature`` of create_gaussian_diffusion_ddpm, p_sample_loop and ddim_sample_loop;
  * trajectories respaced to 8, batch 2, the loop noises drawn from each case's seed (``case_inputs``) and fed through
    ``randn_like`` in draw order: ``<case>/final`` (the whole final sample), ``<case>/sample/<k>`` and
    ``<case>/pred_xstart/<k>`` (every step, sub-sampled by OUT_STRIDE):
      a  ancestral, eps, FIXED_LARGE, no clip, UNetModel ``legacy``; ``a/decoded``: its final sample decoded by the
         tiny VQ-GAN (p_sample_loop's first_stage_model)
      b  ancestral, x0, FIXED_SMALL, clip, UNetModelSwin ``tiny``
      c  DDIM eta = 0, eps, clip, UNetModelConv ``defaults``
      d  DDIM eta = 1, eps, no clip, UNetModel ``legacy``
  * generic-route cases:
      e  respaced to 80 (above the fused loop's 64 steps), ancestral, eps, FIXED_LARGE, clip, ``legacy``: the final
         sample and steps E_STEPS
      f  learn_sigma=True (LEARNED_RANGE) with ``learned_range_model``, ancestral, eps, no clip: every step whole
The weights are ``random_state_dict`` / ``random_vq_state_dict`` (seed 0), loaded strictly.  Re-running reproduces the
file bit for bit (CPU, fixed seeds).
"""
from __future__ import annotations

import inspect

import numpy as np
import torch

from oracle.make_golden import GOLD, _import_reference

STEPS, BETA_START, BETA_END = 1000, 0.0015, 0.0155
RESPACINGS = (8, 80, None)
OUT_STRIDE = 7
E_STEPS = (0, 40, 79)
TABLES = ("betas", "alphas_cumprod", "alphas_cumprod_prev", "alphas_cumprod_next", "sqrt_alphas_cumprod",
          "sqrt_one_minus_alphas_cumprod", "log_one_minus_alphas_cumprod", "sqrt_recip_alphas_cumprod",
          "sqrt_recipm1_alphas_cumprod", "posterior_variance", "posterior_log_variance_clipped", "posterior_mean_coef1",
          "posterior_mean_coef2")
SIGNATURES = ("create_gaussian_diffusion_ddpm", "p_sample_loop", "ddim_sample_loop")
# case -> (model family, model case, respacing, loop, diffusion kwargs, clip, eta, seed)
CASES = {
    "a": ("unetmodel", "legacy", 8, "ancestral", dict(), False, 0.0, 900),
    "b": ("swin", "tiny", 8, "ancestral", dict(predict_xstart=True, sigma_small=True), True, 0.0, 901),
    "c": ("unetconv", "defaults", 8, "ddim", dict(), True, 0.0, 902),
    "d": ("unetmodel", "legacy", 8, "ddim", dict(), False, 1.0, 903),
    "e": ("unetmodel", "legacy", 80, "ancestral", dict(), True, 0.0, 904),
    "f": ("callable", None, 8, "ancestral", dict(learn_sigma=True), False, 0.0, 905),
}
FUSED = ("a", "b", "c", "d")


def diffusion_kwargs(case: str) -> dict:
    _, _, respacing, _, kw, _, _, _ = CASES[case]
    return dict(beta_start=BETA_START, beta_end=BETA_END, steps=STEPS, timestep_respacing=respacing, **kw)


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


def case_inputs(case: str, batch: int = 2, channels: int = 3, hw=(32, 32), lq_hw=None):
    """lq and the T + 1 loop noises of a case, drawn on the CPU generator from its seed."""
    respacing, seed = CASES[case][2], CASES[case][7]
    g = torch.Generator().manual_seed(seed)
    lq = torch.rand(batch, 3, *(lq_hw or hw), generator=g) * 2 - 1
    noises = torch.stack([torch.randn(batch, channels, *hw, generator=g) for _ in range(respacing + 1)])
    return lq, noises


def learned_range_model(x, t, **kwargs):
    """A fixed denoiser with a learned-range variance head (2 C output channels): eps = 0.3 tanh(x) + 1e-4 t, and
    variance values in [-1, 1] that vary with x and t."""
    tt = t.to(x.dtype).view(-1, 1, 1, 1)
    eps = 0.3 * torch.tanh(x) + 1e-4 * tt
    var = torch.sin(0.7 * x + 0.01 * tt)
    return torch.cat([eps, var], dim=1)


def main():
    from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
    from resshift_b200.weights import random_state_dict

    _import_reference()
    import models.gaussian_diffusion as gd                          # noqa: E402  (reference)
    from models.script_util import create_gaussian_diffusion_ddpm   # noqa: E402  (reference)
    from models.respace import SpacedDiffusionDDPM                  # noqa: E402  (reference)
    from models.unet import UNetModel, UNetModelConv, UNetModelSwin  # noqa: E402  (reference)
    from ldm.models.autoencoder import VQModelTorch                 # noqa: E402  (reference)
    torch.set_grad_enabled(False)
    arrays = {}
    for r in RESPACINGS:
        diff = create_gaussian_diffusion_ddpm(beta_start=BETA_START, beta_end=BETA_END, steps=STEPS, timestep_respacing=r)
        key = str(r or STEPS)
        for name in TABLES:
            arrays[f"tab/{key}/{name}"] = np.asarray(getattr(diff, name), dtype=np.float64)
        arrays[f"tab/{key}/timestep_map"] = np.array(diff.timestep_map, dtype=np.int64)
    for name, fn in zip(SIGNATURES, (create_gaussian_diffusion_ddpm, SpacedDiffusionDDPM.p_sample_loop,
                                     SpacedDiffusionDDPM.ddim_sample_loop)):
        arrays[f"sig/{name}"] = np.array(str(inspect.signature(fn)))

    classes = {"unetmodel": UNetModel, "unetconv": UNetModelConv, "swin": UNetModelSwin}
    for case, (family, _, respacing, loop, _, clip, eta, _) in CASES.items():
        diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs(case))
        T = diff.num_timesteps
        if family == "callable":
            model, hw = learned_range_model, (16, 16)
        else:
            ucfg, hw = model_config(case)
            model = classes[family](**ucfg.to_kwargs()).eval()
            model.load_state_dict(random_state_dict(ucfg, 0), strict=True)
        lq, noises = case_inputs(case, hw=hw)
        queue = list(noises[1:])
        orig = gd.th.randn_like
        gd.th.randn_like = lambda ref: queue.pop(0)
        try:
            kw = dict(noise=noises[0], clip_denoised=clip, denoised_fn=None, model_kwargs={"lq": lq}, device="cpu")
            if loop == "ddim":
                rec = list(diff.ddim_sample_loop_progressive(model, tuple(noises[0].shape), eta=eta, **kw))
            else:
                rec = list(diff.p_sample_loop_progressive(model, tuple(noises[0].shape), **kw))
        finally:
            gd.th.randn_like = orig
        assert not queue and len(rec) == T
        arrays[f"{case}/final"] = rec[-1]["sample"].numpy().copy()
        steps = E_STEPS if case == "e" else range(T)
        stride = 1 if case == "f" else OUT_STRIDE
        for k in steps:
            arrays[f"{case}/sample/{k}"] = rec[k]["sample"].reshape(-1)[::stride].numpy().copy()
            arrays[f"{case}/pred_xstart/{k}"] = rec[k]["pred_xstart"].reshape(-1)[::stride].numpy().copy()
        if case == "a":
            vcfg = vq_preset("tiny")
            vq = VQModelTorch(**vcfg.to_kwargs()).eval()
            vq.load_state_dict(random_vq_state_dict(vcfg, 0), strict=True)
            dec = diff.decode_first_stage(rec[-1]["sample"], vq)
            arrays["a/decoded"] = dec.reshape(-1)[::OUT_STRIDE].numpy().copy()
        print(case, loop, "T=%d final std %.4f max %.4f" % (T, rec[-1]["sample"].std().item(),
                                                          rec[-1]["sample"].abs().max().item()))
    np.savez_compressed(GOLD / "ddpm.npz", **arrays)


if __name__ == "__main__":
    main()
