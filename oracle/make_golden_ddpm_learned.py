"""Golden fixtures of the reference's DDPM process with a learned variance (``create_gaussian_diffusion_ddpm(
learn_sigma=True)`` -> LEARNED_RANGE) on each UNet family with a 2 C output head, recorded by running the UNMODIFIED
reference (needs the reference tree):

    python -m oracle.make_golden_ddpm_learned

Writes ``tests/golden/ddpm_learned.npz`` and ``tests/golden/ddpm_learned_keys.json``.  The JSON is one file keyed by
case: each entry is the reference's ``state_dict`` inventory (names, shapes) of that case's model, so the three
families' 2 C-head inventories sit side by side (UNetModel twice, lq at the latent size and at twice it), rather than in
one file per family as the fixed-head fixtures keep them.  The npz holds:
  * per case, steps=1000, beta_start=0.0015, beta_end=0.0155 respaced to 8, batch 2, the inputs drawn from the case's
    seed (``case_inputs``), the loop noises fed through ``randn_like`` in draw order: ``<case>/final`` (the whole final
    sample), ``<case>/sample/<k>`` and ``<case>/pred_xstart/<k>`` (every step, sub-sampled by OUT_STRIDE):
      a  ancestral, eps, no clip, UNetModel ``lq2x`` with out_channels 6 (in 15: x has 3 channels, lq enters at twice
         the latent size)
      b  ancestral, x0, clip, UNetModelSwin ``tiny`` with out_channels 6
      c  DDIM eta = 0.5, eps, no clip, UNetModelConv ``defaults`` with out_channels 6
      d  DDIM inversion (``ddim_reverse_sample`` walked t = 0 .. T-1, as make_golden_ddim_reverse.py does), eps, no
         clip, UNetModel ``legacy`` with out_channels 6
The weights are ``random_state_dict`` (seed 0), loaded strictly.  Re-running reproduces both files bit for bit (CPU,
fixed seeds).
"""
from __future__ import annotations

import json

import numpy as np
import torch

from oracle.make_golden import GOLD, _import_reference
from oracle.make_golden_ddpm import BETA_END, BETA_START, STEPS

RESPACING = 8
OUT_STRIDE = 7
# case -> (model family, model case, loop, diffusion kwargs, clip, eta, seed)
CASES = {
    "a": ("unetmodel", "lq2x", "ancestral", dict(), False, 0.0, 920),
    "b": ("swin", "tiny", "ancestral", dict(predict_xstart=True), True, 0.0, 921),
    "c": ("unetconv", "defaults", "ddim", dict(), False, 0.5, 922),
    "d": ("unetmodel", "legacy", "reverse", dict(), False, 0.0, 923),
}


def diffusion_kwargs(case: str) -> dict:
    return dict(beta_start=BETA_START, beta_end=BETA_END, steps=STEPS, timestep_respacing=RESPACING, learn_sigma=True,
                **CASES[case][3])


def model_config(case: str):
    """(config, latent H, W) of a case's denoiser: its family's fixture model with the head widened to 2 C"""
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
    kw = ucfg.to_kwargs()
    kw["out_channels"] = 2 * ucfg.out_channels
    return type(ucfg)(**kw), hw


def case_inputs(case: str, batch: int = 2, channels: int = 3):
    """lq and the loop's inputs of a case, drawn on the CPU generator from its seed: the T + 1 noises (x_T first) of
    the forward loops, or x_start (a clean latent in [-1, 1]) of the inversion."""
    ucfg, hw = model_config(case)
    g = torch.Generator().manual_seed(CASES[case][6])
    f = getattr(ucfg, "lq_factor", 1)
    lq = torch.rand(batch, 3, hw[0] * f, hw[1] * f, generator=g) * 2 - 1
    if CASES[case][2] == "reverse":
        return lq, torch.rand(batch, channels, *hw, generator=g) * 2 - 1
    return lq, torch.stack([torch.randn(batch, channels, *hw, generator=g) for _ in range(RESPACING + 1)])


def main():
    from resshift_b200.weights import random_state_dict

    _import_reference()
    import models.gaussian_diffusion as gd                          # noqa: E402  (reference)
    from models.script_util import create_gaussian_diffusion_ddpm   # noqa: E402  (reference)
    from models.unet import UNetModel, UNetModelConv, UNetModelSwin  # noqa: E402  (reference)
    torch.set_grad_enabled(False)
    arrays, keys = {}, {}
    classes = {"unetmodel": UNetModel, "unetconv": UNetModelConv, "swin": UNetModelSwin}
    for case, (family, _, loop, _, clip, eta, _) in CASES.items():
        diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs(case))
        assert diff.model_var_type == gd.ModelVarTypeDDPM.LEARNED_RANGE
        T = diff.num_timesteps
        ucfg, _ = model_config(case)
        model = classes[family](**ucfg.to_kwargs()).eval()
        keys[case] = {k: list(v.shape) for k, v in model.state_dict().items()}
        model.load_state_dict(random_state_dict(ucfg, 0), strict=True)
        lq, inputs = case_inputs(case)
        if loop == "reverse":
            x, rec = inputs, []
            for i in range(T):
                out = diff.ddim_reverse_sample(model, x, torch.tensor([i] * x.shape[0]), clip_denoised=clip,
                                               denoised_fn=None, model_kwargs={"lq": lq})
                rec.append(out)
                x = out["sample"]
        else:
            queue = list(inputs[1:])
            orig = gd.th.randn_like
            gd.th.randn_like = lambda ref: queue.pop(0)
            try:
                kw = dict(noise=inputs[0], clip_denoised=clip, denoised_fn=None, model_kwargs={"lq": lq}, device="cpu")
                if loop == "ddim":
                    rec = list(diff.ddim_sample_loop_progressive(model, tuple(inputs[0].shape), eta=eta, **kw))
                else:
                    rec = list(diff.p_sample_loop_progressive(model, tuple(inputs[0].shape), **kw))
            finally:
                gd.th.randn_like = orig
            assert not queue
        assert len(rec) == T
        arrays[f"{case}/final"] = rec[-1]["sample"].numpy().copy()
        for k in range(T):
            arrays[f"{case}/sample/{k}"] = rec[k]["sample"].reshape(-1)[::OUT_STRIDE].numpy().copy()
            arrays[f"{case}/pred_xstart/{k}"] = rec[k]["pred_xstart"].reshape(-1)[::OUT_STRIDE].numpy().copy()
        print(case, family, loop, "T=%d final std %.4f max %.4f" % (T, rec[-1]["sample"].std().item(),
                                                                   rec[-1]["sample"].abs().max().item()))
    np.savez_compressed(GOLD / "ddpm_learned.npz", **arrays)
    (GOLD / "ddpm_learned_keys.json").write_text(json.dumps(keys, separators=(",", ":")))


if __name__ == "__main__":
    main()
