"""Golden fixtures of the reference's ``UNetModelConv``, recorded by running the UNMODIFIED reference
``models.unet.UNetModelConv`` (like ``oracle/make_golden_unetmodel.py``; needs the reference tree):

    python -m oracle.make_golden_unetconv

Writes ``tests/golden/unetconv.npz`` and ``tests/golden/unet_keys_unetconv.json``:
  * per case: the reference's ``state_dict`` inventory (names, shapes);
  * per case: one forward at batch 2 with two different timesteps (x, lq re-drawn from the stored seed by
    ``case_inputs``), its output and block probes, sub-sampled;
  * the ``p_sample_loop_progressive`` trajectory (T = 4) of case ``defaults``.
The weights are ``resshift_b200.weights.random_state_dict``, loaded strictly: every tensor is drawn, so the
``out_layers.1`` convs the reference zero-initialises are random too.  Re-running reproduces the files bit for bit
(CPU, fixed seeds).
"""
from __future__ import annotations

import json

import numpy as np
import torch

from oracle.make_golden import GOLD, _import_reference
from oracle.make_golden_variants import _IdentityAE

_BASE = dict(in_channels=6, model_channels=32, out_channels=3, num_res_blocks=1, channel_mult=(1, 2, 2))
# name -> (UNetModelConvConfig kwargs, latent H, W); tiny widths keep tests/golden small
CASES = {
    # (a) the constructor defaults: no scale-shift, conv resampling
    "defaults": (dict(_BASE), 32, 32),
    # (b) scale-shift (FiLM after the SiLU), ResBlockConv down / up, pooled resampling inside them
    "ss_updown": (dict(_BASE, use_scale_shift_norm=True, resblock_updown=True, conv_resample=False), 32, 32),
    # (c) lq at twice the latent size: pixel_unshuffle(lq, 2) -> 12 channels; pooled / nearest Downsample / Upsample
    "lq2x": (dict(_BASE, in_channels=15, conv_resample=False), 32, 32),
    # (d) uneven num_res_blocks (channel changes through 1x1 skips) on a non-square latent
    "uneven": (dict(_BASE, num_res_blocks=(2, 1, 0), channel_mult=(1, 2, 3)), 24, 40),
}
OUT_STRIDE, PROBE_STRIDE = 7, 401
TIMESTEPS = (3, 1)
SEEDS = {"defaults": 500, "ss_updown": 501, "lq2x": 502, "uneven": 503}


def case_config(name: str):
    from resshift_b200.config import DiffusionConfig, UNetModelConvConfig
    kw, h, w = CASES[name]
    return UNetModelConvConfig(**kw), DiffusionConfig(steps=4, min_noise_level=0.2, sf=1), (h, w)


def case_inputs(cfg, batch: int, h: int, w: int, seed: int):
    """x, lq of a fixture, drawn on the CPU generator."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(batch, cfg.out_channels, h, w, generator=g)
    f = cfg.lq_factor
    lq = torch.rand(batch, 3, h * f, w * f, generator=g) * 2 - 1
    return x, lq


def trajectory_inputs(batch: int, T: int, hw=(32, 32), seed: int = 779):
    """y and the T + 1 loop noises of the trajectory of case ``defaults``."""
    g = torch.Generator().manual_seed(seed)
    y = torch.rand(batch, 3, *hw, generator=g) * 2 - 1
    noises = torch.stack([torch.randn(batch, 3, *hw, generator=g) for _ in range(T + 1)])
    return y, noises


def main():
    from resshift_b200.weights import random_state_dict

    _, create_gaussian_diffusion, gd = _import_reference()
    from models.unet import UNetModelConv      # noqa: E402  (reference)
    torch.set_grad_enabled(False)
    arrays, keys = {}, {}
    for name in CASES:
        ucfg, dcfg, (h, w) = case_config(name)
        kw = ucfg.to_kwargs()
        model = UNetModelConv(**kw).eval()
        keys[name] = {k: list(v.shape) for k, v in model.state_dict().items()}
        model.load_state_dict(random_state_dict(ucfg, 0), strict=True)
        x, lq = case_inputs(ucfg, 2, h, w, SEEDS[name])
        probes, hooks = {}, []
        blocks = [(f"input_blocks.{i}", m) for i, m in enumerate(model.input_blocks)] + [("middle_block", model.middle_block)]
        blocks += [(f"output_blocks.{i}", m) for i, m in enumerate(model.output_blocks)]
        for k, m in blocks:
            hooks.append(m.register_forward_hook(lambda _m, _i, o, k=k: probes.__setitem__(k, o)))
        out = model(x, torch.tensor(TIMESTEPS), lq=lq)
        for hk in hooks:
            hk.remove()
        arrays[f"{name}/seed"] = np.array([SEEDS[name], h, w], dtype=np.int64)
        arrays[f"{name}/t"] = np.array(TIMESTEPS, dtype=np.int64)
        arrays[f"{name}/out_sub"] = out.reshape(-1)[::OUT_STRIDE].numpy().copy()
        for k, v in probes.items():
            arrays[f"{name}/probe_sub/{k}"] = v.reshape(-1)[::PROBE_STRIDE].numpy().copy()
        print(name, "out std %.4f" % out.std().item())
        if name == "defaults":
            diff = create_gaussian_diffusion(**dcfg.to_kwargs())
            T = diff.num_timesteps
            y, noises = trajectory_inputs(2, T)
            queue = list(noises[1:])
            orig = gd.th.randn_like
            gd.th.randn_like = lambda ref: queue.pop(0)
            try:
                rec = list(diff.p_sample_loop_progressive(
                    y, model, first_stage_model=_IdentityAE(), noise=noises[0], noise_repeat=False,
                    clip_denoised=False, denoised_fn=None, model_kwargs={"lq": y}, device="cpu"))
            finally:
                gd.th.randn_like = orig
            arrays["loop/final_sub"] = rec[-1]["sample"].reshape(-1)[::OUT_STRIDE].numpy().copy()
            for k in range(T):
                arrays[f"loop/pred_xstart/{k}"] = rec[k]["pred_xstart"].reshape(-1)[::OUT_STRIDE].numpy().copy()
            print("loop T=%d final std %.4f" % (T, rec[-1]["sample"].std().item()))

    np.savez_compressed(GOLD / "unetconv.npz", **arrays)
    (GOLD / "unet_keys_unetconv.json").write_text(json.dumps(keys, separators=(",", ":")))


if __name__ == "__main__":
    main()
