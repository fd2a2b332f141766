"""Golden fixtures of UNetModelSwin built with 16x16 windows and / or 64-wide heads, recorded by running the UNMODIFIED
reference (like ``oracle/make_golden_variants.py``; needs the reference tree):

    python -m oracle.make_golden_windows

Writes ``tests/golden/unet_windows.npz`` and ``tests/golden/unet_keys_windows.json``:
  * per model: the reference's ``state_dict`` inventory (names, shapes);
  * per model: one forward at batch 2 with two different timesteps (inputs re-drawn from the stored seed by
    ``make_golden_variants.variant_inputs``), its output and block probes, sub-sampled;
  * the window 16 / head 64 model at a 64x128 latent and its ``p_sample_loop_progressive`` trajectory (T = 4);
  * the reference's shift masks for 16x16 windows: the ``attn_mask`` buffers of the 64x64 and 32x32 levels and a
    ``calculate_mask`` call for a 64x128 map, as int8 (0 / 1 = masked), exact.
The weights are ``resshift_b200.weights.random_state_dict``, loaded strictly.  Re-running reproduces the files bit for
bit (CPU, fixed seeds).
"""
from __future__ import annotations

import json

import numpy as np
import torch

from oracle.make_golden import GOLD, _import_reference
from oracle.make_golden_variants import OUT_STRIDE, PROBE_STRIDE, TIMESTEPS, _IdentityAE, trajectory_inputs, variant_inputs

# name -> UNetConfig overrides on the tiny width (model_channels 32; swin_embed_dim 64 unless given)
WINDOWS = {
    "w16_h32": dict(window_size=16),                                       # 2 heads of 32
    "w8_h64": dict(num_head_channels=64),                                  # 1 head of 64
    "w16_h64": dict(window_size=16, num_head_channels=64, swin_embed_dim=128),   # 2 heads of 64
    "w16_h64_variant": dict(window_size=16, num_head_channels=64, swin_embed_dim=128, use_scale_shift_norm=False,
                            patch_norm=True),
}
LOOP_MODEL = "w16_h64"


def windows_config(name: str):
    from resshift_b200.config import DiffusionConfig, UNetConfig
    kw = dict(model_channels=32, swin_embed_dim=64)
    kw.update(WINDOWS[name])
    return UNetConfig(**kw), DiffusionConfig(steps=4, min_noise_level=0.2, sf=1)


def main():
    from resshift_b200.weights import random_state_dict

    UNetModelSwin, create_gaussian_diffusion, gd = _import_reference()
    torch.set_grad_enabled(False)
    arrays, keys = {}, {}

    def forward(tag, ucfg, model, hw, seed):
        x, lq, mask = variant_inputs(ucfg, 2, hw[0], hw[1], seed)
        probes, hooks = {}, []
        blocks = [(f"input_blocks.{i}", m) for i, m in enumerate(model.input_blocks)] + [("middle_block", model.middle_block)]
        blocks += [(f"output_blocks.{i}", m) for i, m in enumerate(model.output_blocks)]
        for k, m in blocks:
            hooks.append(m.register_forward_hook(lambda _m, _i, o, k=k: probes.__setitem__(k, o)))
        out = model(x, torch.tensor(TIMESTEPS), lq=lq, mask=mask)
        for h in hooks:
            h.remove()
        arrays[f"{tag}/seed"] = np.array([seed, hw[0], hw[1]], dtype=np.int64)
        arrays[f"{tag}/t"] = np.array(TIMESTEPS, dtype=np.int64)
        arrays[f"{tag}/out_sub"] = out.reshape(-1)[::OUT_STRIDE].numpy().copy()
        for k, v in probes.items():
            arrays[f"{tag}/probe_sub/{k}"] = v.reshape(-1)[::PROBE_STRIDE].numpy().copy()
        print(tag, "out std %.4f" % out.std().item())

    for i, name in enumerate(WINDOWS):
        ucfg, dcfg = windows_config(name)
        model = UNetModelSwin(**ucfg.to_kwargs()).eval()
        keys[name] = {k: list(v.shape) for k, v in model.state_dict().items()}
        model.load_state_dict(random_state_dict(ucfg, 0), strict=True)
        forward(name, ucfg, model, (64, 64), 300 + i)
        if name != LOOP_MODEL:
            continue
        forward(f"{name}_64x128", ucfg, model, (64, 128), 400)
        # shift masks of the shifted blocks: the 64x64 level (input_blocks.1), the 32x32 level (input_blocks.4), and the
        # 64x64 level's block asked for a 64x128 map
        b64, b32 = model.input_blocks[1][1].blocks[1], model.input_blocks[4][1].blocks[1]
        for tag, m in (("64x64", b64.attn_mask), ("32x32", b32.attn_mask), ("64x128", b64.calculate_mask((64, 128)))):
            assert set(m.unique().tolist()) <= {0.0, -100.0}
            arrays[f"mask/{tag}"] = (m != 0).numpy().astype(np.int8)
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
        print("loop T=%d final std %.4f" % (T, rec[-1]["sample"].std().item()))

    np.savez_compressed(GOLD / "unet_windows.npz", **arrays)
    (GOLD / "unet_keys_windows.json").write_text(json.dumps(keys, separators=(",", ":")))


if __name__ == "__main__":
    main()
