"""Golden fixtures of the UNetModelSwin constructor options the shipped yaml files leave at one value, recorded by
running the UNMODIFIED reference (like ``oracle/make_golden.py``; needs /root/reference):

    python -m oracle.make_golden_variants

Writes ``tests/golden/unet_variants.npz`` and ``tests/golden/unet_keys_variants.json``:
  * per variant: the reference's ``state_dict`` inventory (names, shapes);
  * per variant: one forward at batch 2 with two different timesteps (x, lq, mask re-drawn from the stored seed by
    ``variant_inputs``), its output and block probes, sub-sampled;
  * the combined variant at a 64x128 latent;
  * the combined variant's ``p_sample_loop_progressive`` trajectory (T = 4).
The weights are ``resshift_b200.weights.random_state_dict``, loaded strictly.  Re-running reproduces the files bit for
bit (CPU, fixed seeds).
"""
from __future__ import annotations

import json

import numpy as np
import torch

from oracle.make_golden import GOLD, _import_reference

# name -> UNetConfig overrides on the tiny width (model_channels 32, swin_embed_dim 64)
VARIANTS = {
    "scale_shift_off": dict(use_scale_shift_norm=False),
    "updown": dict(resblock_updown=True),
    "pooled": dict(conv_resample=False),
    "patch_norm": dict(patch_norm=True),
    "mask_latent": dict(cond_mask=True, lq_size=64),
    "combined": dict(use_scale_shift_norm=False, resblock_updown=True, patch_norm=True, dropout=0.1),
}
OUT_STRIDE, PROBE_STRIDE = 7, 401
TIMESTEPS = (3, 1)


def variant_config(name: str):
    from resshift_b200.config import DiffusionConfig, UNetConfig
    return UNetConfig(model_channels=32, swin_embed_dim=64, **VARIANTS[name]), DiffusionConfig(steps=4, min_noise_level=0.2, sf=1)


def variant_inputs(cfg, batch: int, h: int, w: int, seed: int):
    """x, lq, mask (or None) of a fixture, drawn on the CPU generator."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(batch, cfg.in_channels, h, w, generator=g)
    lq = torch.rand(batch, 3, h << cfg.fe_stages, w << cfg.fe_stages, generator=g) * 2 - 1
    mask = None
    if cfg.cond_mask:
        mask = -torch.ones(batch, 1, h << cfg.fe_stages, w << cfg.fe_stages)
        mask[:, :, mask.shape[2] // 4: mask.shape[2] // 4 * 3, mask.shape[3] // 8: mask.shape[3] // 2] = 1.0
    return x, lq, mask


def trajectory_inputs(batch: int, T: int, seed: int = 777):
    """y and the T + 1 loop noises of the combined variant's trajectory."""
    g = torch.Generator().manual_seed(seed)
    y = torch.rand(batch, 3, 64, 64, generator=g) * 2 - 1
    noises = torch.stack([torch.randn(batch, 3, 64, 64, generator=g) for _ in range(T + 1)])
    return y, noises


def main():
    from resshift_b200.weights import random_state_dict

    UNetModelSwin, create_gaussian_diffusion, gd = _import_reference()
    torch.set_grad_enabled(False)
    arrays, keys = {}, {}

    def build(name):
        ucfg, dcfg = variant_config(name)
        model = UNetModelSwin(**ucfg.to_kwargs()).eval()
        keys[name] = {k: list(v.shape) for k, v in model.state_dict().items()}
        model.load_state_dict(random_state_dict(ucfg, 0), strict=True)
        return ucfg, dcfg, model

    def forward(tag, name, ucfg, model, hw, seed):
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

    for i, name in enumerate(VARIANTS):
        ucfg, dcfg, model = build(name)
        forward(name, name, ucfg, model, (64, 64), 100 + i)
        if name == "combined":
            forward("combined_64x128", name, ucfg, model, (64, 128), 200)
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

    np.savez_compressed(GOLD / "unet_variants.npz", **arrays)
    (GOLD / "unet_keys_variants.json").write_text(json.dumps(keys, separators=(",", ":")))


class _IdentityAE(torch.nn.Module):
    """Stand-in first stage (see make_golden.py): the loop under test is the latent-space loop."""
    def __init__(self):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1))

    def encode(self, x):
        return x

    def decode(self, x):
        return x


if __name__ == "__main__":
    main()
