"""Generate the fixtures of the first-stage Encoder / Decoder options under tests/golden/ by running the UNMODIFIED
reference (build container only):

    python -m oracle.make_golden_vq_options

Imports the reference's own ``VQModelTorch`` / ``AutoencoderKLTorch`` (ldm/models/autoencoder.py) built from ddconfigs
with level attention (``attn_resolutions``), ``attn_type: none``, ``resamp_with_conv: False``, ``tanh_out: True`` and a
non-zero ``dropout``; loads the deterministic synthetic weights of ``resshift_b200.vq_arch.random_*_state_dict``
strictly (names, shapes AND order are asserted against the reference's ``state_dict``) and records encode / decode
outputs of the models in eval mode.  Writes one ``vq_opt_*.npz`` per run (outputs only: the inputs come from
``inputs()``) and ``vq_keys_options.json``.
Nothing here copies reference source.
"""
from __future__ import annotations

import json
import os
import sys
from dataclasses import replace
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
REF = Path(os.environ.get("RESSHIFT_REFERENCE", "/root/reference"))
GOLD = ROOT / "tests" / "golden"


def configs():
    """name -> VQConfig of every case (fixtures and inventories); shared with tests/test_oracle_vq_options_golden.py."""
    from resshift_b200.vq_arch import kl_preset, ldm_vq_preset, vq_preset
    tiny = vq_preset("tiny")
    return {
        "levels": replace(tiny, attn_resolutions=(32, 16), dropout=0.1),
        "noattn_pool_tanh": replace(tiny, attn_type="none", resamp_with_conv=False, tanh_out=True),
        "kl_levels": replace(kl_preset("tiny"), attn_resolutions=(16,), resamp_with_conv=False),
        "ldm_f8": ldm_vq_preset("vq-f8"),
        "res90": replace(tiny, resolution=90, attn_resolutions=(45,)),      # encoder level 1 has attention, no decoder level
    }


# case -> [(batch, image H, image W, fixture file)] of each recorded run
RUNS = {"levels": [(2, 64, 64, "vq_opt_levels_64.npz"), (2, 96, 160, "vq_opt_levels_96x160.npz")],
        "noattn_pool_tanh": [(2, 64, 64, "vq_opt_noattn_pool_tanh.npz")],
        "kl_levels": [(2, 64, 64, "vq_opt_kl_levels.npz")],
        "ldm_f8": [(1, 64, 64, "vq_opt_ldm_f8.npz")]}


def inputs(name: str, r: int):
    """The image batch x and (VQ cases) the latent batch z of run r of case ``name``: drawn from a fixed CPU generator
    seed, so the fixtures store only outputs."""
    cfg = configs()[name]
    batch, hh, ww, _ = RUNS[name][r]
    g = torch.Generator().manual_seed(2468 + r)
    x = torch.rand(batch, 3, hh, ww, generator=g) * 2 - 1
    f = cfg.downscale
    z = None if cfg.kl else torch.randn(batch, cfg.embed_dim, hh // f, ww // f, generator=g) * 0.6
    return x, z


def main():
    sys.path.insert(0, str(ROOT / "oracle" / "_shims"))
    sys.path.insert(0, str(REF))
    sys.path.insert(0, str(ROOT))
    from ldm.models.autoencoder import AutoencoderKLTorch, VQModelTorch          # noqa: E402  (reference)
    from resshift_b200.vq_arch import kl_param_spec, random_kl_state_dict, random_vq_state_dict, vq_param_spec

    torch.set_grad_enabled(False)
    GOLD.mkdir(parents=True, exist_ok=True)

    def build(cfg):
        cls = AutoencoderKLTorch if cfg.kl else VQModelTorch
        return cls(**cfg.to_kwargs()).eval()

    inv = {}
    for name, cfg in configs().items():
        m = build(cfg)
        inv[name] = [[k, list(v.shape)] for k, v in m.state_dict().items()]
        spec = kl_param_spec(cfg) if cfg.kl else vq_param_spec(cfg)
        assert [(k, tuple(s)) for k, s in inv[name]] == [(n, tuple(s)) for n, s, _ in spec], name
    (GOLD / "vq_keys_options.json").write_text(json.dumps(inv))

    for name, runs in RUNS.items():
        cfg = configs()[name]
        model = build(cfg)
        model.load_state_dict((random_kl_state_dict if cfg.kl else random_vq_state_dict)(cfg, 0), strict=True)
        for r, (batch, hh, ww, fname) in enumerate(runs):
            x, z = inputs(name, r)
            if cfg.kl:
                # the mode is moments[:, :embed_dim] (DiagonalGaussianDistribution.mode)
                mode, moments = model.encode(x, sample_posterior=False, return_moments=True)
                assert torch.equal(mode, moments[:, :cfg.embed_dim])
                out = {"moments": moments.numpy(), "dec": model.decode(mode).numpy()}
            else:
                _, _, info = model.quantize(z)
                dec_nq = model.decode(z, force_not_quantize=True)
                # the quantised decode is the decoder on the chosen codes: pinned through the code map and dec_nq
                out = {"enc": model.encode(x).numpy(), "dec_nq": dec_nq.numpy(),
                       "idx": info[2].view(batch, hh // cfg.downscale, ww // cfg.downscale).numpy().astype(np.int16)}
            np.savez_compressed(GOLD / fname, **out)
            print(fname, {k: "%.3f" % float(np.std(v)) for k, v in out.items()})


if __name__ == "__main__":
    main()
