"""Generate the KL first-stage fixtures under tests/golden/ by running the UNMODIFIED reference (build container only):

    python -m oracle.make_golden_kl

Imports the reference's own ``AutoencoderKLTorch`` (ldm/models/autoencoder.py), loads the deterministic synthetic
weights of ``resshift_b200.vq_arch.random_kl_state_dict`` strictly (names, shapes AND order are asserted against the
reference's ``state_dict``) and records the moments, ``mode()``, ``sample()`` under a recorded CPU seed, and the
decoded image.  Nothing here copies reference source.
"""
from __future__ import annotations

import json
import os
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
REF = Path(os.environ.get("RESSHIFT_REFERENCE", "/root/reference"))
GOLD = ROOT / "tests" / "golden"
SAMPLE_SEED = 97531


def main():
    sys.path.insert(0, str(ROOT / "oracle" / "_shims"))
    sys.path.insert(0, str(REF))
    sys.path.insert(0, str(ROOT))
    from ldm.models.autoencoder import AutoencoderKLTorch          # noqa: E402  (reference)
    from resshift_b200.vq_arch import kl_param_spec, kl_preset, random_kl_state_dict

    torch.set_grad_enabled(False)
    GOLD.mkdir(parents=True, exist_ok=True)

    inv = {}
    for name in ("tiny", "f8"):
        cfg = kl_preset(name)
        m = AutoencoderKLTorch(**cfg.to_kwargs())
        inv[name] = [[k, list(v.shape)] for k, v in m.state_dict().items()]
        assert [(k, tuple(s)) for k, s in inv[name]] == [(n, tuple(s)) for n, s, _ in kl_param_spec(cfg)]
    (GOLD / "kl_keys.json").write_text(json.dumps(inv))

    def fixture(name, batch, h, w, fname, seed=0):
        cfg = kl_preset(name)
        model = AutoencoderKLTorch(**cfg.to_kwargs()).eval()
        model.load_state_dict(random_kl_state_dict(cfg, seed), strict=True)
        g = torch.Generator().manual_seed(2468)
        x = torch.rand(batch, 3, h, w, generator=g) * 2 - 1
        mode, moments = model.encode(x, sample_posterior=False, return_moments=True)
        torch.manual_seed(SAMPLE_SEED)                               # sample() draws on the CPU default generator
        sample = model.encode(x, sample_posterior=True)
        noise = (sample - mode) / torch.exp(0.5 * torch.clamp(moments[:, cfg.embed_dim:], -30.0, 20.0))
        dec = model.decode(mode)
        np.savez_compressed(GOLD / fname, x=x.numpy(), moments=moments.numpy(), mode=mode.numpy(), sample=sample.numpy(),
                            sample_seed=np.int64(SAMPLE_SEED), dec=dec.numpy())
        torch.manual_seed(SAMPLE_SEED)
        assert torch.allclose(noise, torch.randn(mode.shape), atol=1e-3)
        print(fname, "moments std %.3f" % moments.std().item(), "dec std %.3f" % dec.std().item())

    fixture("tiny", 2, 64, 64, "kl_tiny.npz")
    fixture("f8", 1, 64, 96, "kl_f8.npz")


if __name__ == "__main__":
    main()
