"""Generate the wide-latent first-stage fixtures under tests/golden/ by running the UNMODIFIED reference (build container
only):

    python -m oracle.make_golden_wide_latents

Imports the reference's own ``AutoencoderKLTorch`` and ``VQModelTorch`` (ldm/models/autoencoder.py), loads the
deterministic synthetic weights of ``resshift_b200.vq_arch.random_kl_state_dict`` / ``random_vq_state_dict`` strictly
(names, shapes AND order are asserted against the reference's ``state_dict``) for the "tiny" topology with 16- and
64-channel latents, and records the KL moments, ``mode()``, ``sample()`` under a recorded CPU seed and the decoded
image, and the VQ encode, code indices and decode.  Also lists the state_dict inventories of LDM's kl-f16 and kl-f32.
Nothing here copies reference source.
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
SAMPLE_SEED = 97533


def main():
    sys.path.insert(0, str(ROOT / "oracle" / "_shims"))
    sys.path.insert(0, str(REF))
    sys.path.insert(0, str(ROOT))
    from ldm.models.autoencoder import AutoencoderKLTorch, VQModelTorch          # noqa: E402  (reference)
    from resshift_b200.vq_arch import (kl_param_spec, kl_preset, random_kl_state_dict, random_vq_state_dict,
                                       vq_param_spec, wide_vq_preset)

    torch.set_grad_enabled(False)
    GOLD.mkdir(parents=True, exist_ok=True)

    inv = {}
    for name in ("tiny16", "tiny64", "f16", "f32"):
        cfg = kl_preset(name)
        m = AutoencoderKLTorch(**cfg.to_kwargs())
        inv["kl_" + name] = [[k, list(v.shape)] for k, v in m.state_dict().items()]
        assert [(k, tuple(s)) for k, s in inv["kl_" + name]] == [(n, tuple(s)) for n, s, _ in kl_param_spec(cfg)]
    for name in ("tiny16", "tiny64"):
        cfg = wide_vq_preset(name)
        m = VQModelTorch(**cfg.to_kwargs())
        inv["vq_" + name] = [[k, list(v.shape)] for k, v in m.state_dict().items()]
        assert [(k, tuple(s)) for k, s in inv["vq_" + name]] == [(n, tuple(s)) for n, s, _ in vq_param_spec(cfg)]
    (GOLD / "wide_latents_keys.json").write_text(json.dumps(inv))

    out = {}
    for name in ("tiny16", "tiny64"):
        cfg = kl_preset(name)
        model = AutoencoderKLTorch(**cfg.to_kwargs()).eval()
        model.load_state_dict(random_kl_state_dict(cfg, 0), strict=True)
        g = torch.Generator().manual_seed(2468)
        x = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1
        mode, moments = model.encode(x, sample_posterior=False, return_moments=True)
        torch.manual_seed(SAMPLE_SEED)                               # sample() draws on the CPU default generator
        sample = model.encode(x, sample_posterior=True)
        torch.manual_seed(SAMPLE_SEED)
        noise = torch.randn(mode.shape)
        assert torch.allclose(sample, mode + torch.exp(0.5 * torch.clamp(moments[:, cfg.embed_dim:], -30.0, 20.0)) * noise,
                              atol=1e-5)
        dec = model.decode(mode)
        out.update({f"kl_{name}_x": x, f"kl_{name}_moments": moments, f"kl_{name}_mode": mode, f"kl_{name}_sample": sample,
                    f"kl_{name}_dec": dec})
        print("kl", name, "moments std %.3f" % moments.std().item(), "dec std %.3f" % dec.std().item())

        cfg = wide_vq_preset(name)
        model = VQModelTorch(**cfg.to_kwargs()).eval()
        sd = random_vq_state_dict(cfg, 0)
        model.load_state_dict(sd, strict=True)
        x = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1
        z = torch.randn(1, cfg.embed_dim, 16, 16, generator=g) * 0.6
        enc = model.encode(x)
        _, _, info = model.quantize(z)
        idx = info[2].view(1, 16, 16)
        dec = model.decode(z)
        dec_nq = model.decode(z, force_not_quantize=True)
        out.update({f"vq_{name}_x": x, f"vq_{name}_z": z, f"vq_{name}_enc": enc, f"vq_{name}_idx": idx.to(torch.int32),
                    f"vq_{name}_dec": dec, f"vq_{name}_dec_nq": dec_nq})
        print("vq", name, "enc std %.3f" % enc.std().item(), "dec std %.3f" % dec.std().item(),
              "codes used", idx.unique().numel())
    np.savez_compressed(GOLD / "wide_latents.npz", sample_seed=np.int64(SAMPLE_SEED),
                        **{k: v.numpy() for k, v in out.items()})


if __name__ == "__main__":
    main()
