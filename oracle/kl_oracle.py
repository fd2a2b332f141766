"""ORACLE (test infrastructure, never shipped / never measured as the product).

CPU fp32 functional restatement of the KL first stage — ``AutoencoderKLTorch.encode`` / ``.decode`` (reference
ldm/models/autoencoder.py:52-86) with ``DiagonalGaussianDistribution`` (ldm/modules/distributions/distributions.py:24-62)
— on the Encoder / Decoder of ``oracle/vq_oracle.py``, working directly on a reference-named ``state_dict``.
Pinned against outputs of the imported reference (``oracle/make_golden_kl.py`` -> ``tests/golden/kl_*.npz``).

Only ``tests/`` and the profiling scripts may import this module.
"""
from __future__ import annotations

from typing import Optional

import torch

from oracle.vq_oracle import SD, _conv, decoder, encoder
from resshift_b200.vq_arch import VQConfig


@torch.no_grad()
def moments(x, sd: SD, cfg: VQConfig):
    """quant_conv(Encoder(x)): [B, 2 embed_dim, H/f, W/f] — reference autoencoder.py:66-67."""
    return _conv(encoder(x, sd, cfg), sd, "quant_conv")


def posterior(m):
    """DiagonalGaussianDistribution(m): (mean, std) — reference distributions.py:25-31."""
    mean, logvar = torch.chunk(m, 2, dim=1)
    logvar = torch.clamp(logvar, -30.0, 20.0)
    return mean, torch.exp(0.5 * logvar)


@torch.no_grad()
def kl_encode(x, sd: SD, cfg: VQConfig, noise: Optional[torch.Tensor] = None, return_moments: bool = False):
    """AutoencoderKLTorch.encode — reference autoencoder.py:65-76: mode() without ``noise``, else
    sample() = mean + std * noise (distributions.py:35-37) with the given noise."""
    m = moments(x, sd, cfg)
    mean, std = posterior(m)
    z = mean if noise is None else mean + std * noise.to(mean.device)
    return (z, m) if return_moments else z


@torch.no_grad()
def kl_decode(z, sd: SD, cfg: VQConfig):
    """AutoencoderKLTorch.decode — reference autoencoder.py:78-81."""
    return decoder(_conv(z, sd, "post_quant_conv"), sd, cfg)
