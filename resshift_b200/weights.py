"""Deterministic synthetic weights ("random-init weights of that architecture").

BASELINE.json's configs ask for random-init weights; the reference's own initialisation
zeroes the second conv of every ResBlock (reference models/unet.py:172-174), which would
hide GroupNorm / FiLM / conv errors behind ``skip(x) + 0``.  This generator therefore
draws *every* tensor from a seeded CPU generator (same values in this container and on
the GPU box), with fan-in scaling and a reduced gain on the residual-branch outputs so
activations stay well inside fp16 range.
"""
from __future__ import annotations

import math
from typing import Dict

import torch

from .arch import (unet_param_spec, unetconv_param_spec, unetmodel_param_spec, relative_position_index, shifted_window_mask,
                   swin_geometry)
from .config import UNetConfig, UNetModelConfig, UNetModelConvConfig

_BRANCH_OUT = ("out_layers.3.weight", "attn.proj.weight", "mlp.fc2.weight", "proj_out.weight", "out_layers.1.weight")


def param_spec(cfg):
    """The ``state_dict`` inventory of the denoiser a config describes."""
    if isinstance(cfg, UNetModelConvConfig):
        return unetconv_param_spec(cfg)
    return unetmodel_param_spec(cfg) if isinstance(cfg, UNetModelConfig) else unet_param_spec(cfg)


def random_state_dict(cfg, seed: int = 0) -> Dict[str, torch.Tensor]:
    """For a UNetConfig (UNetModelSwin), a UNetModelConfig (UNetModel) or a UNetModelConvConfig (UNetModelConv)."""
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    spec = param_spec(cfg)
    for name, shape, role in spec:
        if role in ("conv3", "conv1", "linear"):
            fan_in = math.prod(shape[1:])
            gain = 0.35 if name.endswith(_BRANCH_OUT) else 1.0
            sd[name] = torch.randn(shape, generator=g) * (gain / math.sqrt(fan_in))
        elif role == "bias":
            sd[name] = torch.randn(shape, generator=g) * 0.05
        elif role == "gn_w":
            sd[name] = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif role == "gn_b":
            sd[name] = 0.1 * torch.randn(shape, generator=g)
        elif role == "relpos":
            sd[name] = 0.5 * torch.randn(shape, generator=g)
        elif role == "buf_relidx":
            win = int(math.isqrt(shape[0]))
            sd[name] = relative_position_index(win)
        elif role == "buf_mask":
            nw, n = shape[0], shape[1]
            win = int(math.isqrt(n))
            side = int(math.isqrt(nw)) * win
            sd[name] = shifted_window_mask(side, side, win, win // 2)
        else:  # pragma: no cover
            raise ValueError(role)
    return sd
