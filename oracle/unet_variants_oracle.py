"""ORACLE (test infrastructure, never shipped / never measured as the product).

``UNetModelSwin.forward`` for every constructor option the reference can run, on top of the functions of
``oracle/unet_oracle.py`` (which restates the shipped topology): ``use_scale_shift_norm=False``, ``resblock_updown``,
``conv_resample=False``, ``patch_norm``, ``cond_mask`` with ``lq_size == image_size`` and dropout (the identity at
inference).  CPU or GPU, fp32, on a reference-named ``state_dict``.  Pinned against outputs of the imported reference
(``oracle/make_golden_variants.py`` -> ``tests/golden/unet_variants.npz``), see ``tests/test_oracle_variants_golden.py``.
For a shipped configuration it computes what ``unet_oracle.unet_forward`` computes.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from oracle.unet_oracle import SD, conv, feature_extractor, group_norm, swin_block, timestep_embedding
from resshift_b200.arch import swin_geometry, unet_block_plan
from resshift_b200.config import UNetConfig


def resample(x, updown: int):
    """h_upd / x_upd (reference models/unet.py:150-158): 2x2 average pool (updown < 0, Downsample without conv,
    :83-108), nearest 2x (updown > 0, Upsample without conv, :53-81), identity (0)."""
    if updown < 0:
        return F.avg_pool2d(x, kernel_size=2, stride=2)
    if updown > 0:
        return F.interpolate(x, scale_factor=2, mode="nearest")
    return x


def res_block(x, emb, sd: SD, p: str, scale_shift: bool, updown: int = 0):
    """reference models/unet.py:186-206; updown -1 / +1: a ResBlock with down / up = True (:187-193)."""
    h = F.silu(group_norm(x, sd, f"{p}.in_layers.0"))
    h, x = resample(h, updown), resample(x, updown)
    h = conv(h, sd, f"{p}.in_layers.2")
    e = F.linear(F.silu(emb), sd[f"{p}.emb_layers.1.weight"], sd[f"{p}.emb_layers.1.bias"])[:, :, None, None]
    if scale_shift:
        scale, shift = torch.chunk(e, 2, dim=1)
        h = group_norm(h, sd, f"{p}.out_layers.0") * (1 + scale) + shift
    else:
        h = group_norm(h + e, sd, f"{p}.out_layers.0")
    h = conv(F.silu(h), sd, f"{p}.out_layers.3")
    if f"{p}.skip_connection.weight" in sd:
        x = conv(x, sd, f"{p}.skip_connection")
    return x + h


def basic_layer(x, sd: SD, p: str, cfg: UNetConfig, ctor_res: int):
    """reference models/swin_transformer.py:427-442, patch_size 1; patch_norm: GroupNorm32 after each projection
    (PatchEmbed / PatchUnEmbed, :452-527)."""
    win, shift = swin_geometry(cfg, ctor_res)
    x = conv(x, sd, f"{p}.patch_embed.proj")
    if cfg.patch_norm:
        x = group_norm(x, sd, f"{p}.patch_embed.norm")
    for i in range(cfg.swin_depth):
        x = swin_block(x, sd, f"{p}.blocks.{i}", cfg.swin_heads, win, shift if i % 2 else 0)
    x = conv(x, sd, f"{p}.patch_unembed.proj")
    if cfg.patch_norm:
        x = group_norm(x, sd, f"{p}.patch_unembed.norm")
    return x


def run_block(h, emb, sd: SD, prefix: str, layers, cfg: UNetConfig):
    for j, layer in enumerate(layers):
        kind, p = layer[0], f"{prefix}.{j}"
        if kind == "conv":
            h = conv(h, sd, p)
        elif kind == "res":
            h = res_block(h, emb, sd, p, cfg.use_scale_shift_norm)
        elif kind in ("res_down", "res_up"):
            h = res_block(h, emb, sd, p, cfg.use_scale_shift_norm, -1 if kind == "res_down" else 1)
        elif kind == "swin":
            h = basic_layer(h, sd, p, cfg, layer[2])
        elif kind == "down":
            h = conv(h, sd, f"{p}.op", stride=2) if cfg.conv_resample else resample(h, -1)
        elif kind == "up":
            h = resample(h, 1)
            if cfg.conv_resample:
                h = conv(h, sd, f"{p}.conv")
        else:  # pragma: no cover
            raise ValueError(kind)
    return h


@torch.no_grad()
def unet_forward(sd: SD, cfg: UNetConfig, x, timesteps, lq=None, mask=None, probes: Optional[dict] = None):
    """reference models/unet.py:865-895.  With cond_mask and no feature extractor, cat([x, lq, mask]) (:876-882)."""
    emb = timestep_embedding(timesteps, cfg.model_channels)
    emb = F.linear(emb, sd["time_embed.0.weight"], sd["time_embed.0.bias"])
    emb = F.linear(F.silu(emb), sd["time_embed.2.weight"], sd["time_embed.2.bias"])
    if lq is not None:
        if mask is not None:
            lq = torch.cat([lq, mask], dim=1)
        x = torch.cat([x, feature_extractor(lq.float(), sd, cfg)], dim=1)
    input_blocks, middle, output_blocks = unet_block_plan(cfg)
    h = x.float()
    hs = []
    for i, layers in enumerate(input_blocks):
        h = run_block(h, emb, sd, f"input_blocks.{i}", layers, cfg)
        hs.append(h)
        if probes is not None:
            probes[f"input_blocks.{i}"] = h
    h = run_block(h, emb, sd, "middle_block", middle, cfg)
    if probes is not None:
        probes["middle_block"] = h
    for i, layers in enumerate(output_blocks):
        h = run_block(torch.cat([h, hs.pop()], dim=1), emb, sd, f"output_blocks.{i}", layers, cfg)
        if probes is not None:
            probes[f"output_blocks.{i}"] = h
    return conv(F.silu(group_norm(h, sd, "out.0")), sd, "out.2")
