"""ORACLE (test infrastructure, never shipped / never measured as the product).

``UNetModel.forward`` (reference models/unet.py:549-585) with ``AttentionBlock`` in both head orders (:224-344, the
einsum path the reference takes without xformers), on top of the ``oracle/unet_oracle.py`` /
``oracle/unet_variants_oracle.py`` functions.  CPU or GPU, fp32, on a reference-named ``state_dict``.  Pinned against
outputs of the imported reference (``oracle/make_golden_unetmodel.py`` -> ``tests/golden/unetmodel.npz``), see
``tests/test_oracle_unetmodel_golden.py``.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn.functional as F

from oracle.unet_oracle import SD, conv, group_norm, timestep_embedding
from oracle.unet_variants_oracle import res_block, resample
from resshift_b200.arch import unetmodel_block_plan
from resshift_b200.config import UNetModelConfig


def qkv_attention(qkv, heads: int, new_order: bool):
    """QKVAttentionLegacy (:274-299) / QKVAttention (:314-340): qkv [b, 3 heads ch, T] -> [b, heads ch, T]."""
    bs, width, length = qkv.shape
    ch = width // (3 * heads)
    scale = 1 / math.sqrt(math.sqrt(ch))
    if new_order:
        q, k, v = qkv.chunk(3, dim=1)
        q, k, v = (t.reshape(bs * heads, ch, length) for t in (q, k, v))
    else:
        q, k, v = qkv.reshape(bs * heads, ch * 3, length).split(ch, dim=1)
    weight = torch.einsum("bct,bcs->bts", q * scale, k * scale)
    weight = torch.softmax(weight.float(), dim=-1).type(weight.dtype)
    return torch.einsum("bts,bcs->bct", weight, v).reshape(bs, -1, length)


def attention_block(x, sd: SD, p: str, heads: int, new_order: bool):
    """AttentionBlock.forward (:257-263): x + proj_out(attention(qkv(norm(x))))."""
    b, c, *spatial = x.shape
    x = x.reshape(b, c, -1)
    qkv = F.conv1d(group_norm(x, sd, f"{p}.norm"), sd[f"{p}.qkv.weight"], sd[f"{p}.qkv.bias"])
    h = F.conv1d(qkv_attention(qkv, heads, new_order), sd[f"{p}.proj_out.weight"], sd[f"{p}.proj_out.bias"])
    return (x + h).reshape(b, c, *spatial)


def run_block(h, emb, sd: SD, prefix: str, layers, cfg: UNetModelConfig):
    for j, layer in enumerate(layers):
        kind, p = layer[0], f"{prefix}.{j}"
        if kind == "conv":
            h = conv(h, sd, p)
        elif kind == "res":
            h = res_block(h, emb, sd, p, cfg.use_scale_shift_norm)
        elif kind in ("res_down", "res_up"):
            h = res_block(h, emb, sd, p, cfg.use_scale_shift_norm, -1 if kind == "res_down" else 1)
        elif kind == "attn":
            h = attention_block(h, sd, p, layer[2], cfg.use_new_attention_order)
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
def unetmodel_forward(sd: SD, cfg: UNetModelConfig, x, timesteps, lq=None, probes: Optional[dict] = None):
    """reference models/unet.py:549-585 (y = None): lq of another size than x goes through pixel_unshuffle(lq, 2)."""
    emb = timestep_embedding(timesteps, cfg.model_channels)
    emb = F.linear(emb, sd["time_embed.0.weight"], sd["time_embed.0.bias"])
    emb = F.linear(F.silu(emb), sd["time_embed.2.weight"], sd["time_embed.2.bias"])
    if lq is not None:
        if lq.shape[2:] != x.shape[2:]:
            lq = F.pixel_unshuffle(lq, 2)
        x = torch.cat([x, lq], dim=1)
    input_blocks, middle, output_blocks = unetmodel_block_plan(cfg)
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
