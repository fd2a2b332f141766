"""ORACLE (test infrastructure, never shipped / never measured as the product).

``UNetModelConv.forward`` (reference models/unet.py:1153-1181) with ``ResBlockConv`` (:914-1004), on top of the
``oracle/unet_oracle.py`` / ``oracle/unet_variants_oracle.py`` functions.  CPU or GPU, fp32, on a reference-named
``state_dict``.  Pinned against outputs of the imported reference (``oracle/make_golden_unetconv.py`` ->
``tests/golden/unetconv.npz``), see ``tests/test_oracle_unetconv_golden.py``.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from oracle.unet_oracle import SD, conv, timestep_embedding
from oracle.unet_variants_oracle import resample
from resshift_b200.arch import unetconv_block_plan
from resshift_b200.config import UNetModelConvConfig


def res_block_conv(x, emb, sd: SD, p: str, scale_shift: bool, updown: int = 0):
    """ResBlockConv.forward (:984-1004).  With scale-shift norm out_layers[0] is the SiLU (there is no norm), so the
    middle is SiLU(h) * (1 + scale) + shift and no SiLU follows the FiLM; without it, out_layers(h + emb_out)."""
    h = F.silu(x)
    h, x = resample(h, updown), resample(x, updown)                 # h_upd / x_upd (:985-990; identity for updown 0)
    h = conv(h, sd, f"{p}.in_layers.1")
    e = F.linear(F.silu(emb), sd[f"{p}.emb_layers.1.weight"], sd[f"{p}.emb_layers.1.bias"])[:, :, None, None]
    if scale_shift:
        scale, shift = e.chunk(2, dim=1)
        h = F.silu(h) * (1 + scale) + shift
    else:
        h = F.silu(h + e)
    h = conv(h, sd, f"{p}.out_layers.1")
    skip = conv(x, sd, f"{p}.skip_connection") if f"{p}.skip_connection.weight" in sd else x
    return skip + h


def run_block(h, emb, sd: SD, prefix: str, layers, cfg: UNetModelConvConfig):
    for j, layer in enumerate(layers):
        kind, p = layer[0], f"{prefix}.{j}"
        if kind == "conv":
            h = conv(h, sd, p)
        elif kind == "res":
            h = res_block_conv(h, emb, sd, p, cfg.use_scale_shift_norm)
        elif kind in ("res_down", "res_up"):
            h = res_block_conv(h, emb, sd, p, cfg.use_scale_shift_norm, -1 if kind == "res_down" else 1)
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
def unetconv_forward(sd: SD, cfg: UNetModelConvConfig, x, timesteps, lq=None, probes: Optional[dict] = None):
    """reference models/unet.py:1153-1181: lq of another size than x goes through pixel_unshuffle(lq, 2); the head is
    conv3x3(SiLU(h)) (:1148-1151)."""
    emb = timestep_embedding(timesteps, cfg.model_channels)
    emb = F.linear(emb, sd["time_embed.0.weight"], sd["time_embed.0.bias"])
    emb = F.linear(F.silu(emb), sd["time_embed.2.weight"], sd["time_embed.2.bias"])
    if lq is not None:
        if lq.shape[2:] != x.shape[2:]:
            lq = F.pixel_unshuffle(lq, 2)
        x = torch.cat([x, lq], dim=1)
    input_blocks, middle, output_blocks = unetconv_block_plan(cfg)
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
    return conv(F.silu(h), sd, "out.1")
