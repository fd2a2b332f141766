"""ORACLE (test infrastructure, never shipped / never measured as the product).

CPU fp32 functional restatement of the first stages (``VQModelTorch``, ``AutoencoderKLTorch``; reference
ldm/models/autoencoder.py:12-86) built with any of the reference's ``Encoder`` / ``Decoder`` options
(ldm/modules/diffusionmodules/model.py:452-660): ``AttnBlock`` after every ResnetBlock of the levels ``VQConfig.enc_attn``
/ ``.dec_attn`` flag, no mid-block attention with ``attn_type: none`` (``nn.Identity``), ``avg_pool2d`` / nearest
resampling without a conv (``resamp_with_conv: False``, :51-88) and ``tanh_out`` (:658-659).  With the shipped options
it computes what ``oracle/vq_oracle.py`` does, from the same building blocks.  Pinned against outputs of the imported
reference (``oracle/make_golden_vq_options.py`` -> ``tests/golden/vq_opt_*.npz``).

Only ``tests/`` and the profiling scripts may import this module.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from oracle.vq_oracle import SD, _conv, _norm, _swish, quantize, resnet_block
from oracle.vq_oracle import downsample as _conv_downsample
from oracle.vq_oracle import upsample as _conv_upsample
from resshift_b200.vq_arch import VQConfig, decoder_blocks, encoder_blocks


def attn_block(x, sd: SD, p: str, chunk: Optional[int] = None):
    """Single-head self-attention over all H*W positions — reference model.py:180-203.  ``chunk`` query rows at a time
    (None: all at once, the reference's sequence of bmm calls): exact either way, as every row's softmax is over all
    keys; a chunk only bounds the T x T score matrix held at once (a GPU run at T = 65536 would need 17 GB per image)."""
    h_ = _norm(x, sd, f"{p}.norm")
    q, k, v = (_conv(h_, sd, f"{p}.{n}") for n in ("q", "k", "v"))
    b, c, h, w = q.shape
    q = q.reshape(b, c, h * w).permute(0, 2, 1)
    k = k.reshape(b, c, h * w)
    v = v.reshape(b, c, h * w)
    step = chunk or h * w
    outs = []
    for r in range(0, h * w, step):
        w_ = F.softmax(torch.bmm(q[:, r:r + step], k) * (int(c) ** (-0.5)), dim=2)
        outs.append(torch.bmm(v, w_.permute(0, 2, 1)))
    return x + _conv(torch.cat(outs, dim=2).reshape(b, c, h, w), sd, f"{p}.proj_out")


def downsample(x, sd: SD, p: str, cfg: VQConfig):
    """Downsample (model.py:78-87): the padded stride-2 conv, or a 2x2 average pool without resamp_with_conv."""
    return _conv_downsample(x, sd, p) if cfg.resamp_with_conv else F.avg_pool2d(x, kernel_size=2, stride=2)


def upsample(x, sd: SD, p: str, cfg: VQConfig):
    """Upsample (model.py:62-66): nearest x2, then the conv unless resamp_with_conv is off."""
    return _conv_upsample(x, sd, p) if cfg.resamp_with_conv else F.interpolate(x, scale_factor=2.0, mode="nearest")


@torch.no_grad()
def encoder(x, sd: SD, cfg: VQConfig, chunk: Optional[int] = None):
    """reference model.py:533-559."""
    h = _conv(x, sd, "encoder.conv_in")
    for i, blocks, down in encoder_blocks(cfg):
        for j in range(len(blocks)):
            h = resnet_block(h, sd, f"encoder.down.{i}.block.{j}")
            if cfg.enc_attn[i]:
                h = attn_block(h, sd, f"encoder.down.{i}.attn.{j}", chunk)
        if down:
            h = downsample(h, sd, f"encoder.down.{i}.downsample", cfg)
    h = resnet_block(h, sd, "encoder.mid.block_1")
    if cfg.has_attn:
        h = attn_block(h, sd, "encoder.mid.attn_1", chunk)
    h = resnet_block(h, sd, "encoder.mid.block_2")
    return _conv(_swish(_norm(h, sd, "encoder.norm_out")), sd, "encoder.conv_out")


@torch.no_grad()
def decoder(z, sd: SD, cfg: VQConfig, chunk: Optional[int] = None):
    """reference model.py:626-660."""
    h = _conv(z, sd, "decoder.conv_in")
    h = resnet_block(h, sd, "decoder.mid.block_1")
    if cfg.has_attn:
        h = attn_block(h, sd, "decoder.mid.attn_1", chunk)
    h = resnet_block(h, sd, "decoder.mid.block_2")
    for i, blocks, up in decoder_blocks(cfg):
        for j in range(len(blocks)):
            h = resnet_block(h, sd, f"decoder.up.{i}.block.{j}")
            if cfg.dec_attn[i]:
                h = attn_block(h, sd, f"decoder.up.{i}.attn.{j}", chunk)
        if up:
            h = upsample(h, sd, f"decoder.up.{i}.upsample", cfg)
    h = _conv(_swish(_norm(h, sd, "decoder.norm_out")), sd, "decoder.conv_out")
    return torch.tanh(h) if cfg.tanh_out else h


@torch.no_grad()
def vq_encode(x, sd: SD, cfg: VQConfig, chunk: Optional[int] = None):
    """VQModelTorch.encode — reference autoencoder.py:28-31."""
    return _conv(encoder(x, sd, cfg, chunk), sd, "quant_conv")


@torch.no_grad()
def vq_decode(h, sd: SD, cfg: VQConfig, force_not_quantize: bool = False, return_indices: bool = False,
              chunk: Optional[int] = None):
    """VQModelTorch.decode — reference autoencoder.py:33-40."""
    idx = None
    if not force_not_quantize:
        h, idx = quantize(h, sd)
    out = decoder(_conv(h, sd, "post_quant_conv"), sd, cfg, chunk)
    return (out, idx) if return_indices else out


@torch.no_grad()
def kl_moments(x, sd: SD, cfg: VQConfig, chunk: Optional[int] = None):
    """quant_conv(Encoder(x)): [B, 2 embed_dim, H/f, W/f] — reference autoencoder.py:66-67; the mode is the first half."""
    return _conv(encoder(x, sd, cfg, chunk), sd, "quant_conv")


@torch.no_grad()
def kl_decode(z, sd: SD, cfg: VQConfig, chunk: Optional[int] = None):
    """AutoencoderKLTorch.decode — reference autoencoder.py:78-81."""
    return decoder(_conv(z, sd, "post_quant_conv"), sd, cfg, chunk)
