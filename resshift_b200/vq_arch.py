"""Architecture description of the VQ-GAN first stage (the bookends around the denoising loop).

Restates the constructor logic of the reference's ``VQModelTorch`` (reference ldm/models/autoencoder.py:12-26),
``Encoder`` / ``Decoder`` (ldm/modules/diffusionmodules/model.py:452-660), ``ResnetBlock`` (:90-149), ``AttnBlock``
(:152-203), ``Downsample`` / ``Upsample`` (:51-88) and ``VectorQuantizer2`` (ldm/modules/vqvae/quantize.py:213-241) as a
flat parameter inventory with the reference's ``state_dict`` key names and shapes, so that released checkpoints
(``autoencoder_vq_f4.pth``, ``ffhq512_vq_f8_dim8_face.pth``) load unchanged.  Shared by the module
(``resshift_b200.models.autoencoder``), the weight generator and the CPU oracle.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, asdict
from typing import Dict, List, Sequence, Tuple

import torch


@dataclass
class VQConfig:
    """``autoencoder.params`` of the shipped yaml files (embed_dim, n_embed, ddconfig.*)."""
    embed_dim: int = 3
    n_embed: int = 8192
    z_channels: int = 3
    resolution: int = 256
    in_channels: int = 3
    out_ch: int = 3
    ch: int = 128
    ch_mult: Sequence[int] = (1, 2, 4)
    num_res_blocks: Sequence[int] = (2, 2, 2)
    attn_resolutions: Sequence[int] = ()
    dropout: float = 0.0
    double_z: bool = False
    kl: bool = False            # AutoencoderKLTorch: double_z encoder, posterior moments, no codebook (n_embed unused)

    def __post_init__(self):
        self.ch_mult = tuple(int(v) for v in self.ch_mult)
        if isinstance(self.num_res_blocks, int):
            self.num_res_blocks = (self.num_res_blocks,) * len(self.ch_mult)
        self.num_res_blocks = tuple(int(v) for v in self.num_res_blocks)
        self.attn_resolutions = tuple(int(v) for v in self.attn_resolutions)
        # what this implementation covers (every shipped yaml satisfies these)
        assert self.double_z == self.kl and self.dropout == 0 and len(self.attn_resolutions) == 0
        assert len(self.num_res_blocks) == len(self.ch_mult)

    @property
    def levels(self) -> int:
        return len(self.ch_mult)

    @property
    def downscale(self) -> int:
        return 2 ** (self.levels - 1)

    def ddconfig(self) -> dict:
        return {"double_z": self.double_z, "z_channels": self.z_channels, "resolution": self.resolution,
                "in_channels": self.in_channels, "out_ch": self.out_ch, "ch": self.ch, "ch_mult": list(self.ch_mult),
                "num_res_blocks": list(self.num_res_blocks), "attn_resolutions": list(self.attn_resolutions),
                "dropout": 0.0, "padding_mode": "zeros"}

    def to_kwargs(self) -> dict:
        if self.kl:
            return {"ddconfig": self.ddconfig(), "embed_dim": self.embed_dim}
        return {"ddconfig": self.ddconfig(), "n_embed": self.n_embed, "embed_dim": self.embed_dim}


def vq_preset(name: str) -> VQConfig:
    if name in ("f4", "autoencoder_vq_f4"):            # realsr / bicsr / inpaint_imagenet (configs/*.yaml autoencoder block)
        return VQConfig()
    if name in ("f8_face", "ffhq512_vq_f8_dim8_face"):  # configs/faceir_gfpgan512_lpips.yaml:47-73
        return VQConfig(embed_dim=8, n_embed=4096, z_channels=8, resolution=512, ch=64, ch_mult=(1, 2, 4, 8),
                        num_res_blocks=(1, 2, 3, 4))
    if name == "tiny":                                  # not shipped: same topology, narrow, for fast tests
        return VQConfig(n_embed=512, resolution=64, ch=32, ch_mult=(1, 2, 4), num_res_blocks=(1, 2, 2))
    raise KeyError(name)


def kl_preset(name: str) -> VQConfig:
    """KL first stages (AutoencoderKLTorch); no shipped ResShift config uses one, so these are test configurations."""
    if name == "f8":                                    # Stable-Diffusion-style f8 KL autoencoder
        return VQConfig(embed_dim=4, z_channels=4, resolution=256, ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=(2, 2, 2, 2),
                        double_z=True, kl=True)
    if name == "tiny":                                  # the VQ "tiny" topology with a KL bottleneck
        return VQConfig(embed_dim=4, z_channels=4, resolution=64, ch=32, ch_mult=(1, 2, 4), num_res_blocks=(1, 2, 2),
                        double_z=True, kl=True)
    raise KeyError(name)


# role: conv3 | conv1 | bias | gn_w | gn_b | codebook
Spec = List[Tuple[str, Tuple[int, ...], str]]


def _conv(name, cin, cout, k) -> Spec:
    return [(f"{name}.weight", (cout, cin, k, k), "conv3" if k == 3 else "conv1"), (f"{name}.bias", (cout,), "bias")]


def _gn(name, c) -> Spec:
    return [(f"{name}.weight", (c,), "gn_w"), (f"{name}.bias", (c,), "gn_b")]


def _resblock(name, cin, cout) -> Spec:
    s = _gn(f"{name}.norm1", cin) + _conv(f"{name}.conv1", cin, cout, 3) + _gn(f"{name}.norm2", cout) + _conv(f"{name}.conv2", cout, cout, 3)
    if cin != cout:
        s += _conv(f"{name}.nin_shortcut", cin, cout, 1)
    return s


def _attn(name, c) -> Spec:
    return _gn(f"{name}.norm", c) + _conv(f"{name}.q", c, c, 1) + _conv(f"{name}.k", c, c, 1) + _conv(f"{name}.v", c, c, 1) + \
        _conv(f"{name}.proj_out", c, c, 1)


def encoder_blocks(cfg: VQConfig):
    """[(level, [(cin, cout), ...], has_downsample)] as Encoder.__init__ builds them (model.py:480-503)."""
    in_mult = (1,) + tuple(cfg.ch_mult)
    out = []
    for i in range(cfg.levels):
        bi, bo = cfg.ch * in_mult[i], cfg.ch * cfg.ch_mult[i]
        blocks = []
        for _ in range(cfg.num_res_blocks[i]):
            blocks.append((bi, bo))
            bi = bo
        out.append((i, blocks, i != cfg.levels - 1))
    return out


def decoder_blocks(cfg: VQConfig):
    """[(level, [(cin, cout), ...], has_upsample)] in EXECUTION order (highest level first; model.py:596-616)."""
    bi = cfg.ch * cfg.ch_mult[-1]
    out = []
    for i in reversed(range(cfg.levels)):
        bo = cfg.ch * cfg.ch_mult[i]
        blocks = []
        for _ in range(cfg.num_res_blocks[i] + 1):
            blocks.append((bi, bo))
            bi = bo
        out.append((i, blocks, i != 0))
    return out


def vq_param_spec(cfg: VQConfig) -> Spec:
    """VQModelTorch's state_dict inventory (reference ldm/models/autoencoder.py:21-26)."""
    assert not cfg.kl
    return _first_stage_spec(cfg)


def kl_param_spec(cfg: VQConfig) -> Spec:
    """AutoencoderKLTorch's state_dict inventory (reference ldm/models/autoencoder.py:58-62): the encoder ends in
    2 z_channels, quant_conv maps them to the 2 embed_dim moments, and there is no codebook."""
    assert cfg.kl
    return _first_stage_spec(cfg)


def _first_stage_spec(cfg: VQConfig) -> Spec:
    z_out = 2 * cfg.z_channels if cfg.double_z else cfg.z_channels
    s: Spec = []
    # encoder
    s += _conv("encoder.conv_in", cfg.in_channels, cfg.ch, 3)
    for i, blocks, down in encoder_blocks(cfg):
        for j, (a, b) in enumerate(blocks):
            s += _resblock(f"encoder.down.{i}.block.{j}", a, b)
        if down:
            s += _conv(f"encoder.down.{i}.downsample.conv", blocks[-1][1], blocks[-1][1], 3)
    top = cfg.ch * cfg.ch_mult[-1]
    s += _resblock("encoder.mid.block_1", top, top) + _attn("encoder.mid.attn_1", top) + _resblock("encoder.mid.block_2", top, top)
    s += _gn("encoder.norm_out", top) + _conv("encoder.conv_out", top, z_out, 3)
    # decoder (state_dict order follows module registration: conv_in, mid, up.0 .. up.L-1, norm_out, conv_out)
    s += _conv("decoder.conv_in", cfg.z_channels, top, 3)
    s += _resblock("decoder.mid.block_1", top, top) + _attn("decoder.mid.attn_1", top) + _resblock("decoder.mid.block_2", top, top)
    by_level = {i: (blocks, up) for i, blocks, up in decoder_blocks(cfg)}
    for i in range(cfg.levels):
        blocks, up = by_level[i]
        for j, (a, b) in enumerate(blocks):
            s += _resblock(f"decoder.up.{i}.block.{j}", a, b)
        if up:
            s += _conv(f"decoder.up.{i}.upsample.conv", blocks[-1][1], blocks[-1][1], 3)
    s += _gn("decoder.norm_out", cfg.ch * cfg.ch_mult[0]) + _conv("decoder.conv_out", cfg.ch * cfg.ch_mult[0], cfg.out_ch, 3)
    # quantiser (VQ) and the two 1x1 convs around it / around the posterior (KL)
    if cfg.kl:
        s += _conv("quant_conv", z_out, 2 * cfg.embed_dim, 1)
    else:
        s += [("quantize.embedding.weight", (cfg.n_embed, cfg.embed_dim), "codebook")]
        s += _conv("quant_conv", cfg.z_channels, cfg.embed_dim, 1)
    s += _conv("post_quant_conv", cfg.embed_dim, cfg.z_channels, 1)
    return s


def random_vq_state_dict(cfg: VQConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Deterministic synthetic weights (same values in the build container and on the GPU box): fan-in scaled convs with a
    reduced gain on the residual-branch outputs so activations stay in fp16 range, and a codebook with the spread of
    the latents it quantises (the reference's uniform(+-1/n_e) init would make every code equally near)."""
    return _random_state_dict(vq_param_spec(cfg), seed)


def random_kl_state_dict(cfg: VQConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Deterministic synthetic weights of AutoencoderKLTorch, drawn as random_vq_state_dict draws them."""
    return _random_state_dict(kl_param_spec(cfg), seed)


def _random_state_dict(spec: Spec, seed: int) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    for name, shape, role in spec:
        if role in ("conv3", "conv1"):
            fan_in = math.prod(shape[1:])
            gain = 0.35 if name.endswith(("conv2.weight", "proj_out.weight")) else 1.0
            sd[name] = torch.randn(shape, generator=g) * (gain / math.sqrt(fan_in))
        elif role == "bias":
            sd[name] = torch.randn(shape, generator=g) * 0.05
        elif role == "gn_w":
            sd[name] = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif role == "gn_b":
            sd[name] = 0.1 * torch.randn(shape, generator=g)
        elif role == "codebook":
            sd[name] = 0.6 * torch.randn(shape, generator=g)
        else:  # pragma: no cover
            raise ValueError(role)
    return sd
