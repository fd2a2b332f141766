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


def latent_channels_ok(c: int) -> bool:
    """Latent widths (z_channels, embed_dim) the first stage runs: 1..8, or a multiple of 8 from 16 to 64."""
    return 1 <= c <= 8 or (c % 8 == 0 and 16 <= c <= 64)


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
    dropout: float = 0.0        # identity at inference
    double_z: bool = False
    kl: bool = False            # AutoencoderKLTorch: double_z encoder, posterior moments, no codebook (n_embed unused)
    attn_type: str = "vanilla"  # "vanilla" / "vanilla-xformers" (AttnBlock, the same math and keys) or "none"
    resamp_with_conv: bool = True   # False: Downsample = avg_pool2d(2, 2), Upsample = nearest x2, no conv
    tanh_out: bool = False      # the decoder's image is tanh(conv_out(h))

    def __post_init__(self):
        self.ch_mult = tuple(int(v) for v in self.ch_mult)
        if isinstance(self.num_res_blocks, int):
            self.num_res_blocks = (self.num_res_blocks,) * len(self.ch_mult)
        self.num_res_blocks = tuple(int(v) for v in self.num_res_blocks)
        self.attn_resolutions = tuple(int(v) for v in self.attn_resolutions)
        self.resamp_with_conv, self.tanh_out = bool(self.resamp_with_conv), bool(self.tanh_out)
        assert self.double_z == self.kl
        assert len(self.num_res_blocks) == len(self.ch_mult)
        for what, c in (("z_channels", self.z_channels), ("embed_dim", self.embed_dim)):
            if not latent_channels_ok(c):
                raise ValueError(f"{what} must be 1..8 or a multiple of 8 from 16 to 64, got {c}: the first-stage kernels "
                                 "run latents of up to 8 channels, and wider ones as whole 16-byte fp16 rows up to 64")
        if self.attn_type in ("linear", "memory-efficient-cross-attn"):
            raise ValueError(f"attn_type {self.attn_type!r}: the reference's make_attn raises NotImplementedError for it "
                             "(ldm/modules/diffusionmodules/model.py:280-298), so no checkpoint of it exists")
        if self.attn_type not in ("vanilla", "vanilla-xformers", "none"):
            raise ValueError(f"attn_type {self.attn_type!r} unknown (vanilla, vanilla-xformers or none)")
        for i, c in enumerate(self.ch_mult):
            if (self.enc_attn[i] or self.dec_attn[i]) and (self.ch * c) % 64:
                raise ValueError(f"attention at level {i} ({self.ch * c} channels): the attention GEMMs need channels that "
                                 "are a multiple of 64")

    @property
    def has_attn(self) -> bool:
        """AttnBlocks are built (attn_type "none" makes every one of them nn.Identity)."""
        return self.attn_type != "none"

    @property
    def enc_attn(self) -> Tuple[bool, ...]:
        """Per encoder level: an AttnBlock after each ResnetBlock.  Encoder.__init__ tests curr_res = resolution halved
        (floor) once per level below (model.py:483-503)."""
        out, r = [], self.resolution
        for _ in range(self.levels):
            out.append(self.has_attn and r in self.attn_resolutions)
            r //= 2
        return tuple(out)

    @property
    def dec_attn(self) -> Tuple[bool, ...]:
        """Per decoder level (indexed by level, not by execution order): Decoder.__init__ tests curr_res =
        (resolution // 2^(L-1)) * 2^(L-1-i) (model.py:576-616), which differs from the encoder's when resolution is
        not a multiple of 2^(L-1)."""
        base = self.resolution // 2 ** (self.levels - 1)
        return tuple(self.has_attn and base * 2 ** (self.levels - 1 - i) in self.attn_resolutions for i in range(self.levels))

    @property
    def levels(self) -> int:
        return len(self.ch_mult)

    @property
    def downscale(self) -> int:
        return 2 ** (self.levels - 1)

    def ddconfig(self) -> dict:
        dd = {"double_z": self.double_z, "z_channels": self.z_channels, "resolution": self.resolution,
              "in_channels": self.in_channels, "out_ch": self.out_ch, "ch": self.ch, "ch_mult": list(self.ch_mult),
              "num_res_blocks": list(self.num_res_blocks), "attn_resolutions": list(self.attn_resolutions),
              "dropout": self.dropout, "padding_mode": "zeros"}
        # the options the shipped configs leave at their defaults are written only when they differ from them
        if self.attn_type != "vanilla":
            dd["attn_type"] = self.attn_type
        if not self.resamp_with_conv:
            dd["resamp_with_conv"] = False
        if self.tanh_out:
            dd["tanh_out"] = True
        return dd

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
    if name == "f16":                                   # LDM's kl-f16 (16-channel latent)
        return VQConfig(embed_dim=16, z_channels=16, resolution=256, ch=128, ch_mult=(1, 1, 2, 2, 4), num_res_blocks=2,
                        attn_resolutions=(16,), double_z=True, kl=True)
    if name == "f32":                                   # LDM's kl-f32 (64-channel latent)
        return VQConfig(embed_dim=64, z_channels=64, resolution=256, ch=128, ch_mult=(1, 1, 2, 2, 4, 4), num_res_blocks=2,
                        attn_resolutions=(16, 8), double_z=True, kl=True)
    if name in ("tiny16", "tiny64"):                    # the "tiny" topology with a 16- / 64-channel latent
        c = int(name[4:])
        return VQConfig(embed_dim=c, z_channels=c, resolution=64, ch=32, ch_mult=(1, 2, 4), num_res_blocks=(1, 2, 2),
                        double_z=True, kl=True)
    raise KeyError(name)


def wide_vq_preset(name: str) -> VQConfig:
    """VQ first stages with 16- or 64-channel latents on the "tiny" topology (test configurations)."""
    if name in ("tiny16", "tiny64"):
        c = int(name[4:])
        return VQConfig(embed_dim=c, n_embed=512, z_channels=c, resolution=64, ch=32, ch_mult=(1, 2, 4),
                        num_res_blocks=(1, 2, 2))
    raise KeyError(name)


def ldm_vq_preset(name: str) -> VQConfig:
    """LDM's VQ first stages with level attention or none, the ones a user would train ResShift's latent space in (not
    shipped with ResShift: test and measurement configurations with synthetic weights)."""
    if name == "vq-f8":
        return VQConfig(embed_dim=4, n_embed=16384, z_channels=4, resolution=256, ch=128, ch_mult=(1, 2, 2, 4),
                        num_res_blocks=2, attn_resolutions=(32,))
    if name == "vq-f8-n256":
        return VQConfig(embed_dim=4, n_embed=256, z_channels=4, resolution=256, ch=128, ch_mult=(1, 2, 2, 4),
                        num_res_blocks=2, attn_resolutions=(32,))
    if name == "vq-f16":
        return VQConfig(embed_dim=8, n_embed=16384, z_channels=8, resolution=256, ch=128, ch_mult=(1, 1, 2, 2, 4),
                        num_res_blocks=2, attn_resolutions=(16,))
    if name == "vq-f4-noattn":
        return VQConfig(embed_dim=3, n_embed=8192, z_channels=3, resolution=256, ch=128, ch_mult=(1, 2, 4),
                        num_res_blocks=2, attn_type="none")
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
        if cfg.enc_attn[i]:
            for j, (_, b) in enumerate(blocks):
                s += _attn(f"encoder.down.{i}.attn.{j}", b)
        if down and cfg.resamp_with_conv:
            s += _conv(f"encoder.down.{i}.downsample.conv", blocks[-1][1], blocks[-1][1], 3)
    top = cfg.ch * cfg.ch_mult[-1]
    mid_attn = (lambda p: _attn(p, top)) if cfg.has_attn else (lambda p: [])
    s += _resblock("encoder.mid.block_1", top, top) + mid_attn("encoder.mid.attn_1") + _resblock("encoder.mid.block_2", top, top)
    s += _gn("encoder.norm_out", top) + _conv("encoder.conv_out", top, z_out, 3)
    # decoder (state_dict order follows module registration: conv_in, mid, up.0 .. up.L-1, norm_out, conv_out)
    s += _conv("decoder.conv_in", cfg.z_channels, top, 3)
    s += _resblock("decoder.mid.block_1", top, top) + mid_attn("decoder.mid.attn_1") + _resblock("decoder.mid.block_2", top, top)
    by_level = {i: (blocks, up) for i, blocks, up in decoder_blocks(cfg)}
    for i in range(cfg.levels):
        blocks, up = by_level[i]
        for j, (a, b) in enumerate(blocks):
            s += _resblock(f"decoder.up.{i}.block.{j}", a, b)
        if cfg.dec_attn[i]:
            for j, (_, b) in enumerate(blocks):
                s += _attn(f"decoder.up.{i}.attn.{j}", b)
        if up and cfg.resamp_with_conv:
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
