"""Model / diffusion configuration mirroring the reference's yaml ``params`` trees.

``UNetConfig`` carries exactly the keyword arguments of ``UNetModelSwin.__init__``
(reference models/unet.py:632-657) and ``DiffusionConfig`` those of
``create_gaussian_diffusion`` (reference models/script_util.py:7-21).  The presets
restate the ``model.params`` / ``diffusion.params`` blocks of the shipped yaml files
(reference configs/*.yaml) so that benchmarks and tests do not need the reference tree.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field, asdict
from typing import Optional, Sequence, Tuple


def _x_channels(in_channels: int, out_channels: int) -> Optional[int]:
    """Channels of x in a UNetModel / UNetModelConv, whose input is x and lq (3 channels at the latent size, or 12 at
    twice it through pixel_unshuffle) concatenated: out_channels, else out_channels / 2 (a learned-variance head outputs
    the mean, then as many variance values).  None when neither reading fits."""
    for x in (out_channels, out_channels // 2 if out_channels % 2 == 0 else None):
        if x is not None and x > 0 and in_channels - x in (3, 12):
            return x
    return None


@dataclass
class UNetConfig:
    image_size: int = 64
    in_channels: int = 3
    model_channels: int = 160
    out_channels: int = 3
    num_res_blocks: Sequence[int] = (2, 2, 2, 2)
    attention_resolutions: Sequence[int] = (64, 32, 16, 8)
    dropout: float = 0.0
    channel_mult: Sequence[int] = (1, 2, 2, 4)
    conv_resample: bool = True
    dims: int = 2
    use_fp16: bool = False
    num_heads: int = 1
    num_head_channels: int = 32
    use_scale_shift_norm: bool = True
    resblock_updown: bool = False
    swin_depth: int = 2
    swin_embed_dim: int = 192
    window_size: int = 8
    mlp_ratio: float = 4.0
    patch_norm: bool = False
    cond_lq: bool = True
    cond_mask: bool = False
    lq_size: int = 64

    def __post_init__(self):
        if isinstance(self.num_res_blocks, int):
            self.num_res_blocks = (self.num_res_blocks,) * len(self.channel_mult)
        self.num_res_blocks = tuple(int(v) for v in self.num_res_blocks)
        self.channel_mult = tuple(int(v) for v in self.channel_mult)
        self.attention_resolutions = tuple(int(v) for v in self.attention_resolutions)
        # What this implementation covers: every constructor option the reference can run, except the attention kernels'
        # specialisations.  dropout is the identity at inference.
        assert len(self.num_res_blocks) == len(self.channel_mult)
        if self.dims != 2:
            raise ValueError(f"dims={self.dims}: only 2-D UNets are covered (every ResShift config uses dims=2)")
        if not self.cond_lq:
            raise ValueError("cond_lq=False: the reference cannot run it either (it widens the first conv by the LQ "
                             "channels but skips the concatenation when lq is None)")
        if self.window_size not in (8, 16):
            raise ValueError(f"window_size={self.window_size}: the window-attention kernels are instantiated for 8x8 and "
                             f"16x16 windows")
        if self.swin_embed_dim % self.swin_heads or self.swin_embed_dim // self.swin_heads not in (32, 64):
            raise ValueError(f"head dim {self.swin_embed_dim / self.swin_heads:g}: the window-attention kernels are "
                             f"instantiated for head dims of 32 and 64 (num_head_channels 32 or 64)")

    # -- derived quantities (reference models/unet.py:689-709) -----------------
    @property
    def swin_heads(self) -> int:
        if self.num_head_channels == -1:
            return self.num_heads
        return self.swin_embed_dim // self.num_head_channels

    @property
    def time_embed_dim(self) -> int:
        return self.model_channels * 4

    @property
    def fe_stages(self) -> int:
        """Number of (conv3x3, SiLU, conv3x3-stride-2) stages in ``feature_extractor``."""
        if self.lq_size == self.image_size:
            return 0
        return int(math.log(self.lq_size / self.image_size) / math.log(2))

    @property
    def lq_in_channels(self) -> int:
        return 4 if self.cond_mask else 3

    @property
    def lq_feat_channels(self) -> int:
        """Channels that get concatenated to x (``base_chn`` in the reference)."""
        if self.lq_size == self.image_size:
            return self.lq_in_channels
        return 16 * (2 ** self.fe_stages)

    @property
    def x_channels(self) -> int:
        """Channels of x (the latent): in_channels; lq enters through its own path"""
        return self.in_channels

    def to_kwargs(self) -> dict:
        d = asdict(self)
        d["num_res_blocks"] = list(self.num_res_blocks)
        d["channel_mult"] = list(self.channel_mult)
        d["attention_resolutions"] = list(self.attention_resolutions)
        return d


@dataclass
class UNetModelConfig:
    """Exactly the keyword arguments of ``UNetModel.__init__`` (reference models/unet.py:373-393), the global-attention
    UNet.  What the native kernels cannot run is refused here with the reason."""
    image_size: int = 64
    in_channels: int = 6
    model_channels: int = 160
    out_channels: int = 3
    num_res_blocks: Sequence[int] = (2, 2, 2, 2)
    attention_resolutions: Sequence[int] = (64, 32, 16, 8)
    cond_lq: bool = True
    dropout: float = 0.0
    channel_mult: Sequence[int] = (1, 2, 4, 8)
    conv_resample: bool = True
    dims: int = 2
    num_classes: Optional[int] = None
    use_fp16: bool = False
    num_heads: int = 1
    num_head_channels: int = -1
    use_scale_shift_norm: bool = False
    resblock_updown: bool = False
    use_new_attention_order: bool = False

    def __post_init__(self):
        if isinstance(self.num_res_blocks, int):
            self.num_res_blocks = (self.num_res_blocks,) * len(self.channel_mult)
        self.num_res_blocks = tuple(int(v) for v in self.num_res_blocks)
        self.channel_mult = tuple(int(v) for v in self.channel_mult)
        self.attention_resolutions = tuple(int(v) for v in self.attention_resolutions)
        if len(self.num_res_blocks) != len(self.channel_mult):
            raise ValueError("num_res_blocks and channel_mult must have the same length")
        if self.dims != 2:
            raise ValueError(f"dims={self.dims}: only 2-D UNets are covered (every ResShift config uses dims=2)")
        if self.num_classes is not None:
            raise ValueError("num_classes: class-conditional UNetModel is not covered (the ResShift sampler never passes "
                             "labels, so the reference's own `y is not None` assert would fire)")
        if not self.cond_lq:
            raise ValueError("cond_lq=False: the ResShift sampler always passes lq, and the reference asserts cond_lq then")
        if _x_channels(self.in_channels, self.out_channels) is None:
            raise ValueError(f"in_channels={self.in_channels}, out_channels={self.out_channels}: x has out_channels "
                             f"channels and lq is a 3-channel image, so in_channels must be out_channels + 3 (lq at the "
                             f"latent size) or out_channels + 12 (lq at twice it, through pixel_unshuffle); with a "
                             f"learned variance (even out_channels) x has out_channels / 2 channels, and in_channels "
                             f"is out_channels / 2 + 3 or + 12")
        if self.model_channels % 32:
            raise ValueError(f"model_channels={self.model_channels}: GroupNorm32 needs channel counts divisible by 32")
        for ch, output_block in self.attention_layers():
            heads = self.heads(ch, output_block)
            if heads <= 0 or ch % heads or ch // heads not in (32, 64, 128):
                where = "an output block" if output_block else "an input / the middle block"
                raise ValueError(f"AttentionBlock of {where} over {ch} channels with {heads} head(s): the attention kernel "
                                 f"is instantiated for head dims 32, 64 and 128; set num_head_channels to 32, 64 or 128 "
                                 f"(with num_head_channels=-1 output blocks have one head over all their channels)")

    def heads(self, ch: int, output_block: bool) -> int:
        """AttentionBlock heads (reference :239-245); output blocks are built without num_heads (:517-523)."""
        if self.num_head_channels != -1:
            return ch // self.num_head_channels
        return 1 if output_block else self.num_heads

    def attention_layers(self):
        """(channels, in an output block) of every AttentionBlock."""
        from .arch import unetmodel_block_plan
        ins, mid, outs = unetmodel_block_plan(self)
        return ([(l[1], False) for b in ins + [mid] for l in b if l[0] == "attn"]
                + [(l[1], True) for b in outs for l in b if l[0] == "attn"])

    @property
    def lq_factor(self) -> int:
        """1: lq enters at the latent size; 2: at twice it, through F.pixel_unshuffle(lq, 2) (reference :569-573)."""
        return 2 if self.in_channels - self.x_channels == 12 else 1

    @property
    def x_channels(self) -> int:
        """Channels of x (the latent): out_channels, or out_channels / 2 when the model also outputs a learned variance
        (learn_sigma).  Where both readings fit (e.g. in 21, out 18) the fixed-variance one wins."""
        return _x_channels(self.in_channels, self.out_channels)

    @property
    def time_embed_dim(self) -> int:
        return self.model_channels * 4

    def to_kwargs(self) -> dict:
        d = asdict(self)
        d["num_res_blocks"] = list(self.num_res_blocks)
        d["channel_mult"] = list(self.channel_mult)
        d["attention_resolutions"] = list(self.attention_resolutions)
        return d


@dataclass
class UNetModelConvConfig:
    """Exactly the keyword arguments of ``UNetModelConv.__init__`` (reference models/unet.py:1026-1040), the UNet of
    attention- and GroupNorm-free ``ResBlockConv`` blocks.  What the native kernels cannot run is refused here with the
    reason.  ``use_fp16`` is accepted and has no effect: precision is fixed by the kernels."""
    in_channels: int = 6
    model_channels: int = 160
    out_channels: int = 3
    num_res_blocks: Sequence[int] = (2, 2, 2, 2)
    cond_lq: bool = True
    channel_mult: Sequence[int] = (1, 2, 4, 8)
    conv_resample: bool = True
    dims: int = 2
    use_scale_shift_norm: bool = False
    resblock_updown: bool = False
    use_fp16: bool = False

    def __post_init__(self):
        if isinstance(self.num_res_blocks, int):
            self.num_res_blocks = (self.num_res_blocks,) * len(self.channel_mult)
        self.num_res_blocks = tuple(int(v) for v in self.num_res_blocks)
        self.channel_mult = tuple(int(v) for v in self.channel_mult)
        if len(self.num_res_blocks) != len(self.channel_mult):
            raise ValueError("num_res_blocks and channel_mult must have the same length")
        if not 1 <= len(self.channel_mult) <= 8:
            raise ValueError(f"{len(self.channel_mult)} levels: the engine takes 1 to 8")
        if self.dims != 2:
            raise ValueError(f"dims={self.dims}: only 2-D UNets are covered (every ResShift config uses dims=2)")
        if not self.cond_lq:
            raise ValueError("cond_lq=False: the ResShift sampler always passes lq, and the reference asserts cond_lq then")
        if _x_channels(self.in_channels, self.out_channels) is None:
            raise ValueError(f"in_channels={self.in_channels}, out_channels={self.out_channels}: x has out_channels "
                             f"channels and lq is a 3-channel image, so in_channels must be out_channels + 3 (lq at the "
                             f"latent size) or out_channels + 12 (lq at twice it, through pixel_unshuffle); with a "
                             f"learned variance (even out_channels) x has out_channels / 2 channels, and in_channels "
                             f"is out_channels / 2 + 3 or + 12")
        for level, mult in enumerate(self.channel_mult):
            if mult <= 0 or self.model_channels <= 0 or (self.model_channels * mult) % 8:
                raise ValueError(f"level {level} has {self.model_channels * mult} channels: the conv kernels read and "
                                 f"write 16-byte channel rows, so model_channels * channel_mult must be a positive "
                                 f"multiple of 8")

    @property
    def lq_factor(self) -> int:
        """1: lq enters at the latent size; 2: at twice it, through F.pixel_unshuffle(lq, 2) (reference :1166-1167)."""
        return 2 if self.in_channels - self.x_channels == 12 else 1

    @property
    def x_channels(self) -> int:
        """Channels of x (the latent): out_channels, or out_channels / 2 when the model also outputs a learned variance
        (learn_sigma).  Where both readings fit (e.g. in 21, out 18) the fixed-variance one wins."""
        return _x_channels(self.in_channels, self.out_channels)

    @property
    def time_embed_dim(self) -> int:
        return self.model_channels * 4

    def to_kwargs(self) -> dict:
        d = asdict(self)
        d["num_res_blocks"] = list(self.num_res_blocks)
        d["channel_mult"] = list(self.channel_mult)
        return d


@dataclass
class DiffusionConfig:
    normalize_input: bool = True
    schedule_name: str = "exponential"
    sf: int = 4
    min_noise_level: float = 0.04
    steps: int = 15
    kappa: float = 2.0
    etas_end: float = 0.99
    schedule_kwargs: dict = field(default_factory=lambda: {"power": 0.3})
    weighted_mse: bool = False
    predict_type: str = "xstart"
    timestep_respacing: Optional[int] = None
    scale_factor: float = 1.0
    latent_flag: bool = True

    def to_kwargs(self) -> dict:
        return asdict(self)


# ---------------------------------------------------------------------------------
# Presets: configs/<name>.yaml  ->  (UNetConfig, DiffusionConfig, latent channels)
# ---------------------------------------------------------------------------------

def preset(name: str, steps: Optional[int] = None) -> Tuple[UNetConfig, DiffusionConfig]:
    if name in ("realsr", "realsr_swinunet_realesrgan256"):
        # configs/realsr_swinunet_realesrgan256.yaml: T=15, min_noise_level 0.04
        u = UNetConfig()
        d = DiffusionConfig()
    elif name in ("realsr_journal", "realsr_swinunet_realesrgan256_journal", "v3", "realsr_v3"):
        # configs/realsr_swinunet_realesrgan256_journal.yaml:38-73 (T=4 native)
        u = UNetConfig()
        d = DiffusionConfig(min_noise_level=0.2, steps=4)
    elif name in ("bicsr", "bicx4_swinunet_lpips"):
        u = UNetConfig()
        d = DiffusionConfig(min_noise_level=0.2, steps=4)
    elif name in ("faceir", "faceir_gfpgan512_lpips"):
        # configs/faceir_gfpgan512_lpips.yaml: f8 VQ (8 latent channels), LQ at 512
        u = UNetConfig(in_channels=8, out_channels=8, lq_size=512)
        d = DiffusionConfig(sf=1, min_noise_level=0.2, steps=4)
    elif name in ("inpaint", "inpaint_imagenet", "inpaint_lama256_imagenet", "inpaint_face", "inpaint_lama256_face"):
        # configs/inpaint_lama256_imagenet.yaml and inpaint_lama256_face.yaml: identical denoiser / schedule; they differ in
        # the VQ-GAN checkpoint only (autoencoder_vq_f4.pth vs celeba256_vq_f4_dim3_face.pth, same f4 architecture)
        u = UNetConfig(cond_mask=True, lq_size=256)
        d = DiffusionConfig(sf=1, min_noise_level=0.2, steps=4)
    elif name in ("realsr_x2", "realsr_realesrgan256_x2"):
        # configs/realsr_realesrgan256_x2.yaml: x2 SR — the LQ image enters at 128x128 through a one-stage feature extractor
        u = UNetConfig(lq_size=128)
        d = DiffusionConfig(sf=2, min_noise_level=0.2, steps=4)
    elif name == "tiny":
        # not a shipped config: a narrow model with the same topology, for fast tests
        u = UNetConfig(model_channels=32, swin_embed_dim=64)
        d = DiffusionConfig(steps=4, min_noise_level=0.2)
    elif name == "tiny_faceir":
        # narrow model with the face-restoration topology: 8 latent channels, three-stage LQ feature extractor at 512
        u = UNetConfig(model_channels=32, swin_embed_dim=64, in_channels=8, out_channels=8, lq_size=512)
        d = DiffusionConfig(sf=1, steps=4, min_noise_level=0.2)
    elif name == "tiny_inpaint":
        u = UNetConfig(model_channels=32, swin_embed_dim=64, cond_mask=True, lq_size=256)
        d = DiffusionConfig(sf=1, steps=4, min_noise_level=0.2)
    else:
        raise KeyError(f"unknown preset {name!r}")
    if steps is not None:
        d.steps = steps
    return u, d


def preset_vq_name(name: str) -> str:
    """VQ-GAN architecture (resshift_b200.vq_arch.vq_preset) each task's yaml names in its `autoencoder:` block."""
    return "f8_face" if name in ("faceir", "faceir_gfpgan512_lpips", "tiny_faceir") else "f4"


# inference_resshift.py --task / --version -> preset (reference inference_resshift.py:15-35,77-126)
TASKS = {
    ("realsr", "v1"): "realsr", ("realsr", "v2"): "realsr", ("realsr", "v3"): "realsr_journal",
    ("bicsr", None): "bicsr", ("inpaint_imagenet", None): "inpaint_imagenet", ("inpaint_face", None): "inpaint_face",
    ("faceir", None): "faceir",
}
