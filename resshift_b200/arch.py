"""Parameter / buffer inventory of the Swin-UNet denoiser, by reference ``state_dict`` name.

The names and shapes restate what ``UNetModelSwin.__init__`` registers (reference
models/unet.py:659-863; ``ResBlock`` :110-184; ``BasicLayer`` / ``SwinTransformerBlock`` /
``WindowAttention`` in models/swin_transformer.py:65-112,163-212,348-425), so that a
released ``.pth`` loads into this package's module unchanged (reference
utils/util_net.py:86-98 iterates the *model's* keys and looks each up in the checkpoint).

Each entry is ``(name, shape, role)``; roles drive packing into the kernel-native arena:

    conv3   Conv2d 3x3 weight  [O, I, 3, 3]
    conv1   Conv2d 1x1 weight  [O, I, 1, 1]
    linear  Linear weight      [O, I]
    bias    conv / linear bias [O]
    gn_w / gn_b   GroupNorm32 affine [C]
    relpos  relative_position_bias_table [(2w-1)^2, heads]
    buf_relidx    relative_position_index buffer [w*w, w*w] (int64)
    buf_mask      attn_mask buffer [nW, w*w, w*w] (float32), shifted blocks only
"""
from __future__ import annotations

from typing import List, Tuple

from .config import UNetConfig, UNetModelConfig, UNetModelConvConfig

Spec = Tuple[str, Tuple[int, ...], str]


def _conv(name: str, cin: int, cout: int, k: int) -> List[Spec]:
    return [(f"{name}.weight", (cout, cin, k, k), "conv3" if k == 3 else "conv1"),
            (f"{name}.bias", (cout,), "bias")]


def _linear(name: str, cin: int, cout: int) -> List[Spec]:
    return [(f"{name}.weight", (cout, cin), "linear"), (f"{name}.bias", (cout,), "bias")]


def _gn(name: str, c: int) -> List[Spec]:
    return [(f"{name}.weight", (c,), "gn_w"), (f"{name}.bias", (c,), "gn_b")]


def _resblock(name: str, cin: int, cout: int, emb: int, scale_shift: bool = True) -> List[Spec]:
    s: List[Spec] = []
    s += _gn(f"{name}.in_layers.0", cin)
    s += _conv(f"{name}.in_layers.2", cin, cout, 3)
    s += _linear(f"{name}.emb_layers.1", emb, (2 if scale_shift else 1) * cout)
    s += _gn(f"{name}.out_layers.0", cout)
    s += _conv(f"{name}.out_layers.3", cout, cout, 3)
    if cin != cout:
        s += _conv(f"{name}.skip_connection", cin, cout, 1)
    return s


def swin_geometry(cfg: UNetConfig, res: int) -> Tuple[int, int]:
    """(window, shift of the odd blocks) at a square resolution ``res``
    (reference models/swin_transformer.py:191-194: no partition / shift when res <= window)."""
    if res <= cfg.window_size:
        return res, 0
    return cfg.window_size, cfg.window_size // 2


def latent_multiple(cfg) -> int:
    """What H and W of a latent must be multiples of: every level's map (H / 2^level) is tiled by that level's window
    (UNetModel: the levels only have to halve evenly)."""
    import math
    if isinstance(cfg, (UNetModelConfig, UNetModelConvConfig)):
        return 2 ** (len(cfg.channel_mult) - 1)
    m = 1
    for level in range(len(cfg.channel_mult)):
        m = math.lcm(m, swin_geometry(cfg, cfg.image_size >> level)[0] << level)
    return m


def _basic_layer(name: str, cfg: UNetConfig, c: int, res: int) -> List[Spec]:
    e, heads = cfg.swin_embed_dim, cfg.swin_heads
    win, shift = swin_geometry(cfg, res)
    hidden = int(e * cfg.mlp_ratio)
    s: List[Spec] = []
    s += _conv(f"{name}.patch_embed.proj", c, e, 1)
    if cfg.patch_norm:
        s += _gn(f"{name}.patch_embed.norm", e)
    s += _conv(f"{name}.patch_unembed.proj", e, c, 1)
    if cfg.patch_norm:
        s += _gn(f"{name}.patch_unembed.norm", c)
    for i in range(cfg.swin_depth):
        b = f"{name}.blocks.{i}"
        if i % 2 == 1 and shift > 0:
            nw = (res // win) ** 2
            s.append((f"{b}.attn_mask", (nw, win * win, win * win), "buf_mask"))
        s += _gn(f"{b}.norm1", e)
        s.append((f"{b}.attn.relative_position_bias_table", ((2 * win - 1) ** 2, heads), "relpos"))
        s.append((f"{b}.attn.relative_position_index", (win * win, win * win), "buf_relidx"))
        s += _linear(f"{b}.attn.qkv", e, 3 * e)
        s += _linear(f"{b}.attn.proj", e, e)
        s += _gn(f"{b}.norm2", e)
        s += _conv(f"{b}.mlp.fc1", e, hidden, 1)
        s += _conv(f"{b}.mlp.fc2", hidden, e, 1)
    return s


def unet_block_plan(cfg: UNetConfig):
    """Topology of the denoiser as a list of blocks, in execution order.

    Returns ``(input_blocks, middle, output_blocks)``; every block is a list of layer tuples
    ``("conv", cin, cout)``, ``("res", cin, cout)``, ``("swin", c, res)``,
    ``("down", c)``, ``("up", c)`` (a conv, or with ``conv_resample=False`` a parameterless pool / upsample), or with
    ``resblock_updown`` ``("res_down", c)``, ``("res_up", c)`` (ResBlocks with down / up = True);
    restates reference models/unet.py:704-857.
    """
    down = "res_down" if cfg.resblock_updown else "down"
    up = "res_up" if cfg.resblock_updown else "up"
    mc = cfg.model_channels
    ch = int(cfg.channel_mult[0] * mc)
    in_ch = cfg.in_channels + cfg.lq_feat_channels
    input_blocks = [[("conv", in_ch, ch)]]
    chans = [ch]
    ds = cfg.image_size
    for level, mult in enumerate(cfg.channel_mult):
        for jj in range(cfg.num_res_blocks[level]):
            layers = [("res", ch, int(mult * mc))]
            ch = int(mult * mc)
            if ds in cfg.attention_resolutions and jj == 0:
                layers.append(("swin", ch, ds))
            input_blocks.append(layers)
            chans.append(ch)
        if level != len(cfg.channel_mult) - 1:
            input_blocks.append([(down, ch)])
            chans.append(ch)
            ds //= 2
    middle = [("res", ch, ch), ("swin", ch, ds), ("res", ch, ch)]
    output_blocks = []
    for level, mult in list(enumerate(cfg.channel_mult))[::-1]:
        for i in range(cfg.num_res_blocks[level] + 1):
            ich = chans.pop()
            layers = [("res", ch + ich, int(mc * mult))]
            ch = int(mc * mult)
            if ds in cfg.attention_resolutions and i == 0:
                layers.append(("swin", ch, ds))
            if level and i == cfg.num_res_blocks[level]:
                layers.append((up, ch))
                ds *= 2
            output_blocks.append(layers)
    return input_blocks, middle, output_blocks


def unet_param_spec(cfg: UNetConfig) -> List[Spec]:
    emb = cfg.time_embed_dim
    s: List[Spec] = []
    s += _linear("time_embed.0", cfg.model_channels, emb)
    s += _linear("time_embed.2", emb, emb)
    # feature_extractor (reference models/unet.py:689-702): [conv3x3, SiLU, Downsample(conv s2)] per stage
    fc, bc = cfg.lq_in_channels, 16
    for st in range(cfg.fe_stages):
        s += _conv(f"feature_extractor.{3 * st}", fc, bc, 3)
        s += _conv(f"feature_extractor.{3 * st + 2}.op", bc, 2 * bc, 3)
        bc *= 2
        fc = bc
    input_blocks, middle, output_blocks = unet_block_plan(cfg)

    def emit(prefix: str, layers):
        out: List[Spec] = []
        for j, layer in enumerate(layers):
            kind = layer[0]
            if kind == "conv":
                out += _conv(f"{prefix}.{j}", layer[1], layer[2], 3)
            elif kind == "res":
                out += _resblock(f"{prefix}.{j}", layer[1], layer[2], emb, cfg.use_scale_shift_norm)
            elif kind in ("res_down", "res_up"):
                out += _resblock(f"{prefix}.{j}", layer[1], layer[1], emb, cfg.use_scale_shift_norm)
            elif kind == "swin":
                out += _basic_layer(f"{prefix}.{j}", cfg, layer[1], layer[2])
            elif kind == "down" and cfg.conv_resample:
                out += _conv(f"{prefix}.{j}.op", layer[1], layer[1], 3)
            elif kind == "up" and cfg.conv_resample:
                out += _conv(f"{prefix}.{j}.conv", layer[1], layer[1], 3)
        return out

    for i, layers in enumerate(input_blocks):
        s += emit(f"input_blocks.{i}", layers)
    s += emit("middle_block", middle)
    for i, layers in enumerate(output_blocks):
        s += emit(f"output_blocks.{i}", layers)
    ch0 = int(cfg.channel_mult[0] * cfg.model_channels)
    s += _gn("out.0", ch0)
    s += _conv("out.2", ch0, cfg.out_channels, 3)
    return s


def unetmodel_block_plan(cfg: UNetModelConfig):
    """Topology of UNetModel (reference models/unet.py:426-541) in the form of ``unet_block_plan``, with
    ``("attn", c, heads)`` for an AttentionBlock: one after EVERY ResBlock of an attention level, and in the middle."""
    down = "res_down" if cfg.resblock_updown else "down"
    up = "res_up" if cfg.resblock_updown else "up"
    mc = cfg.model_channels
    ch = int(cfg.channel_mult[0] * mc)
    input_blocks = [[("conv", cfg.in_channels, ch)]]
    chans = [ch]
    ds = cfg.image_size
    for level, mult in enumerate(cfg.channel_mult):
        for _ in range(cfg.num_res_blocks[level]):
            layers = [("res", ch, int(mult * mc))]
            ch = int(mult * mc)
            if ds in cfg.attention_resolutions:
                layers.append(("attn", ch, cfg.heads(ch, False)))
            input_blocks.append(layers)
            chans.append(ch)
        if level != len(cfg.channel_mult) - 1:
            input_blocks.append([(down, ch)])
            chans.append(ch)
            ds //= 2
    middle = [("res", ch, ch), ("attn", ch, cfg.heads(ch, False)), ("res", ch, ch)]
    output_blocks = []
    for level, mult in list(enumerate(cfg.channel_mult))[::-1]:
        for i in range(cfg.num_res_blocks[level] + 1):
            ich = chans.pop()
            layers = [("res", ch + ich, int(mc * mult))]
            ch = int(mc * mult)
            if ds in cfg.attention_resolutions:
                layers.append(("attn", ch, cfg.heads(ch, True)))
            if level and i == cfg.num_res_blocks[level]:
                layers.append((up, ch))
                ds *= 2
            output_blocks.append(layers)
    return input_blocks, middle, output_blocks


def unetmodel_param_spec(cfg: UNetModelConfig) -> List[Spec]:
    """UNetModel's ``state_dict`` (reference models/unet.py:416-547); AttentionBlock :246-255 (qkv / proj_out are conv1d
    weights [O, I, 1])."""
    emb = cfg.time_embed_dim
    s: List[Spec] = []
    s += _linear("time_embed.0", cfg.model_channels, emb)
    s += _linear("time_embed.2", emb, emb)
    input_blocks, middle, output_blocks = unetmodel_block_plan(cfg)

    def emit(prefix: str, layers):
        out: List[Spec] = []
        for j, layer in enumerate(layers):
            kind, p = layer[0], f"{prefix}.{j}"
            if kind == "conv":
                out += _conv(p, layer[1], layer[2], 3)
            elif kind == "res":
                out += _resblock(p, layer[1], layer[2], emb, cfg.use_scale_shift_norm)
            elif kind in ("res_down", "res_up"):
                out += _resblock(p, layer[1], layer[1], emb, cfg.use_scale_shift_norm)
            elif kind == "attn":
                c = layer[1]
                out += _gn(f"{p}.norm", c)
                out += [(f"{p}.qkv.weight", (3 * c, c, 1), "conv1"), (f"{p}.qkv.bias", (3 * c,), "bias")]
                out += [(f"{p}.proj_out.weight", (c, c, 1), "conv1"), (f"{p}.proj_out.bias", (c,), "bias")]
            elif kind == "down" and cfg.conv_resample:
                out += _conv(f"{p}.op", layer[1], layer[1], 3)
            elif kind == "up" and cfg.conv_resample:
                out += _conv(f"{p}.conv", layer[1], layer[1], 3)
        return out

    for i, layers in enumerate(input_blocks):
        s += emit(f"input_blocks.{i}", layers)
    s += emit("middle_block", middle)
    for i, layers in enumerate(output_blocks):
        s += emit(f"output_blocks.{i}", layers)
    ch0 = int(cfg.channel_mult[0] * cfg.model_channels)
    s += _gn("out.0", ch0)
    s += _conv("out.2", ch0, cfg.out_channels, 3)
    return s


def unetconv_block_plan(cfg: UNetModelConvConfig):
    """Topology of UNetModelConv (reference models/unet.py:1064-1146) in the form of ``unet_block_plan``: ``res`` layers
    are ResBlockConv, no attention, two ResBlockConv in the middle."""
    down = "res_down" if cfg.resblock_updown else "down"
    up = "res_up" if cfg.resblock_updown else "up"
    mc = cfg.model_channels
    ch = int(cfg.channel_mult[0] * mc)
    input_blocks = [[("conv", cfg.in_channels, ch)]]
    chans = [ch]
    for level, mult in enumerate(cfg.channel_mult):
        for _ in range(cfg.num_res_blocks[level]):
            input_blocks.append([("res", ch, int(mult * mc))])
            ch = int(mult * mc)
            chans.append(ch)
        if level != len(cfg.channel_mult) - 1:
            input_blocks.append([(down, ch)])
            chans.append(ch)
    middle = [("res", ch, ch), ("res", ch, ch)]
    output_blocks = []
    for level, mult in list(enumerate(cfg.channel_mult))[::-1]:
        for i in range(cfg.num_res_blocks[level] + 1):
            ich = chans.pop()
            layers = [("res", ch + ich, int(mc * mult))]
            ch = int(mc * mult)
            if level and i == cfg.num_res_blocks[level]:
                layers.append((up, ch))
            output_blocks.append(layers)
    return input_blocks, middle, output_blocks


def _resblock_conv(name: str, cin: int, cout: int, emb: int, scale_shift: bool) -> List[Spec]:
    """ResBlockConv (reference models/unet.py:914-982): in_layers = [SiLU, conv], out_layers = [SiLU, conv]."""
    s: List[Spec] = []
    s += _conv(f"{name}.in_layers.1", cin, cout, 3)
    s += _linear(f"{name}.emb_layers.1", emb, (2 if scale_shift else 1) * cout)
    s += _conv(f"{name}.out_layers.1", cout, cout, 3)
    if cin != cout:
        s += _conv(f"{name}.skip_connection", cin, cout, 1)
    return s


def unetconv_param_spec(cfg: UNetModelConvConfig) -> List[Spec]:
    """UNetModelConv's ``state_dict`` (reference models/unet.py:1057-1151): no GroupNorm parameters, head ``out.1``."""
    emb = cfg.time_embed_dim
    s: List[Spec] = []
    s += _linear("time_embed.0", cfg.model_channels, emb)
    s += _linear("time_embed.2", emb, emb)
    input_blocks, middle, output_blocks = unetconv_block_plan(cfg)

    def emit(prefix: str, layers):
        out: List[Spec] = []
        for j, layer in enumerate(layers):
            kind, p = layer[0], f"{prefix}.{j}"
            if kind == "conv":
                out += _conv(p, layer[1], layer[2], 3)
            elif kind == "res":
                out += _resblock_conv(p, layer[1], layer[2], emb, cfg.use_scale_shift_norm)
            elif kind in ("res_down", "res_up"):
                out += _resblock_conv(p, layer[1], layer[1], emb, cfg.use_scale_shift_norm)
            elif kind == "down" and cfg.conv_resample:
                out += _conv(f"{p}.op", layer[1], layer[1], 3)
            elif kind == "up" and cfg.conv_resample:
                out += _conv(f"{p}.conv", layer[1], layer[1], 3)
        return out

    for i, layers in enumerate(input_blocks):
        s += emit(f"input_blocks.{i}", layers)
    s += emit("middle_block", middle)
    for i, layers in enumerate(output_blocks):
        s += emit(f"output_blocks.{i}", layers)
    s += _conv("out.1", int(cfg.channel_mult[0] * cfg.model_channels), cfg.out_channels, 3)
    return s


# -- derived buffers -----------------------------------------------------------------

def relative_position_index(win: int):
    """[win*win, win*win] int64 index into the (2win-1)^2 bias table
    (restates reference models/swin_transformer.py:93-103)."""
    import torch
    ys, xs = torch.meshgrid(torch.arange(win), torch.arange(win), indexing="ij")
    ys, xs = ys.reshape(-1), xs.reshape(-1)
    dy = ys[:, None] - ys[None, :] + (win - 1)
    dx = xs[:, None] - xs[None, :] + (win - 1)
    return (dy * (2 * win - 1) + dx).long()


def shifted_window_mask(h: int, w: int, win: int, shift: int):
    """[nW, win*win, win*win] float mask (0 / -100) for shifted windows.

    Restates what reference models/swin_transformer.py:214-236 *computes*, which is not the
    textbook Swin mask.  Two quirks compose:

    1. ``img_mask`` is allocated as [1, 1, H, W] but indexed ``[:, h, w, :]``: the "h" slices
       hit the singleton dim (only ``slice(-shift, None)`` is non-empty there) and the "w"
       slices land on the ROW axis, so the region label of a pixel depends on its row only —
       rows [0, H-win) / [H-win, H-shift) / [H-shift, H).
    2. after ``window_partition`` ([nW, r, c, 1]) the extra ``.permute(0, 2, 3, 1)`` (written
       for an NHWC partition) flattens each window as (c, r), i.e. transposed with respect to
       the token order r*win + c used by the attention.

    Net effect: token (r, c) of window (wy, wx) carries label rows[wy*win + c].  Only the last
    row of windows is affected: there, tokens in columns [0, win-shift) and [win-shift, win)
    are masked from each other.  Released checkpoints were trained with this mask, so parity
    means reproducing it exactly.
    """
    import torch

    rows = torch.zeros(h, dtype=torch.long)
    rows[h - win:h - shift] = 1
    rows[h - shift:] = 2
    lab = rows[:, None].expand(h, w)                                     # quirk 1: row-only labels
    lab = lab.reshape(h // win, win, w // win, win).permute(0, 2, 3, 1)  # [wy, wx, c, r]  (quirk 2)
    lab = lab.reshape(-1, win * win)
    diff = lab[:, None, :] - lab[:, :, None]
    return torch.where(diff != 0, torch.tensor(-100.0), torch.tensor(0.0))
