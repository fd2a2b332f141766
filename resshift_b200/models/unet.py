"""``UNetModelSwin`` — same constructor, ``state_dict`` and call surface as the reference's
``models.unet.UNetModelSwin`` (reference models/unet.py:603-912), with the forward pass executed by
the sm_90a kernels of ``librs_b200.so`` through the C ABI (include/resshift_b200.h).

PyTorch owns every allocation (parameters, packed-weight arena, workspace, outputs); the library only
enqueues kernels on the current CUDA stream.  There is no eager / CPU fallback: calling the module
without a CUDA device or without the compiled library raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Tuple

import torch
import torch.nn as nn

from .. import _lib
from ..arch import unet_param_spec, relative_position_index, shifted_window_mask
from ..config import UNetConfig
from ..weights import random_state_dict


class _Node(nn.Module):
    """Anonymous container; only there so that ``state_dict`` keys match the reference's."""


class UNetModelSwin(nn.Module):
    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks,
                 attention_resolutions, dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2,
                 use_fp16=False, num_heads=1, num_head_channels=-1, use_scale_shift_norm=False,
                 resblock_updown=False, swin_depth=2, swin_embed_dim=96, window_size=8, mlp_ratio=2.0,
                 patch_norm=False, cond_lq=True, cond_mask=False, lq_size=256):
        super().__init__()
        self.cfg = UNetConfig(
            image_size=image_size, in_channels=in_channels, model_channels=model_channels,
            out_channels=out_channels, num_res_blocks=num_res_blocks,
            attention_resolutions=tuple(attention_resolutions), dropout=dropout, channel_mult=tuple(channel_mult),
            conv_resample=conv_resample, dims=dims, use_fp16=use_fp16, num_heads=num_heads,
            num_head_channels=num_head_channels, use_scale_shift_norm=use_scale_shift_norm,
            resblock_updown=resblock_updown, swin_depth=swin_depth, swin_embed_dim=swin_embed_dim,
            window_size=window_size, mlp_ratio=mlp_ratio, patch_norm=patch_norm, cond_lq=cond_lq,
            cond_mask=cond_mask, lq_size=lq_size)
        # attributes the reference exposes
        self.image_size, self.in_channels, self.model_channels = image_size, in_channels, model_channels
        self.out_channels, self.cond_lq, self.cond_mask = out_channels, cond_lq, cond_mask
        self.dtype = torch.float32

        self._spec = unet_param_spec(self.cfg)
        init = random_state_dict(self.cfg, seed=0)
        for name, shape, role in self._spec:
            *path, leaf = name.split(".")
            node = self
            for part in path:
                if not hasattr(node, part):
                    node.add_module(part, _Node())
                node = getattr(node, part)
            value = init[name]
            if role.startswith("buf_"):
                node.register_buffer(leaf, value)
            else:
                if name.endswith("out_layers.3.weight") or name.endswith("out_layers.3.bias"):
                    value = torch.zeros_like(value)         # zero_module (reference models/unet.py:172-174)
                node.register_parameter(leaf, nn.Parameter(value))

        # native state (created lazily on the first CUDA call)
        self._engine = None
        self._arena: Optional[torch.Tensor] = None
        self._packed_versions: Optional[Tuple] = None
        self._plans: Dict[Tuple[int, int, int], "_Plan"] = {}

    # ------------------------------------------------------------------ native plumbing
    def _ensure_engine(self, device: torch.device):
        if device.type != "cuda":
            raise RuntimeError("resshift_b200.UNetModelSwin runs on CUDA only (no CPU fallback); call .cuda() first")
        if self._engine is None:
            h = C.c_void_p()
            cfgc = _lib.make_config(self.cfg)
            _lib.check(_lib.lib.rs_unet_create(C.byref(cfgc), C.byref(h)))
            self._engine = h
            n = _lib.lib.rs_unet_param_count(h)
            mine = sorted(name for name, _, _ in self._spec)
            theirs = []
            buf = C.create_string_buffer(256)
            shape = (C.c_int32 * 4)()
            nd, isb = C.c_int32(), C.c_int32()
            for i in range(n):
                _lib.check(_lib.lib.rs_unet_param_info(h, i, buf, 256, shape, C.byref(nd), C.byref(isb)))
                theirs.append(buf.value.decode())
            if sorted(theirs) != mine:
                raise _lib.RsError("parameter inventory of librs_b200 does not match resshift_b200.arch")
        if self._arena is None or self._arena.device != device:
            nbytes = _lib.lib.rs_unet_arena_bytes(self._engine)
            self._arena = torch.zeros(nbytes + 256, dtype=torch.uint8, device=device)
            base = self._arena.data_ptr()
            self._arena_ptr = (base + 255) // 256 * 256
            _lib.check(_lib.lib.rs_unet_set_arena(self._engine, self._arena_ptr))
            self._packed_versions = None
            self._plans.clear()
        return self._engine

    def pack_weights(self, force: bool = False):
        """(Re)pack parameters into the kernel-native fp16/fp32 arena when they changed."""
        params = dict(self.named_parameters())
        self._ensure_engine(next(iter(params.values())).device)      # (a no-op once the engine and its arena exist)
        versions = tuple((p._version, p.data_ptr()) for p in params.values())
        if not force and versions == self._packed_versions:
            return
        stream = _lib.current_stream()
        for name, p in params.items():
            if p.device.type != "cuda":
                raise RuntimeError(f"parameter {name} is not on a CUDA device")
            src = p.detach()
            if src.dtype != torch.float32 or not src.is_contiguous():
                src = src.float().contiguous()
            _lib.check(_lib.lib.rs_unet_load_param(self._engine, name.encode(), src.data_ptr(), stream))
            del src
        torch.cuda.current_stream().synchronize()   # staging copies above may be freed after this
        self._packed_versions = versions

    def plan(self, batch: int, height: int, width: int) -> "_Plan":
        device = next(self.parameters()).device
        self._ensure_engine(device)
        self.pack_weights()
        key = (batch, height, width)
        if key not in self._plans:
            self._plans[key] = _Plan(self, batch, height, width, device)
        return self._plans[key]

    def num_launches(self, batch, height, width) -> int:
        return _lib.lib.rs_plan_num_launches(self.plan(batch, height, width).handle)

    # ------------------------------------------------------------------ reference call surface
    @torch.no_grad()
    def forward(self, x, timesteps, lq=None, mask=None):
        """x [N, C, H, W]; timesteps [N]; lq [N, 3, h, w]; mask [N, 1, h, w] or None -> [N, out_ch, H, W] fp32
        (reference models/unet.py:865-895; the reference returns fp16 under autocast, this returns fp32)."""
        if lq is None:
            raise ValueError("UNetModelSwin is LQ-conditioned (cond_lq=True in every shipped config): pass lq=")
        if x.device.type != "cuda":
            raise RuntimeError("resshift_b200.UNetModelSwin.forward needs CUDA tensors (no CPU fallback)")
        n, _, h, w = x.shape
        plan = self.plan(n, h, w)
        xf = x.detach().float().contiguous()
        tf = timesteps.detach().to(device=x.device, dtype=torch.float32).contiguous()
        lqf = lq.detach().float().contiguous()
        mf = mask.detach().float().contiguous() if mask is not None else None
        exp_lq = (n, 3, h << self.cfg.fe_stages, w << self.cfg.fe_stages)
        if tuple(lqf.shape) != exp_lq:
            raise ValueError(f"lq must have shape {exp_lq}, got {tuple(lqf.shape)}")
        out = torch.empty(n, self.cfg.out_channels, h, w, dtype=torch.float32, device=x.device)
        _lib.check(_lib.lib.rs_plan_forward(plan.handle, xf.data_ptr(), tf.data_ptr(), lqf.data_ptr(),
                                            _lib.ptr(mf), out.data_ptr(), _lib.current_stream()))
        return out

    def probe(self, batch, height, width, block: str) -> torch.Tensor:
        """Block output of the LAST forward as fp32 NCHW (needs RS_NO_REUSE=1 to be valid for every block)."""
        plan = self.plan(batch, height, width)
        c, hh, ww = C.c_int32(), C.c_int32(), C.c_int32()
        _lib.check(_lib.lib.rs_plan_probe(plan.handle, block.encode(), None, C.byref(c), C.byref(hh), C.byref(ww), None))
        out = torch.empty(batch, c.value, hh.value, ww.value, dtype=torch.float32, device=plan.workspace.device)
        _lib.check(_lib.lib.rs_plan_probe(plan.handle, block.encode(), out.data_ptr(), C.byref(c), C.byref(hh),
                                          C.byref(ww), _lib.current_stream()))
        return out

    def convert_to_fp16(self):   # reference API; precision is fixed by the kernels (fp16 storage, fp32 accumulate)
        return self

    def convert_to_fp32(self):
        return self

    def __del__(self):
        try:
            self._plans.clear()
            if self._engine is not None:
                _lib.lib.rs_unet_destroy(self._engine)
        except Exception:
            pass


class _Plan:
    """Engine bound to (batch, H, W): owns the workspace tensor and the native plan handle."""

    def __init__(self, model: UNetModelSwin, batch: int, height: int, width: int, device):
        self.model = model
        h = C.c_void_p()
        _lib.check(_lib.lib.rs_plan_create(model._engine, batch, height, width, C.byref(h)))
        self.handle = h
        nbytes = _lib.lib.rs_plan_workspace_bytes(h)
        self.workspace = torch.empty(nbytes + 256, dtype=torch.uint8, device=device)
        self.workspace_ptr = (self.workspace.data_ptr() + 255) // 256 * 256
        _lib.check(_lib.lib.rs_plan_bind(h, self.workspace_ptr))
        self.batch, self.height, self.width = batch, height, width
        self.samplers = {}

    def __del__(self):
        try:
            for s in self.samplers.values():
                _lib.lib.rs_sampler_destroy(s)
            _lib.lib.rs_plan_destroy(self.handle)
        except Exception:
            pass
