"""``VQModelTorch``, ``AutoencoderKLTorch`` and ``EncoderKLTorch`` — same constructors, ``state_dict`` and call surface
as the reference's ``ldm.models.autoencoder`` classes (reference ldm/models/autoencoder.py:12-112), the first stages
around the denoising loop (SURVEY.md §8f rank 1), executed by the sm_90a kernels of ``librs_b200.so``: the same wgmma
implicit-GEMM conv / GroupNorm kernels as the denoiser, the bottleneck's single-head attention as tensor-core GEMMs + a
row softmax up to 8192 positions and as one fused online-softmax kernel above (any image whose size is a multiple of
8 * 2^(levels-1)), nearest-codebook quantisation (VQ) or quant_conv + posterior sampling (KL) as one small kernel
(csrc/vq.inc, csrc/vq_attn.cuh, csrc/vq_kernels.cuh).

``VQModelTorch``: ``encode(x)`` / ``decode(h, force_not_quantize=False)`` / ``decode_code(code_b)`` / ``forward``.
``AutoencoderKLTorch``: ``encode(x, sample_posterior=True, return_moments=False)`` / ``decode(z)`` / ``forward``; the
posterior noise is drawn as the reference draws it (``torch.randn`` on the CPU default generator) unless the caller
passes it as ``posterior_noise=``.  All take and return fp32 NCHW CUDA tensors.  PyTorch owns every allocation; there
is no eager / CPU fallback.

``with ae.attention_team(member, size, exchange):`` splits the fused bottleneck attention's query rows over a team of
processes (DESIGN.md §6): each member computes its share of the rows and ``exchange`` fills in the others', so the
result is bit-identical to computing all rows here.
"""
from __future__ import annotations

import ctypes as C
from contextlib import contextmanager
from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from .. import _lib
from ..parallel import shard_range
from ..vq_arch import VQConfig, kl_param_spec, random_kl_state_dict, random_vq_state_dict, vq_param_spec


class _Node(nn.Module):
    """Anonymous container; only there so that ``state_dict`` keys match the reference's."""


def _config(ddconfig, embed_dim, n_embed=0, kl=False) -> VQConfig:
    """The VQConfig of a reference ``ddconfig`` (the keyword arguments of Encoder / Decoder, model.py:452-470,563-581);
    ValueError names what the native kernels do not run."""
    dd = dict(ddconfig)
    if dd.get("give_pre_end", False):
        raise ValueError("give_pre_end=True: the decoder would return its pre-norm features instead of an image "
                         "(ldm/modules/diffusionmodules/model.py:651-652); only image decoders are supported")
    attn_type = dd.get("attn_type", "vanilla")
    if dd.get("use_linear_attn", False):
        raise ValueError("use_linear_attn=True selects attn_type 'linear', for which the reference's make_attn raises "
                         "NotImplementedError (ldm/modules/diffusionmodules/model.py:280-298)")
    return VQConfig(embed_dim=embed_dim, n_embed=n_embed, z_channels=dd["z_channels"], resolution=dd.get("resolution", 256),
                    in_channels=dd.get("in_channels", 3), out_ch=dd.get("out_ch", 3), ch=dd["ch"],
                    ch_mult=tuple(dd["ch_mult"]), num_res_blocks=dd["num_res_blocks"],
                    attn_resolutions=tuple(dd.get("attn_resolutions", ())), dropout=dd.get("dropout", 0.0),
                    double_z=dd.get("double_z", kl), kl=kl, attn_type=attn_type,
                    resamp_with_conv=dd.get("resamp_with_conv", True), tanh_out=dd.get("tanh_out", False))


class _FirstStage(nn.Module):
    """What the first stages share: reference-named parameters, the native engine and its weight arena, one plan per
    (pass, batch, image size), and attention teams.  ``_create`` is the engine constructor of the C ABI."""

    _create = "rs_vq_create_ex"
    _name = "VQModelTorch"
    _encoder_only = False          # the module holds the encoder's parameters only (the engine lists the decoder's too)

    def __init__(self, cfg: VQConfig, spec, init: Dict[str, torch.Tensor]):
        super().__init__()
        self.cfg = cfg
        self._spec = spec
        for name, shape, role in self._spec:
            *path, leaf = name.split(".")
            node = self
            for part in path:
                if not hasattr(node, part):
                    node.add_module(part, _Node())
                node = getattr(node, part)
            node.register_parameter(leaf, nn.Parameter(init[name]))
        self._engine = None
        self._arena: Optional[torch.Tensor] = None
        self._packed_versions: Optional[Tuple] = None
        self._plans: Dict[Tuple[int, int, int, int], "_VQPlan"] = {}
        self._team: Optional[Tuple[int, int, Callable]] = None
        # (which, row_begin, row_end) of every team-split attention since the last attention_team() entry: 0 encode, 1 decode
        self.attention_rows: List[Tuple[int, int, int]] = []

    # ------------------------------------------------------------------ native plumbing
    def _ensure_engine(self, device: torch.device):
        if device.type != "cuda":
            raise RuntimeError(f"resshift_b200.{self._name} runs on CUDA only (no CPU fallback); call .cuda() first")
        if self._engine is None:
            h = C.c_void_p()
            cfgc, optc = _lib.make_vq_config(self.cfg), _lib.make_vq_options(self.cfg)
            _lib.check(getattr(_lib.lib, self._create)(C.byref(cfgc), C.byref(optc), C.byref(h)))
            self._engine = h
            n = _lib.lib.rs_unet_param_count(h)
            theirs = []
            buf = C.create_string_buffer(256)
            shape = (C.c_int32 * 4)()
            nd, isb = C.c_int32(), C.c_int32()
            for i in range(n):
                _lib.check(_lib.lib.rs_unet_param_info(h, i, buf, 256, shape, C.byref(nd), C.byref(isb)))
                theirs.append(buf.value.decode())
            if not self._inventory_matches(theirs):
                raise _lib.RsError("parameter inventory of librs_b200 does not match resshift_b200.vq_arch")
        if self._arena is None or self._arena.device != device:
            nbytes = _lib.lib.rs_unet_arena_bytes(self._engine)
            self._arena = torch.zeros(nbytes + 256, dtype=torch.uint8, device=device)
            self._arena_ptr = (self._arena.data_ptr() + 255) // 256 * 256
            with torch.cuda.device(device):                   # the engine belongs to the arena's device
                _lib.check(_lib.lib.rs_unet_set_arena(self._engine, self._arena_ptr))
            self._packed_versions = None
            self._plans.clear()
        return self._engine

    def _inventory_matches(self, theirs) -> bool:
        mine = [name for name, _, _ in self._spec]
        return set(mine) <= set(theirs) if self._encoder_only else sorted(theirs) == sorted(mine)

    def pack_weights(self, force: bool = False):
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
        torch.cuda.current_stream().synchronize()
        self._packed_versions = versions

    def plan(self, which: int, batch: int, image_h: int, image_w: int) -> "_VQPlan":
        device = next(self.parameters()).device
        self._ensure_engine(device)
        self.pack_weights()
        key = (which, batch, image_h, image_w)
        if key not in self._plans:
            self._plans[key] = _VQPlan(self, which, batch, image_h, image_w, device)
        return self._plans[key]

    def probe(self, which: int, batch: int, image_h: int, image_w: int, block: str) -> torch.Tensor:
        """A tensor of the LAST pass of plan (which, batch, image_h, image_w) as fp32 NCHW: an attention block's
        ``<prefix>.in``, ``.norm``, ``.q``, ``.k``, ``.attn`` (before proj_out) or ``<prefix>`` (its output), or the
        decoder's ``quantize`` (post_quant_conv's output).  Needs RS_NO_REUSE=1 when the plan is created to be valid for
        every tensor."""
        plan = self.plan(which, batch, image_h, image_w)
        return _lib.probe(plan.handle, batch, block, plan.workspace.device)

    def _encode_plan(self, x, what):
        """The encode plan of image batch ``x`` and ``x`` as contiguous fp32."""
        if x.device.type != "cuda":
            raise RuntimeError(f"resshift_b200.{self._name}.{what} needs CUDA tensors (no CPU fallback)")
        b, c, hh, ww = x.shape
        if c != self.cfg.in_channels:
            raise ValueError(f"expected {self.cfg.in_channels} input channels, got {c}")
        return self.plan(0, b, hh, ww), x.detach().float().contiguous()

    def _decode_plan(self, h, what):
        """The decode plan of latent batch ``h`` and ``h`` as contiguous fp32."""
        if h.device.type != "cuda":
            raise RuntimeError(f"resshift_b200.{self._name}.{what} needs CUDA tensors (no CPU fallback)")
        b, c, lh, lw = h.shape
        if c != self.cfg.embed_dim:
            raise ValueError(f"expected {self.cfg.embed_dim} latent channels, got {c}")
        f = self.cfg.downscale
        return self.plan(1, b, lh * f, lw * f), h.detach().float().contiguous()

    def _latent(self, x):
        b, _, hh, ww = x.shape
        f = self.cfg.downscale
        return torch.empty(b, self.cfg.embed_dim, hh // f, ww // f, dtype=torch.float32, device=x.device)

    def _image(self, h):
        b, _, lh, lw = h.shape
        f = self.cfg.downscale
        return torch.empty(b, self.cfg.out_ch, lh * f, lw * f, dtype=torch.float32, device=h.device)

    def _run(self, plan: "_VQPlan", which: int, begin: Callable[[], None], end: Callable[[], None], whole: Callable[[], None]):
        """One pass: split at every fused attention inside an attention team, else the single call ``whole``."""
        if self._team is not None and plan.attentions:
            self._run_team_split(plan, which, begin, end)
        else:
            whole()

    # ------------------------------------------------------------------ attention teams
    @contextmanager
    def attention_team(self, member: int, size: int, exchange: Callable[[torch.Tensor, int, int], None]):
        """Inside this context, ``encode`` / ``decode`` on a plan with fused attentions (attention blocks over more than
        8192 positions) compute only this member's query rows of each: 64-row blocks ``parallel.shard_range(T / 64,
        size, member)``.  After the part of the pass up to each such attention, ``exchange(view, row_begin, row_end)`` is
        called with that attention's output ``view`` ([N, T, C] fp16, on the current stream) and this member's rows; it
        must write every other member's rows into ``view``.  Then the pass goes on to the next one, and finishes.  Every
        member must run the same calls on the same inputs.  The attention rows are independent, so the result is
        bit-identical to a call outside the context.  Rows computed are recorded in ``attention_rows``, one entry per
        fused attention in pass order.  Plans without a fused attention run as usual."""
        if not (0 <= member < size):
            raise ValueError(f"team member {member} of {size}")
        if self._team is not None:
            raise RuntimeError("attention_team contexts do not nest")
        self._team = (member, size, exchange)
        self.attention_rows = []
        try:
            yield self
        finally:
            self._team = None

    def _run_team_split(self, plan: "_VQPlan", which: int, begin: Callable[[], None], end: Callable[[], None]):
        """_begin, then rs_vq_run_between for every further fused attention, then _end: each segment computes this
        member's rows of the attention it ends with, and ``exchange`` fills in the others' before the next one reads
        them."""
        member, size, exchange = self._team
        stream = _lib.current_stream()
        for a, view in enumerate(plan.attentions):
            t = view.shape[1]
            b0, e0 = shard_range(t // 64, size, member)
            rb, re = 64 * b0, 64 * e0
            _lib.check(_lib.lib.rs_vq_set_attention_rows_at(plan.handle, a, rb, re))
            try:
                if a == 0:
                    begin()
                else:
                    _lib.check(_lib.lib.rs_vq_run_between(plan.handle, a, stream))
            finally:
                _lib.check(_lib.lib.rs_vq_set_attention_rows_at(plan.handle, a, 0, t))
            exchange(view, rb, re)
            self.attention_rows.append((which, rb, re))
        end()

    def __del__(self):
        try:
            self._plans.clear()
            if self._engine is not None:
                _lib.lib.rs_unet_destroy(self._engine)
        except Exception:
            pass


class VQModelTorch(_FirstStage):
    def __init__(self, ddconfig, n_embed, embed_dim, remap=None, sane_index_shape=False):
        if remap is not None:
            raise NotImplementedError("codebook remapping is not used by any shipped config")
        cfg = _config(ddconfig, embed_dim, n_embed=n_embed)
        super().__init__(cfg, vq_param_spec(cfg), random_vq_state_dict(cfg, seed=0))
        self.sane_index_shape = sane_index_shape
        self.last_indices: Optional[torch.Tensor] = None

    # ------------------------------------------------------------------ reference call surface
    @torch.no_grad()
    def encode(self, x):
        """x [B, 3, H, W] -> h [B, embed_dim, H/f, W/f] (reference autoencoder.py:28-31)."""
        plan, xf = self._encode_plan(x, "encode")
        out = self._latent(x)
        stream = _lib.current_stream()
        self._run(plan, 0, lambda: _lib.check(_lib.lib.rs_vq_encode_begin(plan.handle, xf.data_ptr(), stream)),
                  lambda: _lib.check(_lib.lib.rs_vq_encode_end(plan.handle, out.data_ptr(), stream)),
                  lambda: _lib.check(_lib.lib.rs_vq_encode(plan.handle, xf.data_ptr(), out.data_ptr(), stream)))
        return out

    @torch.no_grad()
    def decode(self, h, force_not_quantize=False):
        """h [B, embed_dim, h, w] -> image [B, 3, h*f, w*f] (reference autoencoder.py:33-40); the code indices of the
        last call stay available as ``self.last_indices`` ([B, h, w] int32, -1 when not quantised)."""
        plan, hf = self._decode_plan(h, "decode")
        b, _, lh, lw = h.shape
        out = self._image(h)
        idx = torch.empty(b, lh, lw, dtype=torch.int32, device=h.device)
        stream, fnq = _lib.current_stream(), int(bool(force_not_quantize))
        self._run(plan, 1, lambda: _lib.check(_lib.lib.rs_vq_decode_begin(plan.handle, hf.data_ptr(), idx.data_ptr(), fnq, stream)),
                  lambda: _lib.check(_lib.lib.rs_vq_decode_end(plan.handle, out.data_ptr(), stream)),
                  lambda: _lib.check(_lib.lib.rs_vq_decode(plan.handle, hf.data_ptr(), out.data_ptr(), idx.data_ptr(), fnq, stream)))
        self.last_indices = idx
        return out

    @torch.no_grad()
    def decode_code(self, code_b):
        """code_b [B, h, w] integer code indices -> image [B, 3, h*f, w*f]: the codebook rows (quantize.embed_code), then
        decode(..., force_not_quantize=True) (reference autoencoder.py:42-45), bit-identical to that call.  Indices
        must lie in [0, n_embed); a position with any other index decodes from NaN."""
        if code_b.device.type != "cuda":
            raise RuntimeError("resshift_b200.VQModelTorch.decode_code needs CUDA tensors (no CPU fallback)")
        if code_b.dim() != 3 or code_b.dtype.is_floating_point or code_b.dtype.is_complex:
            raise ValueError(f"expected integer code indices [B, h, w], got {tuple(code_b.shape)} {code_b.dtype}")
        b, lh, lw = code_b.shape
        f = self.cfg.downscale
        plan = self.plan(1, b, lh * f, lw * f)
        idx = code_b.to(torch.int32).contiguous()
        out = torch.empty(b, self.cfg.out_ch, lh * f, lw * f, dtype=torch.float32, device=code_b.device)
        _lib.check(_lib.lib.rs_vq_decode_code(plan.handle, idx.data_ptr(), out.data_ptr(), _lib.current_stream()))
        return out

    def forward(self, input, force_not_quantize=False):
        return self.decode(self.encode(input), force_not_quantize)


class EncoderKLTorch(_FirstStage):
    """The encoder half of the KL first stage (reference autoencoder.py:88-112): ``encode`` / ``forward`` as in
    AutoencoderKLTorch; its ``state_dict`` holds only ``encoder.*`` and ``quant_conv.*``."""

    _create = "rs_kl_create_ex"
    _name = "EncoderKLTorch"
    _encoder_only = True
    # encode() samples the posterior by default: ResShiftSampler draws that noise ahead of the unit (posterior_noise=)
    samples_posterior = True

    def __init__(self, ddconfig, embed_dim):
        cfg = _config(ddconfig, embed_dim, kl=True)
        spec = kl_param_spec(cfg)
        if self._encoder_only:
            spec = [e for e in spec if e[0].startswith(("encoder.", "quant_conv."))]
        super().__init__(cfg, spec, random_kl_state_dict(cfg, seed=0))
        self.embed_dim = embed_dim

    @torch.no_grad()
    def encode(self, x, sample_posterior=True, return_moments=False, posterior_noise=None):
        """x [B, 3, H, W] -> z [B, embed_dim, H/f, W/f] (and the moments [B, 2 embed_dim, H/f, W/f] with
        ``return_moments``) — reference autoencoder.py:65-76 with DiagonalGaussianDistribution
        (ldm/modules/distributions/distributions.py:24-37,61-62): z = mean + exp(0.5 clamp(logvar, -30, 20)) * noise, or
        the mean without ``sample_posterior``.  The noise is ``posterior_noise`` when given (a [B, embed_dim, H/f, W/f]
        tensor), else ``torch.randn`` of that shape on the CPU default generator, as the reference draws it."""
        plan, xf = self._encode_plan(x, "encode")
        z = self._latent(x)
        moments = torch.empty(z.shape[0], 2 * z.shape[1], *z.shape[2:], dtype=torch.float32, device=x.device) \
            if return_moments else None
        noise = None
        if sample_posterior:
            if posterior_noise is None:
                posterior_noise = torch.randn(z.shape)         # the reference's draw: CPU generator, then to the device
            if tuple(posterior_noise.shape) != tuple(z.shape):
                raise ValueError(f"posterior_noise must have shape {tuple(z.shape)}, got {tuple(posterior_noise.shape)}")
            noise = posterior_noise.to(device=x.device, dtype=torch.float32).contiguous()
        stream = _lib.current_stream()
        args = (_lib.ptr(noise), z.data_ptr(), _lib.ptr(moments), stream)
        self._run(plan, 0, lambda: _lib.check(_lib.lib.rs_kl_encode_begin(plan.handle, xf.data_ptr(), stream)),
                  lambda: _lib.check(_lib.lib.rs_kl_encode_end(plan.handle, *args)),
                  lambda: _lib.check(_lib.lib.rs_kl_encode(plan.handle, xf.data_ptr(), *args)))
        return (z, moments) if return_moments else z

    def forward(self, x, sample_posterior=True, return_moments=False):
        return self.encode(x, sample_posterior, return_moments)


class AutoencoderKLTorch(EncoderKLTorch):
    """KL first stage (reference autoencoder.py:52-86): Encoder with double_z, quant_conv to the posterior's moments,
    post_quant_conv and Decoder."""

    _name = "AutoencoderKLTorch"
    _encoder_only = False

    @torch.no_grad()
    def decode(self, z):
        """z [B, embed_dim, h, w] -> image [B, 3, h*f, w*f] (reference autoencoder.py:78-81)."""
        plan, zf = self._decode_plan(z, "decode")
        out = self._image(z)
        stream = _lib.current_stream()
        self._run(plan, 1, lambda: _lib.check(_lib.lib.rs_kl_decode_begin(plan.handle, zf.data_ptr(), stream)),
                  lambda: _lib.check(_lib.lib.rs_kl_decode_end(plan.handle, out.data_ptr(), stream)),
                  lambda: _lib.check(_lib.lib.rs_kl_decode(plan.handle, zf.data_ptr(), out.data_ptr(), stream)))
        return out

    def forward(self, input, sample_posterior=True):
        return self.decode(self.encode(input, sample_posterior, return_moments=False))


class _VQPlan:
    """First-stage (VQ-GAN or KL) engine bound to (encode | decode, batch, image H, image W): owns the workspace and the
    native plan."""

    def __init__(self, model: _FirstStage, which: int, batch: int, image_h: int, image_w: int, device):
        self.model = model
        h = C.c_void_p()
        _lib.check(_lib.lib.rs_vq_plan_create(model._engine, batch, image_h, image_w, which, C.byref(h)))
        self.handle = h
        nbytes = _lib.lib.rs_plan_workspace_bytes(h)
        self.workspace = torch.empty(nbytes + 256, dtype=torch.uint8, device=device)
        self.workspace_ptr = (self.workspace.data_ptr() + 255) // 256 * 256
        _lib.check(_lib.lib.rs_plan_bind(h, self.workspace_ptr))
        self.launches = _lib.lib.rs_plan_num_launches(h)
        # each fused attention's output [N, T, C] fp16 as a view of the workspace, in pass order
        self.attentions: List[torch.Tensor] = []
        n = C.c_int32()
        _lib.check(_lib.lib.rs_vq_attention_count(h, C.byref(n)))
        ptr, rstride, istride, t, cc = C.c_void_p(), C.c_longlong(), C.c_longlong(), C.c_int32(), C.c_int32()
        for a in range(n.value):
            _lib.check(_lib.lib.rs_vq_attention_output_at(h, a, C.byref(ptr), C.byref(rstride), C.byref(istride), C.byref(t),
                                                          C.byref(cc)))
            off = ptr.value - self.workspace.data_ptr()
            assert off % 2 == 0 and self.workspace.numel() % 2 == 0
            self.attentions.append(torch.as_strided(self.workspace.view(torch.float16), (batch, t.value, cc.value),
                                                    (istride.value, rstride.value, 1), off // 2))
        # the first fused attention's output (None: the plan has none)
        self.attention: Optional[torch.Tensor] = self.attentions[0] if self.attentions else None

    def __del__(self):
        try:
            _lib.lib.rs_plan_destroy(self.handle)
        except Exception:
            pass
