"""ResShift diffusion process: schedule + the residual-shift sampling loop.

Mirrors the call surface of the reference's ``GaussianDiffusion`` / ``SpacedDiffusion``
(reference models/gaussian_diffusion.py:107-609, models/respace.py:20-63) that inference uses:
``p_sample_loop``, ``p_sample_loop_progressive``, ``p_sample``, ``p_mean_variance``, ``prior_sample``,
``encode_first_stage``, ``decode_first_stage``, ``_scale_input``, ``q_sample``, ``num_timesteps``.

When the model is one of this package's UNets the whole T-step loop (input scaling, denoiser, the model output's
conversion to x0 for every predict_type, posterior mean, noise injection, next-input packing) runs inside
``librs_b200.so`` as one CUDA graph; for any other callable, with clipping or with a ``denoised_fn`` the per-step update
still runs through the library's ``rs_p_sample`` kernel.
The VQ-GAN bookends (``encode_first_stage`` / ``decode_first_stage``) stay in PyTorch.
Training (``training_losses``) is out of scope.
"""
from __future__ import annotations

import ctypes as C
import enum
import math
from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F

from .. import _lib
from .unet import UNetModel, UNetModelConv, UNetModelSwin


class ModelMeanType(enum.Enum):
    START_X = enum.auto()
    EPSILON = enum.auto()
    PREVIOUS_X = enum.auto()
    RESIDUAL = enum.auto()
    EPSILON_SCALE = enum.auto()


class LossType(enum.Enum):
    MSE = enum.auto()
    WEIGHTED_MSE = enum.auto()


def get_named_eta_schedule(schedule_name, num_diffusion_timesteps, min_noise_level, etas_end=0.99, kappa=1.0,
                           kwargs=None):
    """sqrt(eta_t) for t = 0..T-1 (reference models/gaussian_diffusion.py:32-66)."""
    if schedule_name != "exponential":
        raise ValueError(f"schedule {schedule_name!r} is not covered (only 'exponential' is used by the shipped configs)")
    power = (kwargs or {}).get("power", None)
    eta0 = min(min_noise_level / kappa, min_noise_level)
    T = num_diffusion_timesteps
    growth = math.exp(math.log(etas_end / eta0) / (T - 1))
    expo = np.linspace(0, 1, T, endpoint=True) ** power * (T - 1)
    return np.power(np.full([T], growth), expo) * eta0


def space_timesteps(num_timesteps, sample_timesteps):
    """reference models/respace.py:6-18"""
    return {int((num_timesteps / sample_timesteps) * x) for x in range(sample_timesteps)}


def bicubic_upsample(y, sf):
    """F.interpolate(y, scale_factor=sf, mode='bicubic') (reference models/gaussian_diffusion.py:503-504) — the library's
    kernel for fp32 CUDA tensors and integer factors (same A = -0.75 / half-pixel / border-clamp arithmetic as ATen)."""
    if y.is_cuda and y.dtype == torch.float32 and float(sf).is_integer():
        yc = y.contiguous()
        n, c, h, w = yc.shape
        out = torch.empty(n, c, h * int(sf), w * int(sf), dtype=torch.float32, device=y.device)
        _lib.check(_lib.lib.rs_op_bicubic_upsample(yc.data_ptr(), n, c, h, w, int(sf), out.data_ptr(), _lib.current_stream()))
        return out
    return F.interpolate(y, scale_factor=sf, mode="bicubic")


def _tab(arr, t, like):
    """``_extract_into_tensor`` (reference models/gaussian_diffusion.py:92-105): float64 table -> fp32 gather."""
    res = torch.from_numpy(np.asarray(arr)).to(device=t.device)[t].float()
    while res.dim() < like.dim():
        res = res[..., None]
    return res.expand(like.shape)


class ResShiftDiffusion:
    """``SpacedDiffusion(GaussianDiffusion)`` of the reference, inference side."""

    def __init__(self, *, use_timesteps, sqrt_etas, kappa, model_mean_type, loss_type, sf=4, scale_factor=None,
                 normalize_input=True, latent_flag=True):
        base = np.asarray(sqrt_etas, dtype=np.float64)
        self.original_num_steps = len(base)
        self.use_timesteps = set(use_timesteps)
        self.timestep_map = [i for i in range(len(base)) if i in self.use_timesteps]
        self.sqrt_etas = base[self.timestep_map]
        self.kappa, self.model_mean_type, self.loss_type = kappa, model_mean_type, loss_type
        self.scale_factor, self.normalize_input, self.latent_flag, self.sf = scale_factor, normalize_input, latent_flag, sf
        # posterior tables (reference models/gaussian_diffusion.py:135-174), float64
        self.etas = self.sqrt_etas ** 2
        assert (self.etas > 0).all() and (self.etas <= 1).all()
        self.num_timesteps = int(self.etas.shape[0])
        self.etas_prev = np.append(0.0, self.etas[:-1])
        self.alpha = self.etas - self.etas_prev
        self.posterior_variance = kappa ** 2 * self.etas_prev / self.etas * self.alpha
        self.posterior_variance_clipped = np.append(self.posterior_variance[1], self.posterior_variance[1:])
        self.posterior_log_variance_clipped = np.log(self.posterior_variance_clipped)
        self.posterior_mean_coef1 = self.etas_prev / self.etas
        self.posterior_mean_coef2 = self.alpha / self.etas

    # ------------------------------------------------------------------ small pieces (torch, boundary side)
    def _scale_input(self, inputs, t):
        """reference models/gaussian_diffusion.py:598-603"""
        if not self.normalize_input:
            return inputs
        if self.latent_flag:
            return inputs / torch.sqrt(_tab(self.etas, t, inputs) * self.kappa ** 2 + 1)
        return inputs / (_tab(self.sqrt_etas, t, inputs) * self.kappa * 3 + 1)

    def prior_sample(self, y, noise=None):
        """reference models/gaussian_diffusion.py:517-529"""
        if noise is None:
            noise = torch.randn_like(y)
        t = torch.full((y.shape[0],), self.num_timesteps - 1, device=y.device, dtype=torch.long)
        return y + _tab(self.kappa * self.sqrt_etas, t, y) * noise

    def q_sample(self, x_start, y, t, noise=None):
        """reference models/gaussian_diffusion.py:190-208"""
        if noise is None:
            noise = torch.randn_like(x_start)
        return _tab(self.etas, t, x_start) * (y - x_start) + x_start + _tab(self.sqrt_etas * self.kappa, t, x_start) * noise

    def encode_first_stage(self, y, first_stage_model, up_sample=False, posterior_noise=None):
        """reference models/gaussian_diffusion.py:500-515 (PyTorch bookend).  ``posterior_noise``: the noise of a first
        stage that samples its posterior (AutoencoderKLTorch.encode(posterior_noise=)); None lets it draw its own."""
        data_dtype = y.dtype
        if up_sample and self.sf != 1:
            y = bicubic_upsample(y, self.sf)
        if first_stage_model is None:
            return y
        model_dtype = next(first_stage_model.parameters()).dtype
        if model_dtype != data_dtype:
            y = y.type(model_dtype)
        with torch.no_grad():
            if posterior_noise is None:
                out = first_stage_model.encode(y) * self.scale_factor
            else:
                out = first_stage_model.encode(y, posterior_noise=posterior_noise) * self.scale_factor
        return out.type(data_dtype) if model_dtype != data_dtype else out

    def decode_first_stage(self, z_sample, first_stage_model=None, consistencydecoder=None):
        """reference models/gaussian_diffusion.py:474-498 (PyTorch bookend)"""
        if first_stage_model is None:
            return z_sample
        if consistencydecoder is not None:
            raise NotImplementedError("consistency decoder is outside the covered path")
        data_dtype = z_sample.dtype
        model_dtype = next(first_stage_model.parameters()).dtype
        with torch.no_grad():
            out = first_stage_model.decode((1 / self.scale_factor * z_sample).type(model_dtype))
        return out.type(data_dtype) if model_dtype != data_dtype else out

    # ------------------------------------------------------------------ one step (generic model callable)
    def step_tables(self):
        """The fp32 tables of every step (coef1, coef2, std, in_scale, timesteps) and the prior coefficient, computed by
        the library exactly as its sampler computes them (rs_schedule_tables), so that both paths step with the same
        bits."""
        if getattr(self, "_step_tables", None) is None:
            T = self.num_timesteps
            dst = (C.c_float * (5 * T + 1))()
            _lib.check(_lib.lib.rs_schedule_tables(T, (C.c_double * T)(*self.sqrt_etas.tolist()), float(self.kappa),
                                                   (C.c_int32 * T)(*self.timestep_map), dst))
            a = np.frombuffer(dst, dtype=np.float32).copy()
            self._step_tables = {k: a[j * T:(j + 1) * T] for j, k in enumerate(("coef1", "coef2", "std", "in_scale", "tsteps"))}
            self._step_tables["prior_coef"] = a[5 * T]
        return self._step_tables

    def _model_t(self, t):
        m = torch.tensor(self.timestep_map, device=t.device, dtype=t.dtype)   # reference models/respace.py:60-63
        return m[t]

    def p_mean_variance(self, model, x_t, y, t, clip_denoised=True, denoised_fn=None, model_kwargs=None):
        """reference models/gaussian_diffusion.py:234-307 (predict_type handling identical)."""
        model_kwargs = model_kwargs or {}
        out = model(self._scale_input(x_t, t), self._model_t(t), **model_kwargs)

        def proc(v):
            if denoised_fn is not None:
                v = denoised_fn(v)
            return v.clamp(-1, 1) if clip_denoised else v

        if self.model_mean_type == ModelMeanType.START_X:
            pred = proc(out)
        elif self.model_mean_type == ModelMeanType.RESIDUAL:
            pred = proc(y - out)
        elif self.model_mean_type == ModelMeanType.EPSILON:
            pred = proc((x_t - _tab(self.sqrt_etas, t, x_t) * self.kappa * out - _tab(self.etas, t, x_t) * y)
                        / _tab(1 - self.etas, t, x_t))
        elif self.model_mean_type == ModelMeanType.EPSILON_SCALE:
            pred = proc((x_t - out - _tab(self.etas, t, x_t) * y) / _tab(1 - self.etas, t, x_t))
        else:
            raise ValueError(self.model_mean_type)
        mean = _tab(self.posterior_mean_coef1, t, x_t) * x_t + _tab(self.posterior_mean_coef2, t, x_t) * pred
        return {"mean": mean, "variance": _tab(self.posterior_variance, t, x_t),
                "log_variance": _tab(self.posterior_log_variance_clipped, t, x_t), "pred_xstart": pred}

    def p_sample(self, model, x, y, t, clip_denoised=True, denoised_fn=None, model_kwargs=None, noise_repeat=False):
        """reference models/gaussian_diffusion.py:332-365; the update itself runs in ``rs_p_sample``."""
        out = self.p_mean_variance(model, x, y, t, clip_denoised, denoised_fn, model_kwargs)
        noise = torch.randn_like(x)
        if noise_repeat:
            noise = noise[0,].repeat(x.shape[0], 1, 1, 1)
        i = int(t[0].item())
        if not bool((t == i).all()):
            raise ValueError("p_sample: all batch elements must share the timestep (as in p_sample_loop)")
        xf = x.float().contiguous()
        pred = out["pred_xstart"].float().contiguous()
        nz = noise.float().contiguous()
        sample = torch.empty_like(xf)
        tabs = self.step_tables()
        c1, c2, sd = (float(tabs[k][i]) for k in ("coef1", "coef2", "std"))
        _lib.check(_lib.lib.rs_p_sample(xf.data_ptr(), pred.data_ptr(), nz.data_ptr(), sample.data_ptr(), c1, c2, sd,
                                        int(i == 0), xf.numel(), _lib.current_stream()))
        return {"sample": sample, "pred_xstart": out["pred_xstart"], "mean": out["mean"]}

    # ------------------------------------------------------------------ the loop
    _NATIVE_MEAN_TYPES = {ModelMeanType.START_X: "xstart", ModelMeanType.EPSILON: "epsilon",
                          ModelMeanType.EPSILON_SCALE: "epsilon_scale", ModelMeanType.RESIDUAL: "residual"}

    def _native_ok(self, model, clip_denoised, denoised_fn, model_kwargs) -> bool:
        return (isinstance(model, (UNetModelSwin, UNetModel, UNetModelConv))
                and self.model_mean_type in self._NATIVE_MEAN_TYPES
                and not clip_denoised and denoised_fn is None
                and model_kwargs is not None and "lq" in model_kwargs
                and 2 <= self.num_timesteps <= 64)       # rs_sampler_create_ex: 2 <= T <= FiLM-table rows of a plan

    def sampler_options(self) -> "_lib.SamplerOptionsC":
        """rs_sampler_options of this process: the step's x0 conversion and the denoiser's input scaling."""
        return _lib.SamplerOptionsC(_lib.MEAN_TYPES[self._NATIVE_MEAN_TYPES[self.model_mean_type]],
                                    int(bool(self.normalize_input)), int(bool(self.latent_flag)))

    @staticmethod
    def _check_native_inputs(model: UNetModelSwin, z_y, lq, mask):
        """Same contract as UNetModelSwin.forward (reference models/unet.py:865-882 asserts `mask is not None` iff
        cond_mask; UNetModel.forward takes no mask and its lq is at the latent size or twice it, :569-573): the library
        receives raw pointers, so every shape is checked here."""
        cfg = model.cfg
        B, Cc, H, W = z_y.shape
        plain_lq = isinstance(model, (UNetModel, UNetModelConv))     # x + lq concatenated, no feature extractor or mask
        latent_ch = cfg.out_channels if plain_lq else cfg.in_channels
        if Cc != latent_ch:
            raise ValueError(f"latent has {Cc} channels, the model expects {latent_ch}")
        exp_lq = model.lq_shape(B, H, W)
        if tuple(lq.shape) != exp_lq:
            raise ValueError(f"lq must have shape {exp_lq}, got {tuple(lq.shape)}")
        if plain_lq:
            if mask is not None:
                raise ValueError(f"{type(model).__name__} takes no mask (its forward has no mask parameter)")
        elif cfg.cond_mask:
            if mask is None:
                raise ValueError("this model is mask-conditioned (cond_mask=True): pass model_kwargs['mask']")
            exp_m = (B, 1) + exp_lq[2:]
            if tuple(mask.shape) != exp_m:
                raise ValueError(f"mask must have shape {exp_m}, got {tuple(mask.shape)}")
        elif mask is not None:
            raise ValueError("a mask was given but the model is not mask-conditioned (cond_mask=False)")

    def native_sampler(self, model: UNetModelSwin, batch, height, width):
        plan = model.plan(batch, height, width)
        opt = self.sampler_options()
        key = (self.num_timesteps, self.kappa, tuple(self.sqrt_etas.tolist()), tuple(self.timestep_map),
               (opt.mean_type, opt.normalize_input, opt.latent_flag))
        if key not in plan.samplers:
            h = C.c_void_p()
            se = (C.c_double * self.num_timesteps)(*self.sqrt_etas.tolist())
            tm = (C.c_int32 * self.num_timesteps)(*self.timestep_map)
            _lib.check(_lib.lib.rs_sampler_create_ex(plan.handle, self.num_timesteps, se, float(self.kappa), tm,
                                                     C.byref(opt), C.byref(h)))
            plan.samplers[key] = h
        return plan.samplers[key]

    def draw_noises(self, z_y, noise=None, noise_repeat=False):
        """T+1 noise tensors in the reference's draw order and dtypes (prior: randn_like(z_y),
        models/gaussian_diffusion.py:445-448; then one randn_like(x) (fp32) per step, :358-360)."""
        first = torch.randn_like(z_y) if noise is None else noise
        if noise_repeat:
            first = first[0,].repeat(z_y.shape[0], 1, 1, 1)
        out = torch.empty((self.num_timesteps + 1,) + tuple(z_y.shape), dtype=torch.float32, device=z_y.device)
        out[0] = first.float()
        for k in range(self.num_timesteps):
            n = torch.randn(z_y.shape, dtype=torch.float32, device=z_y.device)
            out[k + 1] = n[0,].repeat(z_y.shape[0], 1, 1, 1) if noise_repeat else n
        return out

    def p_sample_loop_progressive(self, y, model, first_stage_model=None, noise=None, noise_repeat=False,
                                  clip_denoised=True, denoised_fn=None, model_kwargs=None, device=None, progress=False):
        """reference models/gaussian_diffusion.py:421-472 — yields one dict per step (sample, pred_xstart, mean)."""
        z_y = self.encode_first_stage(y, first_stage_model, up_sample=True)
        if self._native_ok(model, clip_denoised, denoised_fn, model_kwargs):
            B, Cc, H, W = z_y.shape
            T = self.num_timesteps
            noises = self.draw_noises(z_y, noise, noise_repeat)
            s = self.native_sampler(model, B, H, W)
            zf = z_y.float().contiguous()
            lq = model_kwargs["lq"].float().contiguous()
            mask = model_kwargs.get("mask", None)
            mask = mask.float().contiguous() if mask is not None else None
            self._check_native_inputs(model, zf, lq, mask)
            final = torch.empty_like(zf)
            preds = torch.empty((T,) + tuple(zf.shape), dtype=torch.float32, device=zf.device)
            samples = torch.empty_like(preds)
            _lib.check(_lib.lib.rs_sampler_set_taps(s, preds.data_ptr(), samples.data_ptr()))
            try:
                _lib.check(_lib.lib.rs_sampler_run(s, zf.data_ptr(), noises.data_ptr(), lq.data_ptr(), _lib.ptr(mask),
                                                   final.data_ptr(), 0, _lib.current_stream()))
            finally:
                _lib.check(_lib.lib.rs_sampler_set_taps(s, None, None))
            # preds holds the step kernel's converted x0 (pred_xstart); the mean follows from it
            c1 = self.posterior_mean_coef1.astype(np.float32)
            c2 = self.posterior_mean_coef2.astype(np.float32)
            x_prev = self.prior_sample(zf, noises[0])
            for k in range(T):
                i = T - 1 - k
                mean = float(c1[i]) * x_prev + float(c2[i]) * preds[k]
                yield {"sample": samples[k], "pred_xstart": preds[k], "mean": mean}
                x_prev = samples[k]
            return
        # generic path: arbitrary model callable, per-step update through rs_p_sample
        if noise is None:
            noise = torch.randn_like(z_y)
        if noise_repeat:
            noise = noise[0,].repeat(z_y.shape[0], 1, 1, 1)
        z_sample = self.prior_sample(z_y, noise)
        for i in list(range(self.num_timesteps))[::-1]:
            t = torch.tensor([i] * y.shape[0], device=z_y.device)
            with torch.no_grad():
                out = self.p_sample(model, z_sample, z_y, t, clip_denoised=clip_denoised, denoised_fn=denoised_fn,
                                    model_kwargs=model_kwargs, noise_repeat=noise_repeat)
            yield out
            z_sample = out["sample"]

    def p_sample_loop(self, y, model, first_stage_model=None, consistencydecoder=None, noise=None, noise_repeat=False,
                      clip_denoised=True, denoised_fn=None, model_kwargs=None, device=None, progress=False):
        """reference models/gaussian_diffusion.py:367-419 — returns the DECODED sample."""
        if self._native_ok(model, clip_denoised, denoised_fn, model_kwargs):
            z_y = self.encode_first_stage(y, first_stage_model, up_sample=True)
            final = self.sample_latent(z_y, model, model_kwargs, noise=noise, noise_repeat=noise_repeat)
        else:
            final = None
            for sample in self.p_sample_loop_progressive(y, model, first_stage_model=first_stage_model, noise=noise,
                                                         noise_repeat=noise_repeat, clip_denoised=clip_denoised,
                                                         denoised_fn=denoised_fn, model_kwargs=model_kwargs,
                                                         device=device, progress=progress):
                final = sample["sample"]
        with torch.no_grad():
            return self.decode_first_stage(final, first_stage_model=first_stage_model, consistencydecoder=consistencydecoder)

    def sample_latent(self, z_y, model: UNetModelSwin, model_kwargs, noise=None, noise_repeat=False, noises=None,
                      use_graph=True):
        """The hot path proper: z_y -> final latent, all T steps inside librs_b200 (CUDA graph replay)."""
        B, Cc, H, W = z_y.shape
        if noises is None:
            noises = self.draw_noises(z_y, noise, noise_repeat)
        s = self.native_sampler(model, B, H, W)
        # stable device buffers so that the captured graph can be replayed call after call
        plan = model.plan(B, H, W)
        bufs = getattr(plan, "_io", None)
        lq_in = model_kwargs["lq"]
        mask_in = model_kwargs.get("mask", None)
        self._check_native_inputs(model, z_y, lq_in, mask_in)
        if tuple(noises.shape) != (self.num_timesteps + 1,) + tuple(z_y.shape):
            raise ValueError(f"noises must have shape {(self.num_timesteps + 1,) + tuple(z_y.shape)}, got {tuple(noises.shape)}")
        if (bufs is None or bufs["lq"].shape != lq_in.shape or (mask_in is None) != (bufs["mask"] is None)
                or bufs["noise"].shape != noises.shape):
            bufs = {"zy": torch.empty(B, Cc, H, W, dtype=torch.float32, device=z_y.device),
                    "noise": torch.empty_like(noises),
                    "lq": torch.empty(lq_in.shape, dtype=torch.float32, device=z_y.device),
                    "mask": None if mask_in is None else torch.empty(mask_in.shape, dtype=torch.float32, device=z_y.device),
                    "out": torch.empty(B, Cc, H, W, dtype=torch.float32, device=z_y.device)}
            plan._io = bufs
        bufs["zy"].copy_(z_y)
        bufs["noise"].copy_(noises)
        bufs["lq"].copy_(lq_in)
        if mask_in is not None:
            bufs["mask"].copy_(mask_in)
        _lib.check(_lib.lib.rs_sampler_run(s, bufs["zy"].data_ptr(), bufs["noise"].data_ptr(), bufs["lq"].data_ptr(),
                                           _lib.ptr(bufs["mask"]), bufs["out"].data_ptr(), int(use_graph),
                                           _lib.current_stream()))
        return bufs["out"].clone()

    def training_losses(self, *a, **k):
        raise NotImplementedError("training is outside the covered hot path (inference only)")
