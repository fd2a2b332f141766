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

``SpacedDiffusionDDPM`` is the reference's other process, the classic DDPM / DDIM one (``GaussianDiffusionDDPM``,
reference models/gaussian_diffusion.py:611-1239, models/respace.py:65-99), with its ancestral ``p_sample_loop`` and
``ddim_sample_loop``, and DDIM inversion (``ddim_reverse_sample``, reference :1030-1066, walked t = 0 .. T-1 by this
package's ``ddim_reverse_sample_loop``).  With one of this package's UNets, eps or x0 prediction, a fixed variance, no
``denoised_fn``, an ``lq`` in ``model_kwargs`` and 2 <= T <= 64, the whole loop (denoiser, x0 conversion, clamp,
ancestral, DDIM or reverse update, next-input packing) runs inside ``librs_b200.so`` as one CUDA graph; everything else
runs this module's torch port of the reference on the caller's device.
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


class ModelVarTypeDDPM(enum.Enum):
    """What the DDPM process uses as the model's output variance (reference models/gaussian_diffusion.py:82-90)."""
    LEARNED = enum.auto()
    LEARNED_RANGE = enum.auto()
    FIXED_LARGE = enum.auto()
    FIXED_SMALL = enum.auto()


def get_named_beta_schedule(schedule_name, num_diffusion_timesteps, beta_start, beta_end):
    """Betas of the DDPM process, float64 (reference models/gaussian_diffusion.py:14-30): "linear" only."""
    if schedule_name == "linear":
        return np.linspace(beta_start ** 0.5, beta_end ** 0.5, num_diffusion_timesteps, dtype=np.float64) ** 2
    raise NotImplementedError(f"unknown beta schedule: {schedule_name}")


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


def _cached_sampler(plan, key, create):
    """The plan's native sampler for `key` (a process and its options), made on first use by create(out_handle)."""
    if key not in plan.samplers:
        h = C.c_void_p()
        _lib.check(create(C.byref(h)))
        plan.samplers[key] = h
    return plan.samplers[key]


def _native_inputs(model, x, model_kwargs):
    """lq and mask of model_kwargs as contiguous fp32, checked against the model for the latent x."""
    lq = model_kwargs["lq"].float().contiguous()
    mask = model_kwargs.get("mask", None)
    mask = mask.float().contiguous() if mask is not None else None
    ResShiftDiffusion._check_native_inputs(model, x, lq, mask)
    return lq, mask


def _run_tapped(s, T, x, lq, mask, z_y=None, noises=None):
    """Sampler s run eagerly with the per-step taps on inputs shaped like the latent x: returns (final, preds,
    samples), preds / samples [T, *x.shape] holding every step's pred_xstart / sample."""
    final = torch.empty_like(x)
    preds = torch.empty((T,) + tuple(x.shape), dtype=torch.float32, device=x.device)
    samples = torch.empty_like(preds)
    _lib.check(_lib.lib.rs_sampler_set_taps(s, preds.data_ptr(), samples.data_ptr()))
    try:
        _lib.check(_lib.lib.rs_sampler_run(s, _lib.ptr(z_y), _lib.ptr(noises), lq.data_ptr(), _lib.ptr(mask),
                                           final.data_ptr(), 0, _lib.current_stream()))
    finally:
        _lib.check(_lib.lib.rs_sampler_set_taps(s, None, None))
    return final, preds, samples


def _run_graphed(model, s, shape, model_kwargs, z_y=None, noises=None, use_graph=True):
    """Sampler s run on the plan's stable device buffers (plan._io), so that its captured CUDA graph replays call after
    call: z_y and noises (whichever the process reads), lq and mask are copied in, and the final latent of `shape`
    comes back as a new tensor.  Every sampler of the plan shares the buffers; each is made again when its shape
    changes."""
    B, _, H, W = shape
    plan = model.plan(B, H, W)
    dev = (z_y if z_y is not None else noises).device
    io = getattr(plan, "_io", None)
    if io is None:
        io = plan._io = {}

    def buf(name, shp):
        if name not in io or tuple(io[name].shape) != tuple(shp):
            io[name] = torch.empty(tuple(shp), dtype=torch.float32, device=dev)
        return io[name]

    def stage(name, src):
        return None if src is None else buf(name, src.shape).copy_(src)

    zy, nz, lq, mask = (stage(k, v) for k, v in (("zy", z_y), ("noise", noises), ("lq", model_kwargs["lq"]),
                                                  ("mask", model_kwargs.get("mask", None))))
    out = buf("out", shape)
    _lib.check(_lib.lib.rs_sampler_run(s, _lib.ptr(zy), _lib.ptr(nz), lq.data_ptr(), _lib.ptr(mask), out.data_ptr(),
                                       int(use_graph), _lib.current_stream()))
    return out.clone()


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
        latent_ch = model.x_channels
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
        T = self.num_timesteps
        return _cached_sampler(plan, key, lambda out: _lib.lib.rs_sampler_create_ex(
            plan.handle, T, (C.c_double * T)(*self.sqrt_etas.tolist()), float(self.kappa),
            (C.c_int32 * T)(*self.timestep_map), C.byref(opt), out))

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
            lq, mask = _native_inputs(model, zf, model_kwargs)
            _, preds, samples = _run_tapped(s, T, zf, lq, mask, z_y=zf, noises=noises)
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
        self._check_native_inputs(model, z_y, model_kwargs["lq"], model_kwargs.get("mask", None))
        if tuple(noises.shape) != (self.num_timesteps + 1,) + tuple(z_y.shape):
            raise ValueError(f"noises must have shape {(self.num_timesteps + 1,) + tuple(z_y.shape)}, got {tuple(noises.shape)}")
        return _run_graphed(model, s, z_y.shape, model_kwargs, z_y=z_y, noises=noises, use_graph=use_graph)

    def training_losses(self, *a, **k):
        raise NotImplementedError("training is outside the covered hot path (inference only)")


class SpacedDiffusionDDPM:
    """``SpacedDiffusionDDPM(GaussianDiffusionDDPM)`` of the reference (models/respace.py:65-99,
    models/gaussian_diffusion.py:611-1239), inference side: the respaced schedule, ``p_mean_variance`` for every
    variance and mean type, the ancestral and DDIM steps and loops, DDIM inversion (``ddim_reverse_sample`` and this
    package's loop around it), and the first-stage bookends."""

    def __init__(self, use_timesteps, *, betas, model_mean_type, model_var_type, scale_factor=None, sf=4):
        # respacing (reference models/respace.py:74-88): the kept steps' betas from the base process's alphas_cumprod
        self.use_timesteps = set(use_timesteps)
        base = np.array(betas, dtype=np.float64)
        self.original_num_steps = len(base)
        self.timestep_map = []
        new_betas, last = [], 1.0
        for i, acp in enumerate(np.cumprod(1.0 - base, axis=0)):
            if i in self.use_timesteps:
                new_betas.append(1 - acp / last)
                last = acp
                self.timestep_map.append(i)
        self.model_mean_type, self.model_var_type = model_mean_type, model_var_type
        self.scale_factor, self.sf = scale_factor, sf
        # float64 tables (reference models/gaussian_diffusion.py:642-680)
        betas = np.array(new_betas, dtype=np.float64)
        self.betas = betas
        assert len(betas.shape) == 1, "betas must be 1-D"
        assert (betas > 0).all() and (betas <= 1).all()
        self.num_timesteps = int(betas.shape[0])
        alphas = 1.0 - betas
        self.alphas_cumprod = np.cumprod(alphas, axis=0)
        self.alphas_cumprod_prev = np.append(1.0, self.alphas_cumprod[:-1])
        self.alphas_cumprod_next = np.append(self.alphas_cumprod[1:], 0.0)
        self.sqrt_alphas_cumprod = np.sqrt(self.alphas_cumprod)
        self.sqrt_one_minus_alphas_cumprod = np.sqrt(1.0 - self.alphas_cumprod)
        self.log_one_minus_alphas_cumprod = np.log(1.0 - self.alphas_cumprod)
        self.sqrt_recip_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod)
        self.sqrt_recipm1_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod - 1)
        self.posterior_variance = betas * (1.0 - self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_log_variance_clipped = np.log(np.append(self.posterior_variance[1], self.posterior_variance[1:]))
        self.posterior_mean_coef1 = betas * np.sqrt(self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_mean_coef2 = (1.0 - self.alphas_cumprod_prev) * np.sqrt(alphas) / (1.0 - self.alphas_cumprod)
        # FIXED_LARGE's variance (p_mean_variance :791-794)
        self.variance_fixed_large = np.append(self.posterior_variance[1], self.betas[1:])
        self.log_variance_fixed_large = np.log(self.variance_fixed_large)
        # LEARNED_RANGE's max_log (p_mean_variance :781)
        self.log_betas = np.log(self.betas)

    # ------------------------------------------------------------------ small pieces (torch)
    def _scale_input(self, inputs, t):
        """reference models/gaussian_diffusion.py:1213-1214"""
        return inputs

    def _model_t(self, t):
        """_WrappedModel's timestep map (reference models/respace.py:60-63)"""
        return torch.tensor(self.timestep_map, device=t.device, dtype=t.dtype)[t]

    def q_mean_variance(self, x_start, t):
        """reference models/gaussian_diffusion.py:681-696"""
        return (_tab(self.sqrt_alphas_cumprod, t, x_start) * x_start, _tab(1.0 - self.alphas_cumprod, t, x_start),
                _tab(self.log_one_minus_alphas_cumprod, t, x_start))

    def q_sample(self, x_start, t, noise=None):
        """reference models/gaussian_diffusion.py:698-716"""
        if noise is None:
            noise = torch.randn_like(x_start)
        assert noise.shape == x_start.shape
        return (_tab(self.sqrt_alphas_cumprod, t, x_start) * x_start
                + _tab(self.sqrt_one_minus_alphas_cumprod, t, x_start) * noise)

    def q_posterior_mean_variance(self, x_start, x_t, t):
        """reference models/gaussian_diffusion.py:718-740"""
        assert x_start.shape == x_t.shape
        mean = _tab(self.posterior_mean_coef1, t, x_t) * x_start + _tab(self.posterior_mean_coef2, t, x_t) * x_t
        return mean, _tab(self.posterior_variance, t, x_t), _tab(self.posterior_log_variance_clipped, t, x_t)

    def _predict_xstart_from_eps(self, x_t, t, eps):
        """reference models/gaussian_diffusion.py:838-843"""
        assert x_t.shape == eps.shape
        return _tab(self.sqrt_recip_alphas_cumprod, t, x_t) * x_t - _tab(self.sqrt_recipm1_alphas_cumprod, t, x_t) * eps

    def _predict_xstart_from_xprev(self, x_t, t, xprev):
        """reference models/gaussian_diffusion.py:845-853"""
        assert x_t.shape == xprev.shape
        return (_tab(1.0 / self.posterior_mean_coef1, t, x_t) * xprev
                - _tab(self.posterior_mean_coef2 / self.posterior_mean_coef1, t, x_t) * x_t)

    def _predict_eps_from_xstart(self, x_t, t, pred_xstart):
        """reference models/gaussian_diffusion.py:855-859"""
        return (_tab(self.sqrt_recip_alphas_cumprod, t, x_t) * x_t - pred_xstart) / _tab(self.sqrt_recipm1_alphas_cumprod, t, x_t)

    def p_mean_variance(self, model, x, t, clip_denoised=True, denoised_fn=None, model_kwargs=None):
        """reference models/gaussian_diffusion.py:742-836, the model's timesteps mapped as models/respace.py:90-91 does."""
        if model_kwargs is None:
            model_kwargs = {}
        B, Cc = x.shape[:2]
        assert t.shape == (B,)
        model_output = model(x, self._model_t(t), **model_kwargs)
        if self.model_var_type in (ModelVarTypeDDPM.LEARNED, ModelVarTypeDDPM.LEARNED_RANGE):
            assert model_output.shape == (B, Cc * 2, *x.shape[2:])
            model_output, model_var_values = torch.split(model_output, Cc, dim=1)
            if self.model_var_type == ModelVarTypeDDPM.LEARNED:
                model_log_variance = model_var_values
                model_variance = torch.exp(model_log_variance)
            else:
                min_log = _tab(self.posterior_log_variance_clipped, t, x)
                max_log = _tab(self.log_betas, t, x)
                frac = (model_var_values + 1) / 2               # [-1, 1] -> [min_var, max_var]
                model_log_variance = frac * max_log + (1 - frac) * min_log
                model_variance = torch.exp(model_log_variance)
        else:
            var, log_var = {
                ModelVarTypeDDPM.FIXED_LARGE: (self.variance_fixed_large, self.log_variance_fixed_large),
                ModelVarTypeDDPM.FIXED_SMALL: (self.posterior_variance, self.posterior_log_variance_clipped),
            }[self.model_var_type]
            model_variance, model_log_variance = _tab(var, t, x), _tab(log_var, t, x)

        def process_xstart(v):
            if denoised_fn is not None:
                v = denoised_fn(v)
            return v.clamp(-1, 1) if clip_denoised else v

        if self.model_mean_type == ModelMeanType.PREVIOUS_X:
            pred_xstart = process_xstart(self._predict_xstart_from_xprev(x_t=x, t=t, xprev=model_output))
            model_mean = model_output
        elif self.model_mean_type in (ModelMeanType.START_X, ModelMeanType.EPSILON):
            if self.model_mean_type == ModelMeanType.START_X:
                pred_xstart = process_xstart(model_output)
            else:
                pred_xstart = process_xstart(self._predict_xstart_from_eps(x_t=x, t=t, eps=model_output))
            model_mean, _, _ = self.q_posterior_mean_variance(x_start=pred_xstart, x_t=x, t=t)
        else:
            raise NotImplementedError(self.model_mean_type)
        assert model_mean.shape == model_log_variance.shape == pred_xstart.shape == x.shape
        return {"mean": model_mean, "variance": model_variance, "log_variance": model_log_variance,
                "pred_xstart": pred_xstart}

    # ------------------------------------------------------------------ one step (torch, any model callable)
    def _p_finish(self, x, t, out, noise):
        """the rest of reference p_sample (models/gaussian_diffusion.py:887-892) on p_mean_variance's output"""
        nonzero_mask = (t != 0).float().view(-1, *([1] * (len(x.shape) - 1)))      # no noise when t == 0
        sample = out["mean"] + nonzero_mask * torch.exp(0.5 * out["log_variance"]) * noise
        return {"sample": sample, "pred_xstart": out["pred_xstart"]}

    def _ddim_finish(self, x, t, out, noise, eta):
        """the rest of reference ddim_sample (models/gaussian_diffusion.py:1010-1028) on p_mean_variance's output"""
        eps = self._predict_eps_from_xstart(x, t, out["pred_xstart"])
        alpha_bar = _tab(self.alphas_cumprod, t, x)
        alpha_bar_prev = _tab(self.alphas_cumprod_prev, t, x)
        sigma = eta * torch.sqrt((1 - alpha_bar_prev) / (1 - alpha_bar)) * torch.sqrt(1 - alpha_bar / alpha_bar_prev)
        mean_pred = out["pred_xstart"] * torch.sqrt(alpha_bar_prev) + torch.sqrt(1 - alpha_bar_prev - sigma ** 2) * eps
        nonzero_mask = (t != 0).float().view(-1, *([1] * (len(x.shape) - 1)))      # no noise when t == 0
        return {"sample": mean_pred + nonzero_mask * sigma * noise, "pred_xstart": out["pred_xstart"]}

    def p_sample(self, model, x, t, clip_denoised=True, denoised_fn=None, model_kwargs=None):
        """reference models/gaussian_diffusion.py:861-892"""
        out = self.p_mean_variance(model, x, t, clip_denoised=clip_denoised, denoised_fn=denoised_fn,
                                   model_kwargs=model_kwargs)
        return self._p_finish(x, t, out, torch.randn_like(x))

    def ddim_sample(self, model, x, t, clip_denoised=True, denoised_fn=None, model_kwargs=None, eta=0.0):
        """reference models/gaussian_diffusion.py:985-1028"""
        out = self.p_mean_variance(model, x, t, clip_denoised=clip_denoised, denoised_fn=denoised_fn,
                                   model_kwargs=model_kwargs)
        return self._ddim_finish(x, t, out, torch.randn_like(x), eta)

    def _ddim_reverse_finish(self, x, t, out):
        """the rest of reference ddim_reverse_sample (models/gaussian_diffusion.py:1052-1066) on p_mean_variance's
        output: eps re-derived from pred_xstart, then x_{t+1} = x0 sqrt(acp_next) + sqrt(1 - acp_next) eps"""
        eps = self._predict_eps_from_xstart(x, t, out["pred_xstart"])
        alpha_bar_next = _tab(self.alphas_cumprod_next, t, x)
        mean_pred = out["pred_xstart"] * torch.sqrt(alpha_bar_next) + torch.sqrt(1 - alpha_bar_next) * eps
        return {"sample": mean_pred, "pred_xstart": out["pred_xstart"]}

    def ddim_reverse_sample(self, model, x, t, clip_denoised=True, denoised_fn=None, model_kwargs=None, eta=0.0):
        """reference models/gaussian_diffusion.py:1030-1066 — x_{t+1} from x_t by the deterministic DDIM ODE."""
        assert eta == 0.0, "Reverse ODE only for deterministic path"
        out = self.p_mean_variance(model, x, t, clip_denoised=clip_denoised, denoised_fn=denoised_fn,
                                   model_kwargs=model_kwargs)
        return self._ddim_reverse_finish(x, t, out)

    # ------------------------------------------------------------------ the loops
    def draw_noises(self, shape, noise=None, device=None):
        """The T + 1 noise tensors of a loop in the reference's draw order: x_T = ``noise`` or randn(*shape)
        (models/gaussian_diffusion.py:959-962, :1122-1125), then one randn_like(x) per step (:887, :1019; DDIM draws
        one at eta = 0 too).  Drawn ahead, so that the fused and the torch route see the same values under one seed."""
        first = torch.randn(*shape, device=device) if noise is None else noise
        out = torch.empty((self.num_timesteps + 1,) + tuple(first.shape), dtype=first.dtype, device=first.device)
        out[0] = first
        for k in range(self.num_timesteps):
            out[k + 1] = torch.randn_like(first)
        return out

    _NATIVE_MEAN_TYPES = {ModelMeanType.EPSILON: 1, ModelMeanType.START_X: 0}        # rs_mean_type
    _NATIVE_VAR_TYPES = {ModelVarTypeDDPM.FIXED_LARGE: 0, ModelVarTypeDDPM.FIXED_SMALL: 1,   # rs_ddpm_var_type
                         ModelVarTypeDDPM.LEARNED_RANGE: 3, ModelVarTypeDDPM.LEARNED: 4}
    _LEARNED = (ModelVarTypeDDPM.LEARNED, ModelVarTypeDDPM.LEARNED_RANGE)

    def _native_ok(self, model, denoised_fn, model_kwargs) -> bool:
        """Whether the fused loop runs this call.  A learned variance needs a model whose output has twice the latent's
        channels (mean, then variance values), a fixed one the same count; any other model goes to the torch route,
        where the reference's own shape assertion speaks."""
        if not (isinstance(model, (UNetModelSwin, UNetModel, UNetModelConv))
                and self.model_mean_type in self._NATIVE_MEAN_TYPES
                and self.model_var_type in self._NATIVE_VAR_TYPES
                and denoised_fn is None
                and model_kwargs is not None and "lq" in model_kwargs
                and 2 <= self.num_timesteps <= 64):      # rs_ddpm_sampler_create: 2 <= T <= FiLM-table rows of a plan
            return False
        return model.cfg.out_channels == model.x_channels * (2 if self.model_var_type in self._LEARNED else 1)

    def ddpm_tables(self) -> np.ndarray:
        """[8, T] float64: the rows of rs_ddpm_sampler_create (rs_ddpm_table_row)"""
        return np.ascontiguousarray(np.stack([getattr(self, name) for name in _lib.DDPM_TABLE_ROWS]), dtype=np.float64)

    def ddpm_learned_range_tables(self) -> np.ndarray:
        """[9, T] float64: the rows of rs_ddpm_sampler_create with RS_VAR_LEARNED_RANGE (ddpm_tables, then log(betas))"""
        return np.ascontiguousarray(np.stack([getattr(self, name) for name in _lib.DDPM_LEARNED_RANGE_TABLE_ROWS]),
                                    dtype=np.float64)

    def ddim_reverse_tables(self) -> np.ndarray:
        """[9, T] float64: the rows of rs_ddim_reverse_sampler_create (ddpm_tables, then alphas_cumprod_next)"""
        return np.ascontiguousarray(np.stack([getattr(self, name) for name in _lib.DDIM_REVERSE_TABLE_ROWS]),
                                    dtype=np.float64)

    def native_sampler(self, model, batch, height, width, kind: str, clip_denoised: bool, eta: float = 0.0):
        """The plan's DDPM sampler for this process and these options ("ancestral", "ddim", or "reverse" for DDIM
        inversion, which has no eta), created once."""
        plan = model.plan(batch, height, width)
        T = self.num_timesteps
        process = (T, tuple(self.betas.tolist()), tuple(self.timestep_map))
        if kind == "reverse":
            ropt = _lib.DdimReverseOptionsC(self._NATIVE_MEAN_TYPES[self.model_mean_type], int(bool(clip_denoised)))
            tabs = self.ddim_reverse_tables()
            return _cached_sampler(plan, ("ddim_reverse",) + process + ((ropt.mean_type, ropt.clip),),
                                   lambda out: _lib.lib.rs_ddim_reverse_sampler_create(
                                       plan.handle, T, tabs.ctypes.data_as(C.POINTER(C.c_double)),
                                       (C.c_int32 * T)(*self.timestep_map), C.byref(ropt), out))
        opt = _lib.DdpmOptionsC(_lib.DDPM_KINDS[kind], self._NATIVE_MEAN_TYPES[self.model_mean_type],
                                self._NATIVE_VAR_TYPES[self.model_var_type], int(bool(clip_denoised)), float(eta))
        tabs = (self.ddpm_learned_range_tables() if self.model_var_type == ModelVarTypeDDPM.LEARNED_RANGE
                else self.ddpm_tables())
        return _cached_sampler(plan, ("ddpm",) + process + ((opt.kind, opt.mean_type, opt.var_type, opt.clip, opt.eta),),
                               lambda out: _lib.lib.rs_ddpm_sampler_create(
                                   plan.handle, T, tabs.ctypes.data_as(C.POINTER(C.c_double)),
                                   (C.c_int32 * T)(*self.timestep_map), C.byref(opt), out))

    def sample_latent(self, model, noises, model_kwargs, kind="ancestral", clip_denoised=True, eta=0.0, use_graph=True):
        """The fused loop: noises [T + 1, B, C, H, W] (draw_noises) -> the final latent, all T steps inside librs_b200
        (CUDA graph replay)."""
        T = self.num_timesteps
        if noises.dim() != 5 or noises.shape[0] != T + 1:
            raise ValueError(f"noises must have shape (T + 1 = {T + 1}, B, C, H, W), got {tuple(noises.shape)}")
        B, Cc, H, W = noises.shape[1:]
        lq_in, mask_in = model_kwargs["lq"], model_kwargs.get("mask", None)
        ResShiftDiffusion._check_native_inputs(model, noises[0], lq_in, mask_in)
        s = self.native_sampler(model, B, H, W, kind, clip_denoised, eta)
        return _run_graphed(model, s, noises.shape[1:], model_kwargs, noises=noises, use_graph=use_graph)

    def _native_progressive(self, model, noises, model_kwargs, kind, clip_denoised, eta):
        """The fused loop run eagerly with the per-step taps: yields sample / pred_xstart of every step."""
        T = self.num_timesteps
        x = noises[0].float().contiguous()
        B, Cc, H, W = x.shape
        lq, mask = _native_inputs(model, x, model_kwargs)
        s = self.native_sampler(model, B, H, W, kind, clip_denoised, eta)
        _, preds, samples = _run_tapped(s, T, x, lq, mask, noises=noises.float().contiguous())
        for k in range(T):
            yield {"sample": samples[k], "pred_xstart": preds[k]}

    def reverse_latent(self, model, x_start, model_kwargs, clip_denoised=True, use_graph=True):
        """The fused DDIM inversion: x_start [B, C, H, W] -> x_T, all T steps inside librs_b200 (CUDA graph replay)."""
        if x_start.dim() != 4:
            raise ValueError(f"x_start must have shape (B, C, H, W), got {tuple(x_start.shape)}")
        B, Cc, H, W = x_start.shape
        lq_in, mask_in = model_kwargs["lq"], model_kwargs.get("mask", None)
        ResShiftDiffusion._check_native_inputs(model, x_start, lq_in, mask_in)
        s = self.native_sampler(model, B, H, W, "reverse", clip_denoised)
        return _run_graphed(model, s, x_start.shape, model_kwargs, z_y=x_start, use_graph=use_graph)

    def _native_reverse_progressive(self, model, x_start, model_kwargs, clip_denoised):
        """The fused DDIM inversion run eagerly with the per-step taps: yields sample / pred_xstart of every step."""
        T = self.num_timesteps
        x = x_start.float().contiguous()
        B, Cc, H, W = x.shape
        lq, mask = _native_inputs(model, x, model_kwargs)
        s = self.native_sampler(model, B, H, W, "reverse", clip_denoised)
        _, preds, samples = _run_tapped(s, T, x, lq, mask, z_y=x)
        for k in range(T):
            yield {"sample": samples[k], "pred_xstart": preds[k]}

    def _progressive(self, kind, model, shape, noise, clip_denoised, denoised_fn, model_kwargs, device, progress, eta):
        if device is None:
            device = next(model.parameters()).device
        assert isinstance(shape, (tuple, list))
        noises = self.draw_noises(shape, noise, device)
        if self._native_ok(model, denoised_fn, model_kwargs):
            yield from self._native_progressive(model, noises, model_kwargs, kind, clip_denoised, eta)
            return
        img = noises[0]
        indices = list(range(self.num_timesteps))[::-1]
        if progress:
            from tqdm.auto import tqdm      # lazy, as the reference does
            indices = tqdm(indices)
        for k, i in enumerate(indices):
            t = torch.tensor([i] * shape[0], device=device)
            if kind == "ddim":
                t = t.long()
            with torch.no_grad():
                out = self.p_mean_variance(model, img, t, clip_denoised=clip_denoised, denoised_fn=denoised_fn,
                                           model_kwargs=model_kwargs)
                if kind == "ddim":
                    out = self._ddim_finish(img, t, out, noises[k + 1], eta)
                else:
                    out = self._p_finish(img, t, out, noises[k + 1])
                yield out
                img = out["sample"]

    def p_sample_loop_progressive(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None,
                                  model_kwargs=None, device=None, progress=False):
        """reference models/gaussian_diffusion.py:937-983 — one dict (sample, pred_xstart) per step."""
        yield from self._progressive("ancestral", model, shape, noise, clip_denoised, denoised_fn, model_kwargs, device,
                                     progress, 0.0)

    def ddim_sample_loop_progressive(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None,
                                     model_kwargs=None, device=None, progress=False, eta=0.0):
        """reference models/gaussian_diffusion.py:1101-1147 — one dict (sample, pred_xstart) per step."""
        yield from self._progressive("ddim", model, shape, noise, clip_denoised, denoised_fn, model_kwargs, device,
                                     progress, eta)

    def _loop(self, kind, model, shape, noise, clip_denoised, denoised_fn, first_stage_model, model_kwargs, device,
              progress, eta):
        if self._native_ok(model, denoised_fn, model_kwargs):
            if device is None:
                device = next(model.parameters()).device
            assert isinstance(shape, (tuple, list))
            noises = self.draw_noises(shape, noise, device)
            final = self.sample_latent(model, noises, model_kwargs, kind, clip_denoised, eta)
        else:
            final = None
            for sample in self._progressive(kind, model, shape, noise, clip_denoised, denoised_fn, model_kwargs, device,
                                            progress, eta):
                final = sample["sample"]
        return self.decode_first_stage(final, first_stage_model)

    def p_sample_loop(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, first_stage_model=None,
                      model_kwargs=None, device=None, progress=False):
        """reference models/gaussian_diffusion.py:894-935 — returns the DECODED sample."""
        return self._loop("ancestral", model, shape, noise, clip_denoised, denoised_fn, first_stage_model, model_kwargs,
                          device, progress, 0.0)

    def ddim_sample_loop(self, model, shape, noise=None, first_stage_model=None, clip_denoised=True, denoised_fn=None,
                         model_kwargs=None, device=None, progress=False, eta=0.0):
        """reference models/gaussian_diffusion.py:1068-1099 — returns the DECODED sample."""
        return self._loop("ddim", model, shape, noise, clip_denoised, denoised_fn, first_stage_model, model_kwargs,
                          device, progress, eta)

    def ddim_reverse_sample_loop_progressive(self, model, x_start, clip_denoised=True, denoised_fn=None,
                                             model_kwargs=None, device=None, progress=False):
        """DDIM inversion, x_0 -> x_T: ``ddim_reverse_sample`` (reference models/gaussian_diffusion.py:1030-1066) for
        t = 0 .. T-1, each step fed the previous step's sample; one dict (sample, pred_xstart) per step.  The reference
        has the step only; this loop is this package's addition.  ``x_start`` is a latent (encode an image with
        ``encode_first_stage`` first); ``device`` defaults to x_start's."""
        img = x_start if device is None else x_start.to(device)
        if self._native_ok(model, denoised_fn, model_kwargs):
            yield from self._native_reverse_progressive(model, img, model_kwargs, clip_denoised)
            return
        indices = list(range(self.num_timesteps))
        if progress:
            from tqdm.auto import tqdm      # lazy, as the reference's loops do
            indices = tqdm(indices)
        for i in indices:
            t = torch.tensor([i] * img.shape[0], device=img.device)
            with torch.no_grad():
                out = self.ddim_reverse_sample(model, img, t, clip_denoised=clip_denoised, denoised_fn=denoised_fn,
                                               model_kwargs=model_kwargs)
                yield out
                img = out["sample"]

    def ddim_reverse_sample_loop(self, model, x_start, clip_denoised=True, denoised_fn=None, model_kwargs=None,
                                 device=None, progress=False):
        """DDIM inversion, x_0 -> x_T (this package's loop around the reference's ``ddim_reverse_sample``, see
        ``ddim_reverse_sample_loop_progressive``): returns the last step's sample, the latent x_T (not decoded)."""
        if self._native_ok(model, denoised_fn, model_kwargs):
            return self.reverse_latent(model, x_start if device is None else x_start.to(device), model_kwargs,
                                       clip_denoised)
        final = None
        for sample in self.ddim_reverse_sample_loop_progressive(model, x_start, clip_denoised, denoised_fn,
                                                                model_kwargs, device, progress):
            final = sample["sample"]
        return final

    # ------------------------------------------------------------------ first-stage bookends (PyTorch)
    def decode_first_stage(self, z_sample, first_stage_model=None):
        """reference models/gaussian_diffusion.py:1216-1225"""
        ori_dtype = z_sample.dtype
        if first_stage_model is None:
            return z_sample
        with torch.no_grad():
            z_sample = 1 / self.scale_factor * z_sample
            z_sample = z_sample.type(next(first_stage_model.parameters()).dtype)
            return first_stage_model.decode(z_sample).type(ori_dtype)

    def encode_first_stage(self, y, first_stage_model, up_sample=False):
        """reference models/gaussian_diffusion.py:1227-1239"""
        ori_dtype = y.dtype
        if up_sample:
            y = bicubic_upsample(y, self.sf)
        if first_stage_model is None:
            return y
        with torch.no_grad():
            y = y.type(dtype=next(first_stage_model.parameters()).dtype)
            return (first_stage_model.encode(y) * self.scale_factor).type(ori_dtype)

    def training_losses(self, *a, **k):
        raise NotImplementedError("training is outside the covered hot path (inference only)")
