"""Learned-variance DDPM models (learn_sigma: LEARNED / LEARNED_RANGE, a 2 C output head) in the fused loop, on the
H100.

  * The step kernel (rs_op_ddpm_step with the output's image stride and var_type): the ancestral step takes its log
    variance from the variance half, element by element bit-identical to the port's torch fp32 expression on the
    device (p_mean_variance :772-786 and p_sample), for eps and x0, both learned types, clip on and off, t = T - 1, a
    middle step and 0.  The variance values span [-1.5, 1.5], so frac leaves [0, 1] as the reference allows.  DDIM and
    inversion read the mean half only: bit-identical to the torch expression, and unchanged when the variance half
    changes.
  * Each family's fused loop (UNetModel, UNetModelSwin, UNetModelConv with out_channels = 6) on the fixtures of
    oracle/make_golden_ddpm_learned.py: bit-identical to the torch route driving the same native UNet step by step,
    and within test_gpu_ddpm's loop bounds of the reference's trajectories, widened by what the variance half's error
    carries into the ancestral sample.
  * Graph replay == eager == replay with a learned ancestral and a learned DDIM sampler alternating on one plan, and
    the C ABI's refusals.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import tests.gpu_util as G
from oracle.make_golden_ddpm_learned import CASES, OUT_STRIDE, case_inputs, diffusion_kwargs, model_config
from resshift_b200 import _lib
from resshift_b200.models import gaussian_diffusion as gd
from resshift_b200.models.script_util import create_gaussian_diffusion, create_gaussian_diffusion_ddpm
from resshift_b200.models.unet import UNetModel, UNetModelConv, UNetModelSwin
from resshift_b200.weights import random_state_dict
from tests.sampler_ref import bound, cached_model, compare, dev32, ulps

pytestmark = pytest.mark.gpu

KW8 = dict(beta_start=0.0015, beta_end=0.0155, steps=1000, timestep_respacing=8)
V = gd.ModelVarTypeDDPM
VAR_TYPES = {V.LEARNED: _lib.DDPM_VAR_TYPES["learned"], V.LEARNED_RANGE: _lib.DDPM_VAR_TYPES["learned_range"]}


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(golden_dir / "ddpm_learned.npz")


_MODELS = {}


def learned_model(case):
    """a case's model (its family's fixture model with out_channels = 6), random weights, on the device"""
    if case not in _MODELS:
        ucfg, hw = model_config(case)
        cls = {"unetmodel": UNetModel, "unetconv": UNetModelConv, "swin": UNetModelSwin}[CASES[case][0]]
        m = cls(**ucfg.to_kwargs())
        m.load_state_dict(random_state_dict(ucfg, 0), strict=True)
        _MODELS[case] = (m.cuda().eval(), hw)
    return _MODELS[case]


def _diff(var, **kw):
    diff = create_gaussian_diffusion_ddpm(learn_sigma=True, **KW8, **kw)
    diff.model_var_type = var                   # the factory builds LEARNED_RANGE; LEARNED is the process's other type
    return diff


def _step_args(diff, kind, mean_eps, clip, eta, t, x, out, noise, x_next, x0_out, next_in=None, counters=None,
               n_counters=0):
    names = ("sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_mean_coef1", "posterior_mean_coef2",
             "posterior_log_variance_clipped", "alphas_cumprod", "alphas_cumprod_prev", "log_betas")
    tabs = [dev32(getattr(diff, n)) for n in names]
    N, Cc, H, W = x.shape
    a = _lib.DdpmStepArgsC(out.data_ptr(), x.data_ptr(), noise.data_ptr(), x_next.data_ptr(),
                           *(tb.data_ptr() for tb in tabs[:7]), diff.num_timesteps, t, N, Cc, H * W,
                           _lib.DDPM_KINDS[kind], 1 if mean_eps else 0, int(clip), float(eta),
                           _lib.ptr(next_in), 0 if next_in is None else next_in.shape[-1], _lib.ptr(counters), n_counters,
                           _lib.ptr(x0_out), out.shape[1] * H * W, VAR_TYPES[diff.model_var_type], tabs[7].data_ptr())
    return a, tabs


def _torch_step(diff, kind, clip, eta, t, x, out, noise):
    """the port's fp32 expression: p_mean_variance (:742-836, the learned variance :772-786) then p_sample
    (:887-891) / ddim_sample (:1010-1027) / ddim_reverse_sample (:1052-1066)"""
    tt = torch.full((x.shape[0],), t, device="cuda", dtype=torch.long)
    pmv = diff.p_mean_variance(lambda xx, ts, **k: out, x, tt, clip_denoised=clip)
    if kind == "reverse":
        return diff._ddim_reverse_finish(x, tt, pmv)
    return diff._ddim_finish(x, tt, pmv, noise, eta) if kind == "ddim" else diff._p_finish(x, tt, pmv, noise)


def _draw(g, mean, N=2, Cc=3, H=10, W=13):
    """x, a 2 C model output (variance values over [-1.5, 1.5]), noise; 780 elements per half: a partial last block"""
    x = torch.randn(N, Cc, H, W, device="cuda", generator=g) * 1.5
    out = torch.empty(N, 2 * Cc, H, W, device="cuda")
    out[:, :Cc] = torch.randn(N, Cc, H, W, device="cuda", generator=g) * (1.5 if mean == "x0" else 1.0)
    out[:, Cc:] = torch.rand(N, Cc, H, W, device="cuda", generator=g) * 3 - 1.5
    return x, out, torch.randn(N, Cc, H, W, device="cuda", generator=g)


# ------------------------------------------------------------------------------------------------ step kernel

@pytest.mark.parametrize("clip", [0, 1])
@pytest.mark.parametrize("var", [V.LEARNED, V.LEARNED_RANGE], ids=["learned", "learned_range"])
@pytest.mark.parametrize("mean", ["eps", "x0"])
def test_ancestral_step_reads_the_variance_half(mean, var, clip):
    diff = _diff(var, predict_xstart=mean == "x0")
    T = diff.num_timesteps
    g = torch.Generator(device="cuda").manual_seed(70 + 4 * clip + 2 * (mean == "x0") + (var == V.LEARNED))
    for t in (T - 1, T // 2, 0):
        x, out, noise = _draw(g, mean)
        N, Cc, H, W = x.shape
        x_next, x0 = torch.full_like(x, float("nan")), torch.full_like(x, float("nan"))
        cpad = Cc + 5
        next_in = torch.full((N * H * W, cpad), 7.0, dtype=torch.float16, device="cuda")
        counters = torch.full((9,), 5, dtype=torch.int32, device="cuda")
        a, _ = _step_args(diff, "ancestral", mean == "eps", clip, 0.0, t, x, out, noise, x_next, x0, next_in, counters, 6)
        _lib.check(_lib.lib.rs_op_ddpm_step(C.byref(a), G.stream()))
        torch.cuda.synchronize()
        ref = _torch_step(diff, "ancestral", bool(clip), 0.0, t, x, out, noise)
        tag = f"{mean} {var.name} clip={clip} t={t}"
        assert torch.equal(G.bits(x0), G.bits(ref["pred_xstart"])), f"{tag}: pred_xstart, {ulps(x0, ref['pred_xstart'])} ulp"
        assert torch.equal(G.bits(x_next), G.bits(ref["sample"])), f"{tag}: sample, {ulps(x_next, ref['sample'])} ulp"
        exp_next = torch.full_like(next_in, 7.0)
        if t > 0:
            exp_next[:, :Cc] = ref["sample"].permute(0, 2, 3, 1).reshape(-1, Cc).half()
        assert torch.equal(G.bits(next_in), G.bits(exp_next)), f"{tag}: next_in"
        assert counters[:6].eq(0).all() and counters[6:].eq(5).all(), f"{tag}: counters"
        if t > 0:
            # the variance half matters: other values give another sample
            out2 = out.clone()
            out2[:, Cc:] = -out[:, Cc:]
            a2, _ = _step_args(diff, "ancestral", mean == "eps", clip, 0.0, t, x, out2, noise, x_next, x0)
            _lib.check(_lib.lib.rs_op_ddpm_step(C.byref(a2), G.stream()))
            torch.cuda.synchronize()
            assert not torch.equal(x_next, ref["sample"]), f"{tag}: the variance half was not read"


@pytest.mark.parametrize("kind", ["ddim", "reverse"])
@pytest.mark.parametrize("mean", ["eps", "x0"])
def test_ddim_and_inversion_ignore_the_variance_half(kind, mean):
    diff = _diff(V.LEARNED_RANGE, predict_xstart=mean == "x0")
    T = diff.num_timesteps
    g = torch.Generator(device="cuda").manual_seed(80 + (mean == "x0") + 2 * (kind == "ddim"))
    for eta in ((0.0, 0.5, 1.0) if kind == "ddim" else (0.0,)):
        for clip in (0, 1):
            for t in (T - 1, T // 2, 0):
                x, out, noise = _draw(g, mean)
                N, Cc, H, W = x.shape
                ref = _torch_step(diff, kind, bool(clip), eta, t, x, out, noise)
                other = out.clone()
                other[:, Cc:] = torch.randn(N, Cc, H, W, device="cuda", generator=g) * 1e3
                tag = f"{kind} {mean} eta={eta} clip={clip} t={t}"
                for o in (out, other):
                    x_next, x0 = torch.full_like(x, float("nan")), torch.full_like(x, float("nan"))
                    if kind == "ddim":
                        a, _ = _step_args(diff, "ddim", mean == "eps", clip, eta, t, x, o, noise, x_next, x0)
                        _lib.check(_lib.lib.rs_op_ddpm_step(C.byref(a), G.stream()))
                    else:
                        tabs = [dev32(diff.sqrt_recip_alphas_cumprod), dev32(diff.sqrt_recipm1_alphas_cumprod),
                                dev32(diff.alphas_cumprod_next)]
                        a = _lib.DdimReverseStepArgsC(o.data_ptr(), x.data_ptr(), x_next.data_ptr(),
                                                      *(tb.data_ptr() for tb in tabs), T, t, N, Cc, H * W,
                                                      1 if mean == "eps" else 0, clip, None, 0, None, 0, x0.data_ptr(),
                                                      2 * Cc * H * W)
                        _lib.check(_lib.lib.rs_op_ddim_reverse_step(C.byref(a), G.stream()))
                    torch.cuda.synchronize()
                    assert torch.equal(G.bits(x0), G.bits(ref["pred_xstart"])), f"{tag}: pred_xstart"
                    assert torch.equal(G.bits(x_next), G.bits(ref["sample"])), (
                        f"{tag}: sample, {ulps(x_next, ref['sample'])} ulp")


def test_step_refusals():
    diff = _diff(V.LEARNED_RANGE)
    x = torch.zeros(1, 3, 4, 4, device="cuda")
    out = torch.zeros(1, 6, 4, 4, device="cuda")
    y = torch.empty_like(x)

    def refused(match, kind="ancestral", **over):
        a, tabs = _step_args(diff, kind, True, 0, 0.0, 3, x, out, x, y, None)
        for k, v in over.items():
            setattr(a, k, v)
        assert _lib.lib.rs_op_ddpm_step(C.byref(a), G.stream()) != 0, over
        assert match in _lib.lib.rs_last_error().decode(), (over, _lib.lib.rs_last_error())

    refused("unknown variance type", var_type=2)
    refused("unknown variance type", var_type=5)
    refused("needs log_betas", log_betas=None)
    refused("a learned variance needs at least 2 C * HW", out_sN=3 * 16)
    refused("a learned variance needs at least 2 C * HW", var_type=_lib.DDPM_VAR_TYPES["learned"], out_sN=5 * 16)
    refused("exactly for a fixed variance", var_type=0)
    refused("at least", kind="ddim", out_sN=2 * 16)
    tabs = [dev32(diff.sqrt_recip_alphas_cumprod)] * 3
    a = _lib.DdimReverseStepArgsC(out.data_ptr(), x.data_ptr(), y.data_ptr(), *(tb.data_ptr() for tb in tabs), 8, 3, 1,
                                  3, 16, 1, 0, None, 0, None, 0, None, 2 * 16)
    assert _lib.lib.rs_op_ddim_reverse_step(C.byref(a), G.stream()) != 0
    assert "is below C * HW" in _lib.lib.rs_last_error().decode()


# ------------------------------------------------------------------------------------------------ models


def _torch_route(diff, m, kind, first, noises, lq, clip, eta):
    """the torch route on the native UNet, step by step: every step's model output (for the variance half) and result"""
    T, B = diff.num_timesteps, first.shape[0]
    x, outs, rec = first, [], []
    for k in range(T):
        t = k if kind == "reverse" else T - 1 - k
        tt = torch.full((B,), t, device="cuda", dtype=torch.long)
        out = m(x, diff._model_t(tt), lq=lq)
        pmv = diff.p_mean_variance(lambda xx, ts, **kw: out, x, tt, clip_denoised=clip)
        if kind == "reverse":
            r = diff._ddim_reverse_finish(x, tt, pmv)
        elif kind == "ddim":
            r = diff._ddim_finish(x, tt, pmv, noises[k + 1], eta)
        else:
            r = diff._p_finish(x, tt, pmv, noises[k + 1])
        outs.append(out)
        rec.append(r)
        x = r["sample"]
    return outs, rec


def _fused(diff, m, kind, inputs, lq, clip, eta, monkeypatch):
    """the public progressive loop (fused: _native_ok holds), its randn_like draws fed from the fixture's noises"""
    if kind == "reverse":
        return list(diff.ddim_reverse_sample_loop_progressive(m, inputs, clip_denoised=clip, model_kwargs={"lq": lq}))
    queue = list(inputs[1:])
    monkeypatch.setattr(torch, "randn_like", lambda ref: queue.pop(0))
    kw = dict(noise=inputs[0], clip_denoised=clip, model_kwargs={"lq": lq})
    shape = tuple(inputs[0].shape)
    rec = list(diff.ddim_sample_loop_progressive(m, shape, eta=eta, **kw) if kind == "ddim"
               else diff.p_sample_loop_progressive(m, shape, **kw))
    monkeypatch.undo()
    assert not queue
    return rec


@pytest.mark.parametrize("case", sorted(CASES), ids=[f"{c}-{CASES[c][0]}-{CASES[c][2]}" for c in sorted(CASES)])
def test_fused_loop_matches_torch_route_and_reference(gold, case, monkeypatch):
    _, _, kind, _, clip, eta, _ = CASES[case]
    m, hw = learned_model(case)
    diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs(case))
    assert diff.model_var_type == V.LEARNED_RANGE and m.cfg.out_channels == 2 * m.x_channels == 6
    lq, inputs = (v.cuda() for v in case_inputs(case))
    assert diff._native_ok(m, None, {"lq": lq})
    rec = _fused(diff, m, kind, inputs, lq, clip, eta, monkeypatch)
    T, Cc = diff.num_timesteps, m.x_channels
    outs, ref = _torch_route(diff, m, kind, inputs if kind == "reverse" else inputs[0], inputs, lq, clip, eta)
    for k in range(T):
        assert torch.equal(G.bits(rec[k]["pred_xstart"]), G.bits(ref[k]["pred_xstart"])), f"pred_xstart k={k}"
        assert torch.equal(G.bits(rec[k]["sample"]), G.bits(ref[k]["sample"])), f"sample k={k}"
    if kind == "reverse":
        final = diff.reverse_latent(m, inputs, {"lq": lq}, clip)
    else:
        final = diff.sample_latent(m, inputs, {"lq": lq}, kind, clip, eta)
    assert torch.equal(G.bits(final), G.bits(rec[-1]["sample"])), "graph replay vs the eager taps"

    # against the reference's trajectory: test_gpu_ddpm's / test_gpu_ddim_reverse's bounds, element by element
    eps = diff.model_mean_type == gd.ModelMeanType.EPSILON
    d_prev = 0.0                                    # x_T = noises[0] (x_0 = x_start) exactly
    for k in range(T):
        t = k if kind == "reverse" else T - 1 - k
        f = float(diff.sqrt_recipm1_alphas_cumprod[t]) if eps else 1.0
        A, B = float(diff.sqrt_recip_alphas_cumprod[t]), float(diff.sqrt_recipm1_alphas_cumprod[t])
        ref_s, ref_x = gold[f"{case}/sample/{k}"], gold[f"{case}/pred_xstart/{k}"]
        got_s = rec[k]["sample"].reshape(-1)[::OUT_STRIDE].cpu().double().numpy()
        got_x = rec[k]["pred_xstart"].reshape(-1)[::OUT_STRIDE].cpu().double().numpy()
        mx, mn = bound(ref_x, f)
        carried = A * d_prev if eps else 0.0 * d_prev
        d_x = np.abs(got_x - ref_x)
        print(f"{case} pred_xstart {k}: max|d| {d_x.max():.3e} mean|d| {d_x.mean():.3e} (carried from x_t: max "
              f"{np.max(carried):.3e}; model bounds {mx:.3e} / {mn:.3e})")
        assert (d_x < carried + mx).all() and d_x.mean() < np.mean(carried) + mn, f"{case} pred_xstart {k}"
        var_max = var_mean = 0.0
        if kind == "reverse":
            an = float(diff.alphas_cumprod_next[t])
            carried = np.sqrt(an) * d_x + np.sqrt(1 - an) * (A * d_prev + d_x) / B
        elif kind == "ddim":
            ab, abp = float(diff.alphas_cumprod[t]), float(diff.alphas_cumprod_prev[t])
            sig = eta * np.sqrt((1 - abp) / (1 - ab)) * np.sqrt(1 - ab / abp)
            carried = np.sqrt(abp) * d_x + np.sqrt(max(1 - abp - sig ** 2, 0.0)) * (A * d_prev + d_x) / B
        else:
            carried = float(diff.posterior_mean_coef1[t]) * d_x + float(diff.posterior_mean_coef2[t]) * d_prev
            if t != 0:
                # the variance half's error |d v| (the model bound on v) moves log_var by |d v| |max_log - min_log| / 2,
                # and the sample by |noise| sd |d log_var| / 2 (first order; sd at the device's v, with 10% for the
                # second order and the reference's own sd)
                v = outs[k][:, Cc:].reshape(-1)[::OUT_STRIDE].cpu().double().numpy()
                lo, hi = float(diff.posterior_log_variance_clipped[t]), float(diff.log_betas[t])
                sd = np.exp(0.5 * ((v + 1) / 2 * hi + (1 - (v + 1) / 2) * lo))
                nz = np.abs(inputs[k + 1].reshape(-1)[::OUT_STRIDE].cpu().double().numpy())
                vmx, vmn = bound(v)
                var_max = 1.1 * 0.25 * nz * sd * abs(hi - lo) * vmx
                var_mean = float(np.mean(1.1 * 0.25 * nz * sd * abs(hi - lo))) * vmn
        mx, mn = bound(ref_s, f)
        d_s = np.abs(got_s - ref_s)
        print(f"{case} sample {k}: max|d| {d_s.max():.3e} mean|d| {d_s.mean():.3e} (carried: max "
              f"{np.max(carried):.3e}; variance max {np.max(var_max):.3e}; model bounds {mx:.3e} / {mn:.3e})")
        assert (d_s < carried + var_max + mx).all(), f"{case} sample {k}"
        assert d_s.mean() < np.mean(carried) + np.mean(var_max) + var_mean + mn, f"{case} sample {k}"
        d_prev = d_s
        last = (float(np.max(carried + var_max)) + mx, float(np.mean(carried + var_max)) + var_mean + mn)
    compare(f"{case} final", final.cpu(), gold[f"{case}/final"], last)     # every position, the last step's bounds


# ------------------------------------------------------------------------------------------------ loop properties

def test_learned_samplers_alternate_with_graph_replay():
    m, (H, W) = learned_model("d")
    anc, ddim = _diff(V.LEARNED_RANGE), _diff(V.LEARNED)
    g = torch.Generator(device="cuda").manual_seed(12)
    lq = torch.rand(2, 3, H, W, device="cuda", generator=g) * 2 - 1
    noises = torch.randn(9, 2, 3, H, W, device="cuda", generator=g)
    a1 = anc.sample_latent(m, noises, {"lq": lq}, "ancestral", False)
    d1 = ddim.sample_latent(m, noises, {"lq": lq}, "ddim", True, 0.5)
    a2 = anc.sample_latent(m, noises, {"lq": lq}, "ancestral", False)
    ae = anc.sample_latent(m, noises, {"lq": lq}, "ancestral", False, use_graph=False)
    de = ddim.sample_latent(m, noises, {"lq": lq}, "ddim", True, 0.5, use_graph=False)
    d2 = ddim.sample_latent(m, noises, {"lq": lq}, "ddim", True, 0.5)
    a3 = anc.sample_latent(m, noises, {"lq": lq}, "ancestral", False)
    assert torch.equal(G.bits(a1), G.bits(ae)) and torch.equal(G.bits(a2), G.bits(ae)) and torch.equal(G.bits(a3), G.bits(ae))
    assert torch.equal(G.bits(d1), G.bits(de)) and torch.equal(G.bits(d2), G.bits(de))
    assert not torch.equal(a1, d1)
    # LEARNED reads the variance values as the log variance itself: another sample than LEARNED_RANGE's
    l1 = _diff(V.LEARNED).sample_latent(m, noises, {"lq": lq}, "ancestral", False)
    assert not torch.equal(l1, a1)


def test_c_abi_refusals():
    fixed, (H, W) = cached_model("unetmodel", "legacy")
    learned, (H2, W2) = learned_model("d")
    assert (H, W) == (H2, W2)
    diff = _diff(V.LEARNED_RANGE)
    tabs = diff.ddpm_learned_range_tables()
    tp = tabs.ctypes.data_as(C.POINTER(C.c_double))
    tm = (C.c_int32 * 8)(*diff.timestep_map)

    def refused(model, match, tables=tp, **over):
        o = _lib.DdpmOptionsC(0, 1, 3, 0, 0.0)
        for k, v in over.items():
            setattr(o, k, v)
        h = C.c_void_p()
        rc = _lib.lib.rs_ddpm_sampler_create(model.plan(2, H, W).handle, 8, tables, tm, C.byref(o), C.byref(h))
        assert rc != 0 and not h.value, over
        assert match in _lib.lib.rs_last_error().decode(), (over, _lib.lib.rs_last_error())

    refused(fixed, "a learned variance type (3) needs a model with 6 output channels")
    refused(fixed, "a learned variance type (4) needs a model with 6 output channels", var_type=4, kind=1)
    refused(learned, "a fixed variance type (0) needs a model with 3 output channels", var_type=0)
    refused(learned, "a fixed variance type (1) needs a model with 3 output channels", var_type=1, kind=1)
    refused(learned, "schedule tables are NULL", tables=None)
    refused(learned, "unknown variance type", var_type=2)
    # the same model: a ResShift sampler keeps refusing a 2 C output
    from resshift_b200.config import DiffusionConfig
    rs = create_gaussian_diffusion(**DiffusionConfig(steps=4, min_noise_level=0.2, sf=1).to_kwargs())
    s = rs.native_sampler(learned, 2, H, W)
    buf = torch.zeros(6, 2, 3, H, W, device="cuda")
    lq = torch.zeros(2, 3, H, W, device="cuda")
    rc = _lib.lib.rs_sampler_run(s, buf.data_ptr(), buf.data_ptr(), lq.data_ptr(), None, buf.data_ptr(), 0, G.stream())
    assert rc != 0 and "x0 and x_t share a shape" in _lib.lib.rs_last_error().decode()
    # the inversion sampler takes a C or a 2 C output, and no other width (a UNetModelSwin can build a 3 C head)
    rtabs = diff.ddim_reverse_tables()
    rp = rtabs.ctypes.data_as(C.POINTER(C.c_double))

    def reverse_sampler(plan):
        h = C.c_void_p()
        rc = _lib.lib.rs_ddim_reverse_sampler_create(plan.handle, 8, rp, tm, C.byref(_lib.DdimReverseOptionsC(1, 0)),
                                                     C.byref(h))
        if rc == 0:
            _lib.lib.rs_sampler_destroy(h)
        return rc, h

    for model in (fixed, learned):
        rc, h = reverse_sampler(model.plan(2, H, W))
        assert rc == 0 and h.value, _lib.lib.rs_last_error()
    from resshift_b200.config import preset
    ucfg, _ = preset("tiny")
    ucfg.out_channels = 9
    wide = UNetModelSwin(**ucfg.to_kwargs())
    wide.load_state_dict(random_state_dict(ucfg, 0), strict=True)
    wide = wide.cuda().eval()
    rc, h = reverse_sampler(wide.plan(1, 64, 64))
    assert rc != 0 and not h.value
    assert "or twice as many (a learned variance), this plan's model has 9" in _lib.lib.rs_last_error().decode()
    # the fused route is gated the same way, and the torch route speaks for a mismatched model and variance type
    assert diff._native_ok(learned, None, {"lq": lq}) and not diff._native_ok(fixed, None, {"lq": lq})
    assert not diff._native_ok(wide, None, {"lq": lq})
    with pytest.raises(AssertionError):
        diff.p_sample_loop(fixed, (2, 3, H, W), model_kwargs={"lq": lq}, device="cuda")
