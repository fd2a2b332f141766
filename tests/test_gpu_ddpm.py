"""The DDPM / DDIM process (create_gaussian_diffusion_ddpm -> SpacedDiffusionDDPM) on the H100.

  * The step kernel (rs_op_ddpm_step, the launch the fused loop makes) for every combination: ancestral and DDIM, eps
    and x0 prediction, clip on and off, both fixed variances, eta in {0, 0.5, 1} for DDIM, t = T - 1, a middle step and
    0, element by element against the reference's torch fp32 expression (the port's p_mean_variance and step on the
    same inputs, on the device).  The kernel runs the same fp32 operations in the same order, so sample and pred_xstart
    must be bit-identical; exp (the ancestral step's exp(0.5 log_variance)) is CUDA's expf on both sides.
  * The fused loop of each UNet family, teacher-forced: every step is the native forward of its input at the mapped
    timestep, followed by exactly that step.
  * Fixture cases a-d (fused) against the unmodified reference's trajectories, and e (80 steps) and f (learned-range
    variance) through the torch route.
  * Graph replay == eager == replay, batch independence, a DDPM and a ResShift sampler alternating on one plan, and the
    C ABI's refusals.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import tests.gpu_util as G
from oracle.make_golden_ddpm import CASES, E_STEPS, FUSED, OUT_STRIDE, case_inputs, diffusion_kwargs, learned_range_model, model_config
from resshift_b200 import _lib
from resshift_b200.models import gaussian_diffusion as gd
from resshift_b200.models.script_util import create_gaussian_diffusion, create_gaussian_diffusion_ddpm
from tests.sampler_ref import bound, cached_model, compare, dev32, ulps

pytestmark = pytest.mark.gpu

KW8 = dict(beta_start=0.0015, beta_end=0.0155, steps=1000, timestep_respacing=8)
ROWS = ("sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_mean_coef1", "posterior_mean_coef2")


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(golden_dir / "ddpm.npz")


def _step_args(diff, kind, mean_eps, clip, eta, t, x, out, noise, x_next, x0_out, next_in=None, counters=None, n_counters=0):
    tabs = {n: dev32(getattr(diff, n)) for n in ROWS}
    small = diff.model_var_type == gd.ModelVarTypeDDPM.FIXED_SMALL
    tabs["log_var"] = dev32(diff.posterior_log_variance_clipped if small else diff.log_variance_fixed_large)
    tabs["acp"], tabs["acp_prev"] = dev32(diff.alphas_cumprod), dev32(diff.alphas_cumprod_prev)
    N, Cc, H, W = x.shape
    a = _lib.DdpmStepArgsC(out.data_ptr(), x.data_ptr(), noise.data_ptr(), x_next.data_ptr(),
                           tabs[ROWS[0]].data_ptr(), tabs[ROWS[1]].data_ptr(), tabs[ROWS[2]].data_ptr(),
                           tabs[ROWS[3]].data_ptr(), tabs["log_var"].data_ptr(), tabs["acp"].data_ptr(),
                           tabs["acp_prev"].data_ptr(), diff.num_timesteps, t, N, Cc, H * W,
                           _lib.DDPM_KINDS[kind], 1 if mean_eps else 0, int(clip), float(eta),
                           _lib.ptr(next_in), 0 if next_in is None else next_in.shape[-1], _lib.ptr(counters), n_counters,
                           _lib.ptr(x0_out))
    return a, tabs


def _torch_step(diff, kind, clip, eta, t, x, out, noise):
    """the reference's fp32 expression: p_mean_variance (:742-836) then p_sample (:887-891) / ddim_sample (:1010-1027)"""
    tt = torch.full((x.shape[0],), t, device="cuda", dtype=torch.long)
    pmv = diff.p_mean_variance(lambda xx, ts, **k: out, x, tt, clip_denoised=clip)
    return diff._ddim_finish(x, tt, pmv, noise, eta) if kind == "ddim" else diff._p_finish(x, tt, pmv, noise)


# ------------------------------------------------------------------------------------------------ step kernel

@pytest.mark.parametrize("var", ["fixed_large", "fixed_small"])
@pytest.mark.parametrize("clip", [0, 1])
@pytest.mark.parametrize("mean", ["eps", "x0"])
@pytest.mark.parametrize("kind", ["ancestral", "ddim"])
def test_step_kernel_is_reference_expression(kind, mean, clip, var):
    diff = create_gaussian_diffusion_ddpm(predict_xstart=mean == "x0", sigma_small=var == "fixed_small", **KW8)
    T = diff.num_timesteps
    g = torch.Generator(device="cuda").manual_seed(7 + 2 * clip + (mean == "x0"))
    N, Cc, H, W = 2, 3, 10, 13            # 780 elements: a partial last block
    etas = (0.0, 0.5, 1.0) if kind == "ddim" else (0.0,)
    for eta in etas:
        for t in (T - 1, T // 2, 0):
            x = torch.randn(N, Cc, H, W, device="cuda", generator=g) * 1.5
            out = torch.randn(N, Cc, H, W, device="cuda", generator=g) * (1.5 if mean == "x0" else 1.0)
            noise = torch.randn(N, Cc, H, W, device="cuda", generator=g)
            x_next = torch.full_like(x, float("nan"))
            x0 = torch.full_like(x, float("nan"))
            cpad = Cc + 5
            next_in = torch.full((N * H * W, cpad), 7.0, dtype=torch.float16, device="cuda")
            counters = torch.full((9,), 5, dtype=torch.int32, device="cuda")
            a, _ = _step_args(diff, kind, mean == "eps", clip, eta, t, x, out, noise, x_next, x0, next_in, counters, 6)
            _lib.check(_lib.lib.rs_op_ddpm_step(C.byref(a), G.stream()))
            torch.cuda.synchronize()
            ref = _torch_step(diff, kind, bool(clip), eta, t, x, out, noise)
            tag = f"{kind} {mean} clip={clip} {var} eta={eta} t={t}"
            assert torch.equal(G.bits(x0), G.bits(ref["pred_xstart"])), f"{tag}: pred_xstart, {ulps(x0, ref['pred_xstart'])} ulp"
            assert torch.equal(G.bits(x_next), G.bits(ref["sample"])), f"{tag}: sample, {ulps(x_next, ref['sample'])} ulp"
            if clip:
                assert x0.abs().max() <= 1.0
            exp_next = torch.full_like(next_in, 7.0)
            if t > 0:
                exp_next[:, :Cc] = ref["sample"].permute(0, 2, 3, 1).reshape(-1, Cc).half()
            assert torch.equal(G.bits(next_in), G.bits(exp_next)), f"{tag}: next_in"
            assert counters[:6].eq(0).all() and counters[6:].eq(5).all(), f"{tag}: counters"


def test_step_kernel_refusals():
    diff = create_gaussian_diffusion_ddpm(**KW8)
    x = torch.zeros(1, 3, 4, 4, device="cuda")
    y = torch.empty_like(x)

    def refused(match, **over):
        a, tabs = _step_args(diff, "ddim", True, 0, 0.0, 3, x, x, x, y, None)
        for k, v in over.items():
            setattr(a, k, v)
        rc = _lib.lib.rs_op_ddpm_step(C.byref(a), G.stream())
        assert rc != 0, over
        assert match in _lib.lib.rs_last_error().decode(), (over, _lib.lib.rs_last_error())

    refused("unknown kind", kind=2)
    refused("predict eps or x0", mean_type=_lib.MEAN_TYPES["residual"])
    refused("eta must be >= 0", eta=-0.5)
    refused("clip must be 0 or 1", clip=2)
    refused("t must be in [0, T", t=8)
    refused("t must be in [0, T", t=-1)
    refused("acp / acp_prev", acp=None)
    refused("sqrt_recip_acp", sqrt_recipm1_acp=None)
    refused("next_cpad", next_in=x.data_ptr(), next_cpad=2)
    refused("n_counters", n_counters=4)


# ------------------------------------------------------------------------------------------------ models

# (family, model case, loop, diffusion kwargs, clip, eta)
TEACHER = [
    ("swin", "tiny", "ancestral", dict(predict_xstart=True, sigma_small=True), True, 0.0),
    ("unetmodel", "legacy", "ddim", dict(), False, 0.5),
    ("unetconv", "defaults", "ancestral", dict(), True, 0.0),
    ("unetmodel", "legacy", "ddim", dict(predict_xstart=True), True, 1.0),
]


@pytest.mark.parametrize("family,name,loop,kw,clip,eta", TEACHER, ids=[f"{t[0]}-{t[2]}" for t in TEACHER])
def test_loop_is_forwards_and_steps(family, name, loop, kw, clip, eta):
    m, (H, W) = cached_model(family, name)
    diff = create_gaussian_diffusion_ddpm(**KW8, **kw)
    assert diff.timestep_map != list(range(diff.num_timesteps))
    T, B = diff.num_timesteps, 2
    g = torch.Generator(device="cuda").manual_seed(99)
    lq = torch.rand(B, 3, H, W, device="cuda", generator=g) * 2 - 1
    noises = torch.randn(T + 1, B, 3, H, W, device="cuda", generator=g)
    rec = list(diff._native_progressive(m, noises, {"lq": lq}, loop, clip, eta))
    assert len(rec) == T
    for k in range(T):
        t = T - 1 - k
        x_t = noises[0] if k == 0 else rec[k - 1]["sample"]
        ts = torch.full((B,), float(diff.timestep_map[t]), device="cuda")
        out = m._run_forward(x_t, ts, lq, None)
        ref = _torch_step(diff, loop, clip, eta, t, x_t, out, noises[k + 1])
        assert torch.equal(G.bits(rec[k]["pred_xstart"]), G.bits(ref["pred_xstart"])), f"pred_xstart k={k}"
        assert torch.equal(G.bits(rec[k]["sample"]), G.bits(ref["sample"])), f"sample k={k}"
    final = diff.sample_latent(m, noises, {"lq": lq}, loop, clip, eta)
    assert torch.equal(G.bits(final), G.bits(rec[-1]["sample"])), "graph replay vs the eager taps"


# ------------------------------------------------------------------------------------------------ fixtures a-f

def _case_model(case):
    family, name = CASES[case][:2]
    m, hw = cached_model(family, name)
    assert hw == model_config(case)[1]
    return m, hw


def _progressive(diff, loop, m, noises, lq, clip, eta, monkeypatch):
    """the public progressive loop, its randn / randn_like draws fed from the fixture's noises"""
    queue = list(noises[1:])
    monkeypatch.setattr(torch, "randn_like", lambda ref: queue.pop(0))
    kw = dict(noise=noises[0], clip_denoised=clip, model_kwargs={"lq": lq})
    fn = diff.ddim_sample_loop_progressive if loop == "ddim" else diff.p_sample_loop_progressive
    rec = list(fn(m, tuple(noises[0].shape), eta=eta, **kw) if loop == "ddim" else fn(m, tuple(noises[0].shape), **kw))
    monkeypatch.undo()
    assert not queue
    return rec


@pytest.mark.parametrize("case", FUSED)
def test_fused_case_matches_reference(gold, case, monkeypatch):
    _, _, _, loop, _, clip, eta, _ = CASES[case]
    m, hw = _case_model(case)
    diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs(case))
    lq, noises = (v.cuda() for v in case_inputs(case, hw=hw))
    assert diff._native_ok(m, None, {"lq": lq})
    rec = _progressive(diff, loop, m, noises, lq, clip, eta, monkeypatch)
    eps = diff.model_mean_type == gd.ModelMeanType.EPSILON
    T = diff.num_timesteps
    d_prev = 0.0                                    # x_T = noises[0] exactly
    for k in range(T):
        t = T - 1 - k
        f = float(diff.sqrt_recipm1_alphas_cumprod[t]) if eps else 1.0
        A, B = float(diff.sqrt_recip_alphas_cumprod[t]), float(diff.sqrt_recipm1_alphas_cumprod[t])
        ref_s, ref_x = gold[f"{case}/sample/{k}"], gold[f"{case}/pred_xstart/{k}"]
        got_s = rec[k]["sample"].reshape(-1)[::OUT_STRIDE].cpu().double().numpy()
        got_x = rec[k]["pred_xstart"].reshape(-1)[::OUT_STRIDE].cpu().double().numpy()
        # Element by element (the step is elementwise, and the fixture's sub-sampled positions are the same for every
        # step), each result's error is what the step carries from the errors of its inputs at that position, plus the
        # model-output bound: x0 carries sqrt(1 / acp_t) |d x_t| for eps prediction (the clamp only shrinks errors);
        # the ancestral sample coef1 |d x0| + coef2 |d x_t|; the DDIM sample sqrt(acp_prev) |d x0| + sqrt(1 - acp_prev -
        # sigma^2) |d eps'| with |d eps'| <= (sqrt(1 / acp_t) |d x_t| + |d x0|) / sqrt(1 / acp_t - 1).
        mx, mn = bound(ref_x, f)
        carried = A * d_prev if eps else 0.0 * d_prev
        d_x = np.abs(got_x - ref_x)
        print(f"{case} pred_xstart {k}: max|d| {d_x.max():.3e} mean|d| {d_x.mean():.3e} (carried from x_t: max "
              f"{np.max(carried):.3e}; model bounds {mx:.3e} / {mn:.3e})")
        assert (d_x < carried + mx).all() and d_x.mean() < np.mean(carried) + mn, f"{case} pred_xstart {k}"
        if loop == "ddim":
            ab, abp = float(diff.alphas_cumprod[t]), float(diff.alphas_cumprod_prev[t])
            sig = eta * np.sqrt((1 - abp) / (1 - ab)) * np.sqrt(1 - ab / abp)
            carried = np.sqrt(abp) * d_x + np.sqrt(max(1 - abp - sig ** 2, 0.0)) * (A * d_prev + d_x) / B
        else:
            carried = float(diff.posterior_mean_coef1[t]) * d_x + float(diff.posterior_mean_coef2[t]) * d_prev
        mx, mn = bound(ref_s, f)
        d_s = np.abs(got_s - ref_s)
        print(f"{case} sample {k}: max|d| {d_s.max():.3e} mean|d| {d_s.mean():.3e} (carried: max "
              f"{np.max(carried):.3e}; model bounds {mx:.3e} / {mn:.3e})")
        assert (d_s < carried + mx).all() and d_s.mean() < np.mean(carried) + mn, f"{case} sample {k}"
        d_prev = d_s
        last = (float(np.max(carried)) + mx, float(np.mean(carried)) + mn)
    final = diff.sample_latent(m, noises, {"lq": lq}, loop, clip, eta)
    assert torch.equal(G.bits(final), G.bits(rec[-1]["sample"]))
    compare(f"{case} final", final.cpu(), gold[f"{case}/final"], last)     # every position, the last step's bounds
    if case == "a":
        from resshift_b200.models.autoencoder import VQModelTorch
        from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
        vcfg = vq_preset("tiny")
        vq = VQModelTorch(**vcfg.to_kwargs())
        vq.load_state_dict(random_vq_state_dict(vcfg, 0), strict=True)
        vq = vq.cuda().eval()
        # the bookend on the reference's own final latent: the decode alone
        ref_dec = diff.decode_first_stage(torch.from_numpy(gold["a/final"]).cuda(), vq)
        compare("a decoded (reference latent)", ref_dec.reshape(-1)[::OUT_STRIDE].cpu(), gold["a/decoded"])
        # end to end: the nearest-code quantiser turns the loop's latent error into a whole code wherever it crosses a
        # boundary between codes, so the decoded image is held to the mean bound only
        dec = diff.decode_first_stage(final, vq)
        ref = gold["a/decoded"]
        compare("a decoded", dec.reshape(-1)[::OUT_STRIDE].cpu(), ref, bounds=(float("inf"), bound(ref)[1]))
        # p_sample_loop returns the same decoded image
        queue = list(noises[1:])
        monkeypatch.setattr(torch, "randn_like", lambda ref: queue.pop(0))
        out = diff.p_sample_loop(m, tuple(noises[0].shape), noise=noises[0], clip_denoised=clip,
                                 first_stage_model=vq, model_kwargs={"lq": lq})
        monkeypatch.undo()
        assert torch.equal(G.bits(out), G.bits(dec))


def test_generic_route_80_steps(gold, monkeypatch):
    """case e: T = 80 is above the fused loop's 64 steps, so the torch route runs the native UNet step by step"""
    _, _, _, loop, _, clip, eta, _ = CASES["e"]
    m, hw = _case_model("e")
    diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs("e"))
    lq, noises = (v.cuda() for v in case_inputs("e", hw=hw))
    assert diff.num_timesteps == 80 and not diff._native_ok(m, None, {"lq": lq})
    rec = _progressive(diff, loop, m, noises, lq, clip, eta, monkeypatch)
    for k in E_STEPS:
        compare(f"e sample {k}", rec[k]["sample"].reshape(-1)[::OUT_STRIDE].cpu(), gold[f"e/sample/{k}"])
    compare("e final", rec[-1]["sample"].cpu(), gold["e/final"])


def test_generic_route_learned_range(gold, monkeypatch):
    """case f: LEARNED_RANGE on the torch route, on the device (fp32 torch on CUDA against fp32 torch on the CPU: only
    tanh / sin / exp implementations differ)"""
    diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs("f"))
    lq, noises = (v.cuda() for v in case_inputs("f", hw=(16, 16)))
    queue = list(noises[1:])
    monkeypatch.setattr(torch, "randn_like", lambda ref: queue.pop(0))
    out = diff.p_sample_loop(learned_range_model, tuple(noises[0].shape), noise=noises[0], clip_denoised=False,
                             model_kwargs={"lq": lq}, device="cuda")
    monkeypatch.undo()
    ref = gold["f/final"]
    compare("f final", out.cpu(), ref, bounds=(1e-4 * np.abs(ref).max(), 1e-5 * np.abs(ref).max()))


# ------------------------------------------------------------------------------------------------ loop properties

def test_graph_replay_equals_eager():
    m, (H, W) = cached_model("unetmodel", "legacy")
    diff = create_gaussian_diffusion_ddpm(**KW8)
    g = torch.Generator(device="cuda").manual_seed(5)
    lq = torch.rand(2, 3, H, W, device="cuda", generator=g) * 2 - 1
    noises = torch.randn(9, 2, 3, H, W, device="cuda", generator=g)
    for loop, eta in (("ancestral", 0.0), ("ddim", 0.0), ("ddim", 1.0)):
        r1 = diff.sample_latent(m, noises, {"lq": lq}, loop, True, eta)
        e = diff.sample_latent(m, noises, {"lq": lq}, loop, True, eta, use_graph=False)
        r2 = diff.sample_latent(m, noises, {"lq": lq}, loop, True, eta)
        assert torch.equal(G.bits(r1), G.bits(e)) and torch.equal(G.bits(r2), G.bits(e)), (loop, eta)


def test_image_independent_of_batch():
    m, (H, W) = cached_model("unetconv", "defaults")
    diff = create_gaussian_diffusion_ddpm(**KW8)
    g = torch.Generator(device="cuda").manual_seed(6)
    lq = torch.rand(2, 3, H, W, device="cuda", generator=g) * 2 - 1
    noises = torch.randn(9, 2, 3, H, W, device="cuda", generator=g)
    a = diff.sample_latent(m, noises, {"lq": lq}, "ddim", True, 0.5)
    lq2, n2 = lq.clone(), noises.clone()
    lq2[1] = torch.rand(3, H, W, device="cuda", generator=g)
    n2[:, 1] = torch.randn(9, 3, H, W, device="cuda", generator=g)
    b = diff.sample_latent(m, n2, {"lq": lq2}, "ddim", True, 0.5)
    assert torch.equal(G.bits(a[0]), G.bits(b[0]))
    assert not torch.equal(a[1], b[1])


def test_ddpm_and_resshift_samplers_alternate_on_one_plan():
    from resshift_b200.config import DiffusionConfig
    m, (H, W) = cached_model("unetmodel", "legacy")
    rs = create_gaussian_diffusion(**DiffusionConfig(steps=4, min_noise_level=0.2, sf=1).to_kwargs())
    dd = create_gaussian_diffusion_ddpm(**KW8)
    g = torch.Generator(device="cuda").manual_seed(8)
    zy = torch.randn(2, 3, H, W, device="cuda", generator=g)
    lq = torch.rand(2, 3, H, W, device="cuda", generator=g) * 2 - 1
    rn = torch.randn(5, 2, 3, H, W, device="cuda", generator=g)
    dn = torch.randn(9, 2, 3, H, W, device="cuda", generator=g)
    r1 = rs.sample_latent(zy, m, {"lq": lq}, noises=rn)
    d1 = dd.sample_latent(m, dn, {"lq": lq}, "ancestral", True)
    r2 = rs.sample_latent(zy, m, {"lq": lq}, noises=rn)
    d2 = dd.sample_latent(m, dn, {"lq": lq}, "ancestral", True)
    e1 = dd.sample_latent(m, dn, {"lq": lq}, "ddim", False, 0.3)
    r3 = rs.sample_latent(zy, m, {"lq": lq}, noises=rn, use_graph=False)
    e2 = dd.sample_latent(m, dn, {"lq": lq}, "ddim", False, 0.3, use_graph=False)
    assert torch.equal(G.bits(r1), G.bits(r2)) and torch.equal(G.bits(r1), G.bits(r3))
    assert torch.equal(G.bits(d1), G.bits(d2)) and torch.equal(G.bits(e1), G.bits(e2))
    assert not torch.equal(d1, e1) and not torch.equal(r1, d1)


def test_c_abi_refusals():
    m, (H, W) = cached_model("unetmodel", "legacy")
    plan = m.plan(2, H, W)
    diff = create_gaussian_diffusion_ddpm(**KW8)
    tabs = diff.ddpm_tables()
    tp = tabs.ctypes.data_as(C.POINTER(C.c_double))
    tm = (C.c_int32 * 8)(*diff.timestep_map)

    def refused(match, steps=8, tables=tp, **over):
        o = _lib.DdpmOptionsC(0, 1, 0, 0, 0.0)
        for k, v in over.items():
            setattr(o, k, v)
        h = C.c_void_p()
        rc = _lib.lib.rs_ddpm_sampler_create(plan.handle, steps, tables, tm, C.byref(o), C.byref(h))
        assert rc != 0 and not h.value, over
        assert match in _lib.lib.rs_last_error().decode(), (over, _lib.lib.rs_last_error())

    refused("unknown kind", kind=2)
    refused("unknown kind", kind=-1)
    refused("predict eps or x0", mean_type=_lib.MEAN_TYPES["residual"])
    refused("predict eps or x0", mean_type=_lib.MEAN_TYPES["epsilon_scale"])
    refused("unknown variance type", var_type=2)
    refused("clip must be 0 or 1", clip=2)
    refused("eta must be finite and >= 0", eta=-1e-3)
    refused("eta must be finite and >= 0", eta=float("nan"))
    refused("eta must be finite and >= 0", eta=float("inf"))
    refused("schedule tables are NULL", tables=None)
    refused("steps must be in [2, 64]", steps=1)
    big = np.ones((8, 65)) * 0.5
    refused("steps must be in [2, 64]", steps=65, tables=big.ctypes.data_as(C.POINTER(C.c_double)))
    h = C.c_void_p()
    rc = _lib.lib.rs_ddpm_sampler_create(plan.handle, 8, tp, tm, None, C.byref(h))
    assert rc != 0 and "options are NULL" in _lib.lib.rs_last_error().decode()
    # a DDPM sampler has no residual-shift tables, and ResShift samplers keep refusing a NULL z_y
    h = diff.native_sampler(m, 2, H, W, "ancestral", True)
    assert _lib.lib.rs_sampler_tables(h, (C.c_float * 41)()) != 0
    assert "DDPM sampler" in _lib.lib.rs_last_error().decode()
    from resshift_b200.config import DiffusionConfig
    rs = create_gaussian_diffusion(**DiffusionConfig(steps=4, min_noise_level=0.2, sf=1).to_kwargs())
    s = rs.native_sampler(m, 2, H, W)
    buf = torch.zeros(6, 2, 3, H, W, device="cuda")
    rc = _lib.lib.rs_sampler_run(s, None, buf.data_ptr(), buf.data_ptr(), None, buf.data_ptr(), 0, G.stream())
    assert rc != 0 and "null argument" in _lib.lib.rs_last_error().decode()
