"""DDIM inversion (SpacedDiffusionDDPM.ddim_reverse_sample and ddim_reverse_sample_loop) on the H100.

  * The reverse step kernel (rs_op_ddim_reverse_step, the launch the fused loop makes) for eps and x0 prediction, clip
    on and off, t = 0, a middle step and T - 1 (where acp_next is 0), element by element against the port's torch fp32
    expression on the device: the kernel runs the same fp32 operations in the same order, so sample and pred_xstart
    must be bit-identical.
  * The fused loop of each UNet family, teacher-forced: every step is the native forward of its input at the mapped
    timestep, followed by exactly that step.
  * Fixture cases a-d (fused) against the unmodified reference's trajectories, within test_gpu_ddpm's loop bounds, and
    case e (learned-range variance) through the torch route.
  * Graph replay == eager == replay, batch independence, reverse, DDPM and ResShift samplers alternating on one plan,
    inversion followed by ddim_sample_loop on the fused and on the torch route, the host entry point, and the C ABI's
    refusals.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import tests.gpu_util as G
from oracle.make_golden_ddim_reverse import CASES, FUSED, OUT_STRIDE, case_inputs, diffusion_kwargs, model_config
from oracle.make_golden_ddpm import learned_range_model
from resshift_b200 import _lib
from resshift_b200.models import gaussian_diffusion as gd
from resshift_b200.models.script_util import create_gaussian_diffusion, create_gaussian_diffusion_ddpm
from tests.sampler_ref import bound, cached_model, compare, dev32, ulps

pytestmark = pytest.mark.gpu

KW8 = dict(beta_start=0.0015, beta_end=0.0155, steps=1000, timestep_respacing=8)


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(golden_dir / "ddim_reverse.npz")


def _step_args(diff, mean_eps, clip, t, x, out, x_next, x0_out, next_in=None, counters=None, n_counters=0):
    tabs = [dev32(diff.sqrt_recip_alphas_cumprod), dev32(diff.sqrt_recipm1_alphas_cumprod),
            dev32(diff.alphas_cumprod_next)]
    N, Cc, H, W = x.shape
    a = _lib.DdimReverseStepArgsC(out.data_ptr(), x.data_ptr(), x_next.data_ptr(),
                                  tabs[0].data_ptr(), tabs[1].data_ptr(), tabs[2].data_ptr(),
                                  diff.num_timesteps, t, N, Cc, H * W, 1 if mean_eps else 0, int(clip),
                                  _lib.ptr(next_in), 0 if next_in is None else next_in.shape[-1], _lib.ptr(counters),
                                  n_counters, _lib.ptr(x0_out))
    return a, tabs


def _torch_step(diff, clip, t, x, out):
    """the port's fp32 expression: p_mean_variance (:742-836), then ddim_reverse_sample's eps and update (:1052-1066)"""
    tt = torch.full((x.shape[0],), t, device="cuda", dtype=torch.long)
    return diff.ddim_reverse_sample(lambda xx, ts, **k: out, x, tt, clip_denoised=clip)


# ------------------------------------------------------------------------------------------------ step kernel

@pytest.mark.parametrize("clip", [0, 1])
@pytest.mark.parametrize("mean", ["eps", "x0"])
def test_step_kernel_is_reference_expression(mean, clip):
    diff = create_gaussian_diffusion_ddpm(predict_xstart=mean == "x0", **KW8)
    T = diff.num_timesteps
    assert diff.alphas_cumprod_next[T - 1] == 0.0
    g = torch.Generator(device="cuda").manual_seed(17 + 2 * clip + (mean == "x0"))
    N, Cc, H, W = 2, 3, 10, 13            # 780 elements: a partial last block
    for t in (0, T // 2, T - 1):
        x = torch.randn(N, Cc, H, W, device="cuda", generator=g) * 1.5
        out = torch.randn(N, Cc, H, W, device="cuda", generator=g) * (1.5 if mean == "x0" else 1.0)
        x_next = torch.full_like(x, float("nan"))
        x0 = torch.full_like(x, float("nan"))
        cpad = Cc + 5
        next_in = torch.full((N * H * W, cpad), 7.0, dtype=torch.float16, device="cuda")
        counters = torch.full((9,), 5, dtype=torch.int32, device="cuda")
        a, _ = _step_args(diff, mean == "eps", clip, t, x, out, x_next, x0, next_in, counters, 6)
        _lib.check(_lib.lib.rs_op_ddim_reverse_step(C.byref(a), G.stream()))
        torch.cuda.synchronize()
        ref = _torch_step(diff, bool(clip), t, x, out)
        tag = f"{mean} clip={clip} t={t}"
        assert torch.equal(G.bits(x0), G.bits(ref["pred_xstart"])), f"{tag}: pred_xstart, {ulps(x0, ref['pred_xstart'])} ulp"
        assert torch.equal(G.bits(x_next), G.bits(ref["sample"])), f"{tag}: sample, {ulps(x_next, ref['sample'])} ulp"
        if clip:
            assert x0.abs().max() <= 1.0
        exp_next = torch.full_like(next_in, 7.0)
        if t < T - 1:
            exp_next[:, :Cc] = ref["sample"].permute(0, 2, 3, 1).reshape(-1, Cc).half()
        assert torch.equal(G.bits(next_in), G.bits(exp_next)), f"{tag}: next_in"
        assert counters[:6].eq(0).all() and counters[6:].eq(5).all(), f"{tag}: counters"


def test_step_kernel_refusals():
    diff = create_gaussian_diffusion_ddpm(**KW8)
    x = torch.zeros(1, 3, 4, 4, device="cuda")
    y = torch.empty_like(x)

    def refused(match, **over):
        a, tabs = _step_args(diff, True, 0, 3, x, x, y, None)
        for k, v in over.items():
            setattr(a, k, v)
        rc = _lib.lib.rs_op_ddim_reverse_step(C.byref(a), G.stream())
        assert rc != 0, over
        assert match in _lib.lib.rs_last_error().decode(), (over, _lib.lib.rs_last_error())

    refused("predict eps or x0", mean_type=_lib.MEAN_TYPES["residual"])
    refused("clip must be 0 or 1", clip=2)
    refused("t must be in [0, T", t=8)
    refused("t must be in [0, T", t=-1)
    refused("acp_next are NULL", acp_next=None)
    refused("acp_next are NULL", sqrt_recip_acp=None)
    refused("acp_next are NULL", sqrt_recipm1_acp=None)
    refused("next_cpad", next_in=x.data_ptr(), next_cpad=2)
    refused("n_counters", n_counters=4)


# ------------------------------------------------------------------------------------------------ teacher-forced loop

# (family, model case, diffusion kwargs, clip)
TEACHER = [
    ("swin", "tiny", dict(predict_xstart=True), True),
    ("unetmodel", "legacy", dict(), False),
    ("unetconv", "defaults", dict(), True),
    ("unetmodel", "legacy", dict(predict_xstart=True), False),
]


@pytest.mark.parametrize("family,name,kw,clip", TEACHER,
                         ids=[f"{t[0]}-{'x0' if t[2] else 'eps'}-clip{int(t[3])}" for t in TEACHER])
def test_loop_is_forwards_and_steps(family, name, kw, clip):
    m, (H, W) = cached_model(family, name)
    diff = create_gaussian_diffusion_ddpm(**KW8, **kw)
    assert diff.timestep_map != list(range(diff.num_timesteps))
    T, B = diff.num_timesteps, 2
    g = torch.Generator(device="cuda").manual_seed(199)
    lq = torch.rand(B, 3, H, W, device="cuda", generator=g) * 2 - 1
    x_start = torch.rand(B, 3, H, W, device="cuda", generator=g) * 2 - 1
    rec = list(diff._native_reverse_progressive(m, x_start, {"lq": lq}, clip))
    assert len(rec) == T
    for t in range(T):
        x_t = x_start if t == 0 else rec[t - 1]["sample"]
        ts = torch.full((B,), float(diff.timestep_map[t]), device="cuda")
        out = m._run_forward(x_t, ts, lq, None)
        ref = _torch_step(diff, clip, t, x_t, out)
        assert torch.equal(G.bits(rec[t]["pred_xstart"]), G.bits(ref["pred_xstart"])), f"pred_xstart t={t}"
        assert torch.equal(G.bits(rec[t]["sample"]), G.bits(ref["sample"])), f"sample t={t}"
    final = diff.reverse_latent(m, x_start, {"lq": lq}, clip)
    assert torch.equal(G.bits(final), G.bits(rec[-1]["sample"])), "graph replay vs the eager taps"
    # the public loops take the fused route for this model
    assert diff._native_ok(m, None, {"lq": lq})
    pub = diff.ddim_reverse_sample_loop(m, x_start, clip_denoised=clip, model_kwargs={"lq": lq})
    assert torch.equal(G.bits(pub), G.bits(final))
    prog = list(diff.ddim_reverse_sample_loop_progressive(m, x_start, clip_denoised=clip, model_kwargs={"lq": lq}))
    assert all(torch.equal(G.bits(p["sample"]), G.bits(r["sample"])) for p, r in zip(prog, rec))


# ------------------------------------------------------------------------------------------------ fixtures a-e

@pytest.mark.parametrize("case", FUSED)
def test_fused_case_matches_reference(gold, case):
    family, name, kw, clip, _ = CASES[case]
    m, hw = cached_model(family, name)
    assert hw == model_config(case)[1]
    diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs(case))
    lq, x_start = (v.cuda() for v in case_inputs(case))
    assert diff._native_ok(m, None, {"lq": lq})
    rec = list(diff.ddim_reverse_sample_loop_progressive(m, x_start, clip_denoised=clip, model_kwargs={"lq": lq}))
    eps = diff.model_mean_type == gd.ModelMeanType.EPSILON
    T = diff.num_timesteps
    d_prev = 0.0                                    # x_0 = x_start exactly
    for t in range(T):
        f = float(diff.sqrt_recipm1_alphas_cumprod[t]) if eps else 1.0
        A, B = float(diff.sqrt_recip_alphas_cumprod[t]), float(diff.sqrt_recipm1_alphas_cumprod[t])
        an = float(diff.alphas_cumprod_next[t])
        ref_s, ref_x = gold[f"{case}/sample/{t}"], gold[f"{case}/pred_xstart/{t}"]
        got_s = rec[t]["sample"].reshape(-1)[::OUT_STRIDE].cpu().double().numpy()
        got_x = rec[t]["pred_xstart"].reshape(-1)[::OUT_STRIDE].cpu().double().numpy()
        # test_gpu_ddpm's loop bounds, element by element: each result carries the errors of its inputs at that
        # position, plus the model-output bound.  x0 carries sqrt(1 / acp_t) |d x_t| for eps prediction (the clamp only
        # shrinks errors); the sample sqrt(acp_next) |d x0| + sqrt(1 - acp_next) |d eps'| with
        # |d eps'| <= (sqrt(1 / acp_t) |d x_t| + |d x0|) / sqrt(1 / acp_t - 1).
        mx, mn = bound(ref_x, f)
        carried = A * d_prev if eps else 0.0 * d_prev
        d_x = np.abs(got_x - ref_x)
        print(f"{case} pred_xstart {t}: max|d| {d_x.max():.3e} mean|d| {d_x.mean():.3e} (carried from x_t: max "
              f"{np.max(carried):.3e}; model bounds {mx:.3e} / {mn:.3e})")
        assert (d_x < carried + mx).all() and d_x.mean() < np.mean(carried) + mn, f"{case} pred_xstart {t}"
        carried = np.sqrt(an) * d_x + np.sqrt(1 - an) * (A * d_prev + d_x) / B
        mx, mn = bound(ref_s, f)
        d_s = np.abs(got_s - ref_s)
        print(f"{case} sample {t}: max|d| {d_s.max():.3e} mean|d| {d_s.mean():.3e} (carried: max "
              f"{np.max(carried):.3e}; model bounds {mx:.3e} / {mn:.3e})")
        assert (d_s < carried + mx).all() and d_s.mean() < np.mean(carried) + mn, f"{case} sample {t}"
        d_prev = d_s
        last = (float(np.max(carried)) + mx, float(np.mean(carried)) + mn)
    final = diff.reverse_latent(m, x_start, {"lq": lq}, clip)
    assert torch.equal(G.bits(final), G.bits(rec[-1]["sample"]))
    compare(f"{case} final", final.cpu(), gold[f"{case}/final"], last)     # every position, the last step's bounds


def test_torch_route_learned_range(gold):
    """case e: LEARNED_RANGE on the torch route, on the device (fp32 torch on CUDA against fp32 torch on the CPU: only
    tanh / sin implementations differ)"""
    diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs("e"))
    lq, x_start = (v.cuda() for v in case_inputs("e"))
    out = diff.ddim_reverse_sample_loop(learned_range_model, x_start, clip_denoised=False, model_kwargs={"lq": lq})
    assert out.is_cuda
    ref = gold["e/final"]
    compare("e final", out.cpu(), ref, bounds=(1e-4 * np.abs(ref).max(), 1e-5 * np.abs(ref).max()))


# ------------------------------------------------------------------------------------------------ loop properties

def _inputs(H, W, seed, B=2):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lq = torch.rand(B, 3, H, W, device="cuda", generator=g) * 2 - 1
    x = torch.rand(B, 3, H, W, device="cuda", generator=g) * 2 - 1
    return lq, x, g


def test_graph_replay_equals_eager():
    m, (H, W) = cached_model("unetmodel", "legacy")
    lq, x, _ = _inputs(H, W, 15)
    for kw, clip in ((dict(), True), (dict(predict_xstart=True), False)):
        diff = create_gaussian_diffusion_ddpm(**KW8, **kw)
        r1 = diff.reverse_latent(m, x, {"lq": lq}, clip)
        e = diff.reverse_latent(m, x, {"lq": lq}, clip, use_graph=False)
        r2 = diff.reverse_latent(m, x, {"lq": lq}, clip)
        assert torch.equal(G.bits(r1), G.bits(e)) and torch.equal(G.bits(r2), G.bits(e)), (kw, clip)


def test_image_independent_of_batch():
    m, (H, W) = cached_model("unetconv", "defaults")
    diff = create_gaussian_diffusion_ddpm(**KW8)
    lq, x, g = _inputs(H, W, 16)
    a = diff.reverse_latent(m, x, {"lq": lq}, True)
    lq2, x2 = lq.clone(), x.clone()
    lq2[1] = torch.rand(3, H, W, device="cuda", generator=g)
    x2[1] = torch.rand(3, H, W, device="cuda", generator=g) * 2 - 1
    b = diff.reverse_latent(m, x2, {"lq": lq2}, True)
    assert torch.equal(G.bits(a[0]), G.bits(b[0]))
    assert not torch.equal(a[1], b[1])


def test_reverse_ddpm_and_resshift_samplers_alternate_on_one_plan():
    from resshift_b200.config import DiffusionConfig
    m, (H, W) = cached_model("unetmodel", "legacy")
    rs = create_gaussian_diffusion(**DiffusionConfig(steps=4, min_noise_level=0.2, sf=1).to_kwargs())
    dd = create_gaussian_diffusion_ddpm(**KW8)
    lq, x, g = _inputs(H, W, 18)
    zy = torch.randn(2, 3, H, W, device="cuda", generator=g)
    rn = torch.randn(5, 2, 3, H, W, device="cuda", generator=g)
    dn = torch.randn(9, 2, 3, H, W, device="cuda", generator=g)
    v1 = dd.reverse_latent(m, x, {"lq": lq}, True)
    r1 = rs.sample_latent(zy, m, {"lq": lq}, noises=rn)
    d1 = dd.sample_latent(m, dn, {"lq": lq}, "ddim", True, 0.0)
    v2 = dd.reverse_latent(m, x, {"lq": lq}, True)
    r2 = rs.sample_latent(zy, m, {"lq": lq}, noises=rn)
    d2 = dd.sample_latent(m, dn, {"lq": lq}, "ddim", True, 0.0)
    v3 = dd.reverse_latent(m, x, {"lq": lq}, True, use_graph=False)
    w1 = dd.reverse_latent(m, x, {"lq": lq}, False)
    r3 = rs.sample_latent(zy, m, {"lq": lq}, noises=rn, use_graph=False)
    w2 = dd.reverse_latent(m, x, {"lq": lq}, False, use_graph=False)
    assert torch.equal(G.bits(v1), G.bits(v2)) and torch.equal(G.bits(v1), G.bits(v3))
    assert torch.equal(G.bits(r1), G.bits(r2)) and torch.equal(G.bits(r1), G.bits(r3))
    assert torch.equal(G.bits(d1), G.bits(d2)) and torch.equal(G.bits(w1), G.bits(w2))
    assert not torch.equal(v1, d1) and not torch.equal(r1, v1)


def test_invert_then_ddim_fused_equals_torch_route():
    """x_0 -> x_T by inversion, then x_T -> x_0 by ddim_sample_loop(eta=0): the fused route for both against the torch
    route for both (the same native UNet called step by step through a wrapper the fused gate does not take)"""
    m, (H, W) = cached_model("unetmodel", "legacy")
    diff = create_gaussian_diffusion_ddpm(**KW8)
    lq, x, _ = _inputs(H, W, 19)
    kw = {"lq": lq}
    wrapped = lambda xx, tt, **k: m(xx, tt, **k)                               # noqa: E731
    assert diff._native_ok(m, None, kw) and not diff._native_ok(wrapped, None, kw)
    xt_fused = diff.ddim_reverse_sample_loop(m, x, clip_denoised=False, model_kwargs=kw)
    xt_torch = diff.ddim_reverse_sample_loop(wrapped, x, clip_denoised=False, model_kwargs=kw)
    f = float(np.max(diff.sqrt_recipm1_alphas_cumprod))
    compare("x_T fused vs torch route", xt_fused.cpu(), xt_torch.cpu().double().numpy(),
             bound(xt_torch.cpu().numpy(), f))
    torch.manual_seed(0)
    back_fused = diff.ddim_sample_loop(m, tuple(x.shape), noise=xt_fused, clip_denoised=False, model_kwargs=kw, eta=0.0)
    torch.manual_seed(0)
    back_torch = diff.ddim_sample_loop(wrapped, tuple(x.shape), noise=xt_torch, clip_denoised=False, model_kwargs=kw,
                                       device="cuda", eta=0.0)
    compare("x_0 round trip fused vs torch route", back_fused.cpu(), back_torch.cpu().double().numpy(),
             bound(back_torch.cpu().numpy(), f))
    d = (back_fused - x).abs()
    print(f"round trip vs x_start: max|d| {d.max():.3e} mean|d| {d.mean():.3e}; fused == torch route: "
          f"x_T {torch.equal(xt_fused, xt_torch)}, x_0 {torch.equal(back_fused, back_torch)}")


def test_host_entry_point():
    """rs_sampler_run_host sizes its staging for a sampler that reads no noises, and returns the device run's latent"""
    m, (H, W) = cached_model("unetmodel", "legacy")
    diff = create_gaussian_diffusion_ddpm(**KW8)
    lq, x, _ = _inputs(H, W, 20)
    ref = diff.reverse_latent(m, x, {"lq": lq}, True)
    s = diff.native_sampler(m, 2, H, W, "reverse", True)
    fwd = diff.native_sampler(m, 2, H, W, "ddim", True)
    lat = 2 * 3 * H * W * 4
    nbytes = _lib.lib.rs_sampler_staging_bytes(s)
    assert nbytes < _lib.lib.rs_sampler_staging_bytes(fwd) and nbytes >= 2 * lat
    staging = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    x_h, lq_h = x.cpu().contiguous().numpy(), lq.cpu().contiguous().numpy()
    out_h = np.full(x_h.shape, np.nan, dtype=np.float32)
    fp = lambda a: a.ctypes.data_as(C.c_void_p)                                 # noqa: E731
    for use_graph in (0, 1):
        _lib.check(_lib.lib.rs_sampler_run_host(s, fp(x_h), None, fp(lq_h), None, fp(out_h), staging.data_ptr(), nbytes,
                                                use_graph, G.stream()))
        assert np.array_equal(out_h.view(np.int32), ref.cpu().numpy().view(np.int32)), use_graph
    rc = _lib.lib.rs_sampler_run_host(s, None, None, fp(lq_h), None, fp(out_h), staging.data_ptr(), nbytes, 0, G.stream())
    assert rc != 0 and "x_start (z_y) is NULL" in _lib.lib.rs_last_error().decode()


def test_c_abi_refusals():
    m, (H, W) = cached_model("unetmodel", "legacy")
    plan = m.plan(2, H, W)
    diff = create_gaussian_diffusion_ddpm(**KW8)
    tabs = diff.ddim_reverse_tables()
    tp = tabs.ctypes.data_as(C.POINTER(C.c_double))
    tm = (C.c_int32 * 8)(*diff.timestep_map)

    def refused(match, steps=8, tables=tp, **over):
        o = _lib.DdimReverseOptionsC(1, 0)
        for k, v in over.items():
            setattr(o, k, v)
        h = C.c_void_p()
        rc = _lib.lib.rs_ddim_reverse_sampler_create(plan.handle, steps, tables, tm, C.byref(o), C.byref(h))
        assert rc != 0 and not h.value, over
        assert match in _lib.lib.rs_last_error().decode(), (over, _lib.lib.rs_last_error())

    refused("predict eps or x0", mean_type=_lib.MEAN_TYPES["residual"])
    refused("predict eps or x0", mean_type=_lib.MEAN_TYPES["epsilon_scale"])
    refused("clip must be 0 or 1", clip=2)
    refused("clip must be 0 or 1", clip=-1)
    refused("schedule tables are NULL", tables=None)
    refused("steps must be in [2, 64]", steps=1)
    big = np.ones((9, 65)) * 0.5
    refused("steps must be in [2, 64]", steps=65, tables=big.ctypes.data_as(C.POINTER(C.c_double)))
    h = C.c_void_p()
    rc = _lib.lib.rs_ddim_reverse_sampler_create(plan.handle, 8, tp, tm, None, C.byref(h))
    assert rc != 0 and "options are NULL" in _lib.lib.rs_last_error().decode()
    # a NULL x_start is refused by name; noises may be NULL for this sampler only
    s = diff.native_sampler(m, 2, H, W, "reverse", False)
    buf = torch.zeros(2, 3, H, W, device="cuda")
    lq = torch.zeros(m.lq_shape(2, H, W), device="cuda")
    rc = _lib.lib.rs_sampler_run(s, None, None, lq.data_ptr(), None, buf.data_ptr(), 0, G.stream())
    assert rc != 0 and "x_start (z_y) is NULL" in _lib.lib.rs_last_error().decode()
    assert _lib.lib.rs_sampler_tables(s, (C.c_float * 41)()) != 0
    assert "DDPM sampler" in _lib.lib.rs_last_error().decode()
    d = diff.native_sampler(m, 2, H, W, "ddim", False)
    rc = _lib.lib.rs_sampler_run(d, None, None, lq.data_ptr(), None, buf.data_ptr(), 0, G.stream())
    assert rc != 0 and "null argument" in _lib.lib.rs_last_error().decode()
    # the reference asserts eta == 0 (:1043), before the model runs
    with pytest.raises(AssertionError, match="Reverse ODE only"):
        diff.ddim_reverse_sample(m, buf, torch.zeros(2, dtype=torch.long, device="cuda"), model_kwargs={"lq": lq},
                                 eta=0.5)
