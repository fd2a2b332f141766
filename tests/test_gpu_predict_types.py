"""The fused sampling loop for every predict_type of the reference (xstart, epsilon, epsilon_scale, residual) and every
input scaling (normalize_input, latent_flag).

Step (rs_op_p_sample_pred, the p_sample_kernel instances the loop launches).  x0 is converted in registers op by op in
fp32 with no contraction, on the fp32 tables of rs_schedule_tables_ex: it must be torch.equal to the reference's
expression evaluated the same way in torch fp32 (oracle/predict_types_oracle.predict_xstart) on the same inputs.
x_next is then the xstart step of that x0: within test_gpu_sampler_kernels' float64 step bound, and next_in is
fp16(x_next * in_scale[t - 1]) bit for bit.  Covered at t = 0 and t > 0, with eta_t near 0 (4e-4) and near 1 (0.98).

Loop (rs_sampler_create_ex).  Against the reference's trajectories (tests/golden/loop_predict_types.npz): residual and
the two scalings within the forward bounds of the other loop tests (max 1e-2, mean 2.5e-3).  The epsilon types amplify
the denoiser's fp16 error e: the x0 of step t carries (E_t + a_t e) / (1 - eta_t), with a_t = kappa sqrt_eta_t
(epsilon) or 1 (epsilon_scale) and E_t the error already on x_t, and the step passes it on as
E_{t-1} = coef1 E_t + coef2 (E_t + a_t e) / (1 - eta_t).  For xstart the same recursion (E_{t-1} = coef1 E_t + coef2 e)
never exceeds e, which is how the other loop tests use the forward bounds; here the bounds are the forward bounds times
the gain G of the recursion at e = 1 over the schedule.  Also: every tapped pred_xstart is bit for bit the conversion of
a plain forward of the tapped input, graph replay equals the eager enqueue bit for bit, images are independent of their
batch neighbours, and the multi-GPU modes equal one GPU for an epsilon configuration.
"""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import predict_types_oracle as po
from oracle.make_golden_predict_types import CASES, STRIDE, case_config, trajectory_inputs
from resshift_b200.weights import random_state_dict

if torch.cuda.is_available():
    from resshift_b200 import _lib
    from tests import gpu_util as G
    from tests.sampler_ref import step_bound, step_ref

FWD_MAX, FWD_MEAN = 1e-2, 2.5e-3
KAPPA = 2.0
# sqrt_eta schedules (T = 4) whose etas reach near 0 and near 1: (name, sqrt_etas, the t to test)
SCHEDULES = {"low": ([0.02, 0.04, 0.5, 0.99], (0, 1, 3)), "high": ([0.99, 0.991, 0.993, 0.995], (0, 2))}
STEP_CASES = [(s, t) for s, (_, ts) in SCHEDULES.items() for t in ts]


def _refused(rc, what):
    assert rc != 0, f"accepted: {what}"
    msg = _lib.lib.rs_last_error().decode()
    assert what in msg, msg


def _tables_ex(sqrt_etas, kappa, mean_type, normalize_input=1, latent_flag=1):
    T = len(sqrt_etas)
    opt = _lib.SamplerOptionsC(_lib.MEAN_TYPES[mean_type], normalize_input, latent_flag)
    dst = (C.c_float * (8 * T + 1))()
    _lib.check(_lib.lib.rs_schedule_tables_ex(T, (C.c_double * T)(*sqrt_etas), float(kappa), (C.c_int32 * T)(*range(T)),
                                              C.byref(opt), dst))
    a = np.frombuffer(dst, dtype=np.float32).copy()
    names = ("coef1", "coef2", "std", "in_scale", "tsteps")
    out = {k: a[j * T:(j + 1) * T] for j, k in enumerate(names)}
    out.update({k: a[5 * T + 1 + j * T:5 * T + 1 + (j + 1) * T] for j, k in enumerate(("eps_coef", "eta", "one_minus_eta"))})
    return out


def _tables64(sqrt_etas, kappa):
    from oracle import diffusion_oracle as do
    return do.schedule_tables(np.asarray(sqrt_etas, dtype=np.float64), kappa)


def _pred_args(out, x, y, nz, x_next, dev, T, t, N, Cc, HW, mean_type, next_in=None, cpad=0, x0_out=None):
    a = _lib.PSamplePredArgsC()
    a.out, a.x_t, a.y, a.noise, a.x_next = out.data_ptr(), x.data_ptr(), _lib.ptr(y), nz.data_ptr(), x_next.data_ptr()
    a.coef1, a.coef2, a.stdv, a.in_scale, a.eps_coef, a.eta, a.one_minus_eta = (
        dev[k].data_ptr() for k in ("coef1", "coef2", "std", "in_scale", "eps_coef", "eta", "one_minus_eta"))
    a.T, a.t, a.N, a.C, a.HW, a.mean_type = T, t, N, Cc, HW, _lib.MEAN_TYPES.get(mean_type, mean_type)
    a.next_in, a.next_cpad, a.x0_out = _lib.ptr(next_in), cpad, _lib.ptr(x0_out)
    return a


# ------------------------------------------------------------------------------------------------ step kernel

@pytest.mark.parametrize("sched,t", STEP_CASES)
@pytest.mark.parametrize("mean_type", list(po.MEAN_TYPES))
def test_step_x0_is_the_reference_expression(mean_type, sched, t):
    sqrt_etas = SCHEDULES[sched][0]
    T, N, Cc, H, W = len(sqrt_etas), 2, 3, 37, 9
    HW = H * W
    tabs = _tables_ex(sqrt_etas, KAPPA, mean_type)
    dev = {k: torch.from_numpy(v).cuda() for k, v in tabs.items()}
    g = torch.Generator(device="cuda").manual_seed(77 + 10 * t + len(sched))
    x, out, y, nz = (torch.randn(N, Cc, H, W, device="cuda", generator=g) * s for s in (2.0, 1.0, 0.7, 1.0))
    x_next = torch.full_like(x, float("nan"))
    x0 = torch.full_like(x, float("nan"))
    cpad = Cc + 5
    fill = torch.randn(N * HW + 1, cpad, device="cuda", generator=g).half()   # + one guard row
    nxt = fill.clone()
    a = _pred_args(out, x, y, nz, x_next, dev, T, t, N, Cc, HW, mean_type, nxt, cpad, x0)
    _lib.check(_lib.lib.rs_op_p_sample_pred(C.byref(a), G.stream()))
    torch.cuda.synchronize()
    ref64 = _tables64(sqrt_etas, KAPPA)
    want = po.predict_xstart(mean_type, out.cpu(), x.cpu(), y.cpu(), ref64, t, KAPPA)
    assert torch.equal(G.bits(x0.cpu()), G.bits(want)), f"x0 {mean_type} t={t}: max|d| {(x0.cpu() - want).abs().max()}"
    eta = float(ref64["etas"][t])
    print(f"[step] {mean_type} {sched} t={t} eta={eta:.4g}: x0 bit-identical, max|x0|={want.abs().max().item():.3g}")
    r = step_bound(x, x0, nz, t, ref64)
    err = (x_next.double() - step_ref(x, x0, nz, t, ref64)).abs()
    print(f"[bound] step {mean_type} {sched} t={t}: max |d| / bound = {(err / r.clamp(min=1e-300)).max().item():.3e}")
    assert (err <= r).all()
    expect = fill.clone()
    if t > 0:
        q = (x_next * torch.tensor(tabs["in_scale"][t - 1], device="cuda")).half()
        expect[:N * HW, :Cc] = q.permute(0, 2, 3, 1).reshape(N * HW, Cc)
    assert torch.equal(G.bits(nxt), G.bits(expect)), "next_in"


def test_xstart_pred_step_is_the_shipped_step():
    """rs_op_p_sample_pred with xstart is rs_op_p_sample_ex bit for bit, and its x0 output is the model output."""
    sqrt_etas = SCHEDULES["low"][0]
    T, N, Cc, HW = 4, 2, 3, 64
    tabs = _tables_ex(sqrt_etas, KAPPA, "xstart")
    dev = {k: torch.from_numpy(v).cuda() for k, v in tabs.items()}
    g = torch.Generator(device="cuda").manual_seed(3)
    x, out, nz = (torch.randn(N, Cc, HW, device="cuda", generator=g) for _ in range(3))
    a_out, b_out, x0 = (torch.full_like(x, float("nan")) for _ in range(3))
    a = _pred_args(out, x, None, nz, a_out, dev, T, 2, N, Cc, HW, "xstart", x0_out=x0)
    _lib.check(_lib.lib.rs_op_p_sample_pred(C.byref(a), G.stream()))
    b = _lib.PSampleArgsC()
    b.x_t, b.x0, b.noise, b.x_next = x.data_ptr(), out.data_ptr(), nz.data_ptr(), b_out.data_ptr()
    b.coef1, b.coef2, b.stdv, b.in_scale = (dev[k].data_ptr() for k in ("coef1", "coef2", "std", "in_scale"))
    b.T, b.t, b.N, b.C, b.HW = T, 2, N, Cc, HW
    _lib.check(_lib.lib.rs_op_p_sample_ex(C.byref(b), G.stream()))
    torch.cuda.synchronize()
    assert torch.equal(G.bits(a_out), G.bits(b_out)) and torch.equal(G.bits(x0), G.bits(out))


def test_step_refusals():
    sqrt_etas = SCHEDULES["low"][0]
    dev = {k: torch.from_numpy(v).cuda() for k, v in _tables_ex(sqrt_etas, KAPPA, "epsilon").items()}
    x = torch.zeros(1, 3, 8, 8, device="cuda")
    for mt in (4, -1):
        a = _pred_args(x, x, x, x, x, dev, 4, 1, 1, 3, 64, mt)
        _refused(_lib.lib.rs_op_p_sample_pred(C.byref(a), G.stream()), f"unknown mean type {mt}")
    for mt in ("epsilon", "epsilon_scale", "residual"):
        a = _pred_args(x, x, None, x, x, dev, 4, 1, 1, 3, 64, mt)
        _refused(_lib.lib.rs_op_p_sample_pred(C.byref(a), G.stream()), "reads y (z_y), which is NULL")
    a = _pred_args(x, x, x, x, x, dev, 4, 1, 1, 3, 64, "epsilon")
    a.eps_coef = None
    _refused(_lib.lib.rs_op_p_sample_pred(C.byref(a), G.stream()), "need the eps_coef / eta / one_minus_eta tables")
    for t in (-1, 4):
        a = _pred_args(x, x, x, x, x, dev, 4, t, 1, 3, 64, "residual")
        _refused(_lib.lib.rs_op_p_sample_pred(C.byref(a), G.stream()), "t must be in [0, T = 4)")


def test_sampler_create_ex_refusals():
    m, _ = _model("swin_epsilon")
    plan = m.plan(1, 64, 64)
    se, tm = (C.c_double * 4)(*SCHEDULES["low"][0]), (C.c_int32 * 4)(*range(4))
    h = C.c_void_p()
    for opt, what in (((4, 1, 1), "unknown mean type 4"), ((1, 2, 1), "must be 0 or 1")):
        o = _lib.SamplerOptionsC(*opt)
        _refused(_lib.lib.rs_sampler_create_ex(plan.handle, 4, se, KAPPA, tm, C.byref(o), C.byref(h)), what)
    _refused(_lib.lib.rs_sampler_create_ex(plan.handle, 4, se, KAPPA, tm, None, C.byref(h)), "bad argument")


# ------------------------------------------------------------------------------------------------ the loop

_MODELS = {}


def _model(name):
    ucfg, dcfg, _ = case_config(name)
    family = CASES[name][0]
    if family not in _MODELS:
        from resshift_b200.models.unet import UNetModel, UNetModelSwin
        m = (UNetModelSwin if family == "swin" else UNetModel)(**ucfg.to_kwargs())
        m.load_state_dict(random_state_dict(ucfg, 0), strict=True)
        _MODELS[family] = m.cuda().eval()
    return _MODELS[family], dcfg


def _gain(diff, mean_type):
    """G of the module docstring: the final error of the recursion at a unit denoiser error."""
    E = 0.0
    for t in range(diff.num_timesteps - 1, -1, -1):
        c1, c2 = float(diff.posterior_mean_coef1[t]), float(diff.posterior_mean_coef2[t])
        eta = float(diff.etas[t])
        if mean_type in ("xstart", "residual"):
            E = c1 * E + c2 * 1.0
        else:
            a = diff.kappa * float(diff.sqrt_etas[t]) if mean_type == "epsilon" else 1.0
            E = c1 * E + c2 * (E + a) / (1 - eta)
    return max(E, 1.0)


@pytest.mark.parametrize("name", list(CASES))
def test_loop_vs_reference_trajectory(golden_dir, name):
    from resshift_b200.models.script_util import create_gaussian_diffusion
    g = np.load(golden_dir / "loop_predict_types.npz")
    m, dcfg = _model(name)
    diff = create_gaussian_diffusion(**dcfg.to_kwargs())
    assert diff._native_ok(m, clip_denoised=False, denoised_fn=None, model_kwargs={"lq": None})
    y, noises = (v.cuda() for v in trajectory_inputs(name))
    finals = [diff.sample_latent(y, m, {"lq": y}, noises=noises).clone() for _ in range(2)]   # capture, then replay
    eager = diff.sample_latent(y, m, {"lq": y}, noises=noises, use_graph=False)
    assert torch.equal(finals[0], finals[1]) and torch.equal(finals[0], eager)
    G_ = _gain(diff, dcfg.predict_type)
    bmax, bmean = FWD_MAX * G_, FWD_MEAN * G_
    d = (finals[0].reshape(-1)[::STRIDE].cpu() - torch.from_numpy(g[f"{name}/final_sub"])).abs()
    print(f"[parity] loop {name}: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e} "
          f"(gain {G_:.3f}: bounds {bmax:.3e} / {bmean:.3e})")
    assert not torch.isnan(finals[0]).any()
    assert d.max().item() <= bmax and d.mean().item() <= bmean, name
    # the progressive loop on the fixture's noises: it yields the converted x0 (pred_xstart) of every step
    diff.draw_noises = lambda *a, **k: noises
    rec = list(diff.p_sample_loop_progressive(y, m, first_stage_model=None, noise=noises[0], clip_denoised=False,
                                              model_kwargs={"lq": y}))
    assert torch.equal(rec[-1]["sample"], finals[0])
    for k, r in enumerate(rec):
        dp = (r["pred_xstart"].reshape(-1)[::STRIDE].cpu() - torch.from_numpy(g[f"{name}/pred_xstart/{k}"])).abs()
        print(f"[parity] loop {name} pred_xstart {k}: max|d|={dp.max().item():.3e} mean|d|={dp.mean().item():.3e}")


def _taps(diff, m, zy, lq, noises):
    B, Cc, H, W = zy.shape
    T = diff.num_timesteps
    s = diff.native_sampler(m, B, H, W)
    preds = torch.full((T, B, Cc, H, W), float("nan"), device="cuda")
    samples = torch.full_like(preds, float("nan"))
    final = torch.empty_like(zy)
    _lib.check(_lib.lib.rs_sampler_set_taps(s, preds.data_ptr(), samples.data_ptr()))
    try:
        _lib.check(_lib.lib.rs_sampler_run(s, zy.data_ptr(), noises.data_ptr(), lq.data_ptr(), None, final.data_ptr(), 0,
                                           G.stream()))
    finally:
        _lib.check(_lib.lib.rs_sampler_set_taps(s, None, None))
    torch.cuda.synchronize()
    assert torch.equal(G.bits(final), G.bits(samples[-1]))
    return preds, samples, final


@pytest.mark.parametrize("name", list(CASES))
def test_taps_are_the_converted_forwards(name):
    """pred_xstart[k] is bit for bit the reference conversion of a plain forward of the tapped x_t, scaled by the
    library's in_scale for the configuration; samples[k] is within the step bound of that x0."""
    from resshift_b200.models.script_util import create_gaussian_diffusion
    m, dcfg = _model(name)
    diff = create_gaussian_diffusion(**dcfg.to_kwargs())
    T, mt = diff.num_timesteps, dcfg.predict_type
    tabs = _tables_ex(diff.sqrt_etas.tolist(), diff.kappa, mt, int(dcfg.normalize_input), int(dcfg.latent_flag))
    ref64 = _tables64(diff.sqrt_etas, diff.kappa)
    y, noises = (v.cuda() for v in trajectory_inputs(name))
    preds, samples, _ = _taps(diff, m, y, y, noises)
    # what p_sample_loop_progressive yields is what the taps hold, and its mean follows from the converted x0
    diff.draw_noises = lambda *a, **k: noises
    rec = list(diff.p_sample_loop_progressive(y, m, first_stage_model=None, noise=noises[0], clip_denoised=False,
                                              model_kwargs={"lq": y}))
    c1, c2 = diff.posterior_mean_coef1.astype(np.float32), diff.posterior_mean_coef2.astype(np.float32)
    for k, r in enumerate(rec):
        t = T - 1 - k
        assert torch.equal(r["pred_xstart"], preds[k]) and torch.equal(r["sample"], samples[k]), k
        x_prev = diff.prior_sample(y, noises[0]) if k == 0 else samples[k - 1]
        assert torch.equal(r["mean"], float(c1[t]) * x_prev + float(c2[t]) * preds[k]), k
    for k in range(T):
        t = T - 1 - k
        x_t = diff.prior_sample(y, noises[0]) if k == 0 else samples[k - 1]
        xin = x_t * torch.tensor(tabs["in_scale"][t], device="cuda")
        out = m._run_forward(xin, torch.full((y.shape[0],), float(tabs["tsteps"][t]), device="cuda"), y, None)
        want = po.predict_xstart(mt, out.cpu(), x_t.cpu(), y.cpu(), ref64, t, diff.kappa)
        if k > 0:      # the prior is computed by the kernel, not by torch: its x_t is checked through samples[0]
            assert torch.equal(G.bits(preds[k].cpu()), G.bits(want)), f"{name}: pred_xstart[{k}]"
            r = step_bound(x_t, preds[k], noises[k + 1], t, ref64)
            assert ((samples[k].double() - step_ref(x_t, preds[k], noises[k + 1], t, ref64)).abs() <= r).all(), k


@pytest.mark.parametrize("name", ["swin_epsilon", "swin_residual", "swin_xstart_latent_flag_off"])
def test_images_are_independent_of_their_batch_neighbours(name):
    from resshift_b200.models.script_util import create_gaussian_diffusion
    m, dcfg = _model(name)
    diff = create_gaussian_diffusion(**dcfg.to_kwargs())
    y, noises = (v.cuda() for v in trajectory_inputs(name))
    full = diff.sample_latent(y, m, {"lq": y}, noises=noises)
    y2, n2 = y.clone(), noises.clone()
    y2[1] = torch.rand_like(y[1]) * 2 - 1
    n2[:, 1] = torch.randn_like(noises[:, 1])
    other = diff.sample_latent(y2, m, {"lq": y2}, noises=n2)
    assert torch.equal(other[0], full[0]) and not torch.equal(other[1], full[1])


# ------------------------------------------------------------------------------------------------ the whole pipeline

def _sampler(devices=None):
    from oracle.make_golden_variants import variant_config
    from resshift_b200.sampler import ResShiftSampler, make_configs
    from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
    ucfg, dcfg = variant_config("combined")
    dcfg.sf = 4
    dcfg.predict_type, dcfg.etas_end = "epsilon", 0.5
    vcfg = vq_preset("tiny")
    ae = {"target": "ldm.models.autoencoder.VQModelTorch", "params": vcfg.to_kwargs(), "ckpt_path": random_vq_state_dict(vcfg, 0)}
    configs = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    return ResShiftSampler(configs, sf=4, use_amp=True, seed=123, devices=devices, chop_size=64, chop_stride=48,
                           padding_offset=64)


def test_epsilon_virtual_ranks_and_pool_equal_one_gpu(tmp_path):
    import cv2
    from resshift_b200.parallel import unit_schedule
    from resshift_b200.sampler import tile_counts
    s = _sampler()
    assert s.base_diffusion.model_mean_type.name == "EPSILON"
    assert s.base_diffusion._native_ok(s.model, clip_denoised=False, denoised_fn=None, model_kwargs={"lq": None})
    gen = torch.Generator(device="cuda").manual_seed(8)
    lqs = [torch.rand(b, 3, h, w, device="cuda", generator=gen) * 2 - 1 for b, h, w in [(2, 200, 148), (1, 60, 50)]]
    s.setup_seed()
    ref = [s._sample_tiled(lq, mask=None, noise_repeat=False) for lq in lqs]
    units = s._plan_units([tuple(lq.shape[2:]) for lq in lqs])
    for world in (1, 2, 5):
        schedule = unit_schedule(len(units), world, teams=False)
        shares = []
        for rank in range(world):
            s.setup_seed()
            shares.append(s._run_rank(lqs, [None, None], False, units, schedule, rank))
        counts = tile_counts(units, schedule, world)
        for gi, (lq, r) in enumerate(zip(lqs, ref)):
            assert [sh[gi].shape[0] for sh in shares] == counts[gi]
            assert torch.equal(s._assemble(torch.cat([sh[gi] for sh in shares]), *lq.shape[2:]), r), (world, gi)

    rng = np.random.default_rng(7)
    (tmp_path / "in").mkdir()
    for name, (h, w) in {"a1": (200, 148), "a2": (200, 148), "b": (60, 50)}.items():
        cv2.imwrite(str(tmp_path / "in" / f"{name}.png"), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
    outs = []
    for smp, d in ((s, "ref"), (_sampler("0,0"), "pool")):
        smp.setup_seed()
        smp.inference(tmp_path / "in", tmp_path / d, bs=3)
        outs.append({p.name: p.read_bytes() for p in sorted((tmp_path / d).iterdir())})
    assert len(outs[0]) == 3 and outs[0] == outs[1]
