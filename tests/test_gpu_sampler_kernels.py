"""The small kernels of every sampling step and around it, against float64 references of the same operation.

Notation: u = 2^-24 (the unit roundoff of fp32), ulp32(v) the fp32 spacing at |v|.  Each check prints its worst ratio
|d| / bound (1 = at the bound).

Schedule tables (rs_sampler_tables, host).  coef1 = fp32(prev/eta), coef2 = fp32(alpha/eta) and the prior coefficient
fp32(kappa sqrt_eta[T-1]) are single roundings of float64 values: they must be the correctly rounded fp32 numbers, bit
for bit.  std = expf(0.5 fp32(log var)): the rounding of log var moves the exponent by |log var| u / 2 in relative terms
and expf adds under one ulp, so |std - std64| <= (2 + |log var| / 2) u std64.  in_scale = 1 / sqrt(fp32(eta) kappa^2 + 1)
in fp32: the product and the sum put at most 2u on the radicand (u on the root), the root and the reciprocal one
rounding each, the last half an ulp: |in_scale - ref| <= 2u ref + ulp32(ref) / 2, against the float64 value on the same
fp32 eta (at most 2.5 ulp).  The generic path's coefficients (gaussian_diffusion.p_sample) come from the same host
function and must equal the tables bit for bit.

Step (p_sample_kernel, the kernel the sampler's loop runs).  x_next = c1 x + c2 x0 + [t != 0] std noise in fp32 against
float64 tables: table rounding u (|c1 x| + |c2 x0|), three fp32 roundings 3u (|c1 x| + |c2 x0| + |std noise|), and the std
bound above times |noise|.  next_in must be fp16(x_next * in_scale[t-1]) bit for bit, untouched at t = 0 and outside
channels [0, C); the counters zero.  p_sample_flat_kernel (rs_p_sample) on the same fp32 coefficients: identical bits.

Packing (pack_input_kernel, pack_image_kernel).  Pure conversions: bit-identical to torch's .half() of the same fp32
values (x * scale in fp32 first), pad channels +0 exactly, the guard row after the output untouched.

Embedding and FiLM (rs_plan_embedding).  Each stage against float64 of its own fp32 input (the previous stage's
output) with the fp16-rounded weights.  Sinusoid: the fp32 frequency expf(-logf(10000) k / half) carries the rounding of
logf(10000), of the product and of the quotient on an exponent of at most ln 10^4 < 9.3 (3 * 9.3 u) plus expf's 2 ulp
(4u): under 33u relative; t * freq rounds once more (u), so the argument is off by at most 34u t freq, and cosf / sinf
add 2 ulp of the result: bound 34u t freq + 4u |ref|.  Linears (one warp per output: ceil(K/32) fma per lane, five
shuffle sums, the bias): (ceil(K/32) + 6) u (sum |x w| + |b|).  silu_f = __fdividef(v, 1 + __expf(-v)): __expf is within
(2 + 1.16 |v|) ulp, the sum rounds once, __fdividef is within 2 ulp: (9 + 2.32 |v|) u |silu(v)| (+1e-30 where the
quotient flushes); an error e on v reaches the output as at most 1.1 e (|silu'| <= 1.1).  The FiLM bias of a model
without scale-shift norm is emb_layers.1.bias + in_layers bias, also after either is reloaded alone.

Loop (rs_sampler_run with taps).  preds[k+1] is bit for bit a plain forward of samples[k] * in_scale32[t-1] at
tsteps[t-1]; preds[0] a forward of z_y * in_scale32[T-1] when noise 0 is zero (x_T = z_y exactly); every samples[k]
within the step bound of the float64 step on the tapped x_t, x0 and noise; with a random noise 0, samples[0] within the
step bound plus c1 times the prior's (z_y + coef n: coefficient rounding u |coef n| and two roundings 2u (|z_y| + |coef n|)).

First stage.  pointwise_conv_f32_kernel and the moments of kl_posterior_kernel: a chain of Cin fma from the bias,
Cin u (|b| + sum |w x|).  z = mean + fp32(expf(0.5 clamp(logvar, -30, 20)) noise) against float64 of the kernel's own
moments: expf 2 ulp and the product's rounding (5u |std noise|), the sum's rounding (u |z|).  Without noise z is the mean,
bit for bit.  Bicubic (F.interpolate, A = -0.75, half-pixel, border clamp) against the ATen formula in float64: the fp32
source coordinate is within 3u (|s| + 1), which moves the interpolant by at most 4 max|x| per unit (sum |w'| <= 4 for
A = -0.75), and the weight polynomials and eight sums add 16u sum |wx wy x|: bound 16u (sum |wx wy x| + (|sx| + |sy| + 2)
max|x|).  sf = 1 is the identity.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import diffusion_oracle as do
from resshift_b200.weights import random_state_dict

if torch.cuda.is_available():
    from resshift_b200 import _lib
    from tests import gpu_util as G
    from tests.sampler_ref import step_bound, step_ref

U = 2.0 ** -24
COVERED = {"pack": set(), "t": set(), "family": set()}


def _ulp32(v):
    e = torch.floor(torch.log2(v.double().abs().clamp(min=2.0 ** -126)))
    return torch.exp2(e - 23)


def _check(tag, got, ref, bound):
    """|got - ref| <= bound per element (float64); prints the worst ratio.  NaN fails."""
    err = (got.double() - ref).abs()
    ratio = (err / bound.clamp(min=1e-300)).max().item()
    print(f"[bound] {tag}: max |d| / bound = {ratio:.3e}")
    bad = ~(err <= bound)
    assert not bad.any(), f"{tag}: {int(bad.sum())} of {bad.numel()} elements outside the bound (ratio {ratio:.3e})"
    return ratio


def _refused(rc, what):
    assert rc != 0, f"accepted: {what}"
    msg = _lib.lib.rs_last_error().decode()
    assert what in msg, msg


# ------------------------------------------------------------------------------------------------ schedules

def _diffusion(steps, min_noise, kappa=2.0, respacing=None):
    from resshift_b200.models.script_util import create_gaussian_diffusion
    return create_gaussian_diffusion(normalize_input=True, schedule_name="exponential", min_noise_level=min_noise,
                                     steps=steps, kappa=kappa, schedule_kwargs={"power": 0.3},
                                     timestep_respacing=respacing, sf=1)


SCHEDULES = {"realsr_T15": (15, 0.04, 2.0, None), "journal_T4": (4, 0.2, 2.0, None),
             "respaced_1000_to_15": (1000, 0.04, 2.0, 15), "kappa1_T15": (15, 0.04, 1.0, None),
             "respaced_50_to_4": (50, 0.2, 2.0, 4)}


def _tables64(diff):
    return do.schedule_tables(diff.sqrt_etas, diff.kappa)


def _sampler_tables(s, T):
    dst = (C.c_float * (5 * T + 1))()
    _lib.check(_lib.lib.rs_sampler_tables(s, dst))
    a = np.frombuffer(dst, dtype=np.float32).copy()
    return {k: a[j * T:(j + 1) * T] for j, k in enumerate(("coef1", "coef2", "std", "in_scale", "tsteps"))} | \
        {"prior_coef": a[5 * T]}


_TINY = {}


def _tiny_model():
    if "m" not in _TINY:
        from resshift_b200.config import preset
        from resshift_b200.models.unet import UNetModelSwin
        ucfg, _ = preset("tiny")
        m = UNetModelSwin(**ucfg.to_kwargs())
        m.load_state_dict(random_state_dict(ucfg, 0), strict=True)
        _TINY["m"] = m.cuda().eval()
    return _TINY["m"]


@pytest.mark.parametrize("name", list(SCHEDULES))
def test_schedule_tables_vs_float64(name):
    diff = _diffusion(*SCHEDULES[name])
    T = diff.num_timesteps
    s = diff.native_sampler(_tiny_model(), 1, 64, 64)
    tab = _sampler_tables(s, T)
    ref = _tables64(diff)
    for k in ("coef1", "coef2"):
        assert np.array_equal(tab[k].view(np.int32), ref[k].astype(np.float32).view(np.int32)), k
    assert tab["prior_coef"] == np.float32(diff.kappa * diff.sqrt_etas[-1])
    assert np.array_equal(tab["tsteps"], np.asarray(diff.timestep_map, dtype=np.float32))
    if name.startswith("respaced"):
        assert diff.timestep_map != list(range(T))
    std64 = torch.from_numpy(ref["std"])
    _check(f"std {name}", torch.from_numpy(tab["std"]), std64,
           (2 + 0.5 * torch.from_numpy(np.abs(ref["log_var"]))) * U * std64)
    in64 = 1.0 / torch.sqrt(torch.from_numpy(ref["etas"].astype(np.float32)).double() * diff.kappa ** 2 + 1)
    r = _check(f"in_scale {name}", torch.from_numpy(tab["in_scale"]), in64, 2 * U * in64 + 0.5 * _ulp32(in64))
    ulps = ((torch.from_numpy(tab["in_scale"]).double() - in64).abs() / _ulp32(in64)).max().item()
    print(f"[bound] in_scale {name}: worst {ulps:.2f} ulp (bound ratio {r:.3e})")
    # the generic per-step path steps with the same bits
    gen = diff.step_tables()
    for k in ("coef1", "coef2", "std", "in_scale", "tsteps"):
        assert np.array_equal(gen[k].view(np.int32), tab[k].view(np.int32)), k
    assert gen["prior_coef"] == tab["prior_coef"]


# ------------------------------------------------------------------------------------------------ step kernel

def _dev_tables(diff):
    t = diff.step_tables()
    return {k: torch.from_numpy(t[k]).cuda() for k in ("coef1", "coef2", "std", "in_scale")}


def _p_sample_args(x, x0, nz, out, tabs, T, t, N, Cc, HW, next_in=None, cpad=0, counters=None, n_counters=0):
    a = _lib.PSampleArgsC()
    a.x_t, a.x0, a.noise, a.x_next = x.data_ptr(), x0.data_ptr(), nz.data_ptr(), out.data_ptr()
    a.coef1, a.coef2, a.stdv, a.in_scale = (tabs[k].data_ptr() for k in ("coef1", "coef2", "std", "in_scale"))
    a.T, a.t, a.N, a.C, a.HW = T, t, N, Cc, HW
    a.next_in, a.next_cpad = _lib.ptr(next_in), cpad
    a.counters, a.n_counters = _lib.ptr(counters), n_counters
    return a


@pytest.mark.parametrize("N,Cc,H,W", [(2, 3, 64, 64), (1, 4, 37, 5), (3, 3, 7, 9)])
@pytest.mark.parametrize("tcls", ["0", "1", "T-1"])
def test_p_sample_kernel_vs_float64(N, Cc, H, W, tcls):
    diff = _diffusion(*SCHEDULES["realsr_T15"])
    T = diff.num_timesteps
    t = {"0": 0, "1": 1, "T-1": T - 1}[tcls]
    COVERED["t"].add(tcls)
    ref64 = _tables64(diff)
    tabs = _dev_tables(diff)
    HW = H * W
    g = torch.Generator(device="cuda").manual_seed(1000 * t + HW + N)
    x, x0, nz = (torch.randn(N, Cc, H, W, device="cuda", generator=g) * s for s in (2.0, 1.0, 1.0))
    out = torch.full_like(x, float("nan"))
    cpad = Cc + 5
    fill = torch.randn(N * HW + 1, cpad, device="cuda", generator=g).half()   # + one guard row
    nxt = fill.clone()
    ctr = torch.full((300,), -1, dtype=torch.int32, device="cuda")
    a = _p_sample_args(x, x0, nz, out, tabs, T, t, N, Cc, HW, nxt, cpad, ctr, 257)
    _lib.check(_lib.lib.rs_op_p_sample_ex(C.byref(a), G.stream()))
    torch.cuda.synchronize()
    _check(f"p_sample t={t} {N}x{Cc}x{H}x{W}", out, step_ref(x, x0, nz, t, ref64), step_bound(x, x0, nz, t, ref64))
    assert (ctr[:257] == 0).all() and (ctr[257:] == -1).all()
    expect = fill.clone()
    if t > 0:
        s = diff.step_tables()["in_scale"][t - 1]
        q = (out * torch.tensor(s, device="cuda")).half()
        expect[:N * HW, :Cc] = q.permute(0, 2, 3, 1).reshape(N * HW, Cc)
    assert torch.equal(G.bits(nxt), G.bits(expect)), "next_in"
    # the flat kernel of the generic path on the same fp32 coefficients
    flat = torch.full_like(x, float("nan"))
    tt = diff.step_tables()
    _lib.check(_lib.lib.rs_p_sample(x.data_ptr(), x0.data_ptr(), nz.data_ptr(), flat.data_ptr(), float(tt["coef1"][t]),
                                    float(tt["coef2"][t]), float(tt["std"][t]), int(t == 0), x.numel(), G.stream()))
    torch.cuda.synchronize()
    assert torch.equal(G.bits(flat), G.bits(out))


def test_p_sample_refusals():
    diff = _diffusion(*SCHEDULES["journal_T4"])
    tabs = _dev_tables(diff)
    x = torch.zeros(1, 3, 8, 8, device="cuda")
    nxt = torch.zeros(64, 8, dtype=torch.float16, device="cuda")
    for t in (-1, 4):
        a = _p_sample_args(x, x, x, x, tabs, 4, t, 1, 3, 64)
        _refused(_lib.lib.rs_op_p_sample_ex(C.byref(a), G.stream()), "t must be in [0, T = 4)")
    a = _p_sample_args(x, x, x, x, tabs, 4, 2, 1, 3, 64, nxt, 2)
    _refused(_lib.lib.rs_op_p_sample_ex(C.byref(a), G.stream()), "next_cpad must be at least C")
    ctr = torch.zeros(300, dtype=torch.int32, device="cuda")
    a = _p_sample_args(x, x, x, x, tabs, 4, 2, 1, 3, 64, None, 0, ctr, 257)
    _refused(_lib.lib.rs_op_p_sample_ex(C.byref(a), G.stream()), "n_counters must be in [0, 256]")


# ------------------------------------------------------------------------------------------------ packing

PACK_FORMS = ["x_only", "plain", "mask", "unshuffle", "nhwc"]


@pytest.mark.parametrize("form", PACK_FORMS)
@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("wider", [False, True])
@pytest.mark.parametrize("N,H,W", [(2, 8, 16), (3, 7, 9)])
def test_pack_input_bit_identical_to_torch(form, scaled, wider, N, H, W):
    COVERED["pack"].add(form)
    g = torch.Generator(device="cuda").manual_seed(PACK_FORMS.index(form) * 100 + 10 * scaled + 2 * wider + N)
    HW, Cx = H * W, 3
    x = torch.randn(N, Cx, H, W, device="cuda", generator=g) * 3
    scale_tab = torch.rand(5, device="cuda", generator=g) + 0.2
    lq = mask = lq_nhwc = None
    parts = [(x * scale_tab[3]).half() if scaled else x.half()]
    a = _lib.PackInputArgsC()
    if form in ("plain", "mask"):
        Cl = 3
        lq = torch.rand(N, Cl, H, W, device="cuda", generator=g) * 2 - 1
        parts.append(lq.half())
        if form == "mask":
            mask = (torch.rand(N, 1, H, W, device="cuda", generator=g) > 0.5).float() * 0.75 + 0.1
            parts.append(mask.half())
    elif form == "unshuffle":
        Cl = 12
        lq = torch.rand(N, Cl // 4, 2 * H, 2 * W, device="cuda", generator=g) * 2 - 1
        parts.append(F.pixel_unshuffle(lq, 2).half())
        a.lq_unshuffle, a.W = 1, W
    elif form == "nhwc":
        Cl, ld = 20, 24
        lq_nhwc = torch.randn(N * HW, ld, device="cuda", generator=g).half()
        parts.append(lq_nhwc[:, :Cl].reshape(N, H, W, Cl).permute(0, 3, 1, 2))
        a.lq_nhwc, a.lq_ld = lq_nhwc.data_ptr(), ld
    else:
        Cl = 0
    written = sum(p.shape[1] for p in parts)
    Cpad = written + (13 if wider else 0)
    ref = torch.cat([p.permute(0, 2, 3, 1).reshape(N * HW, -1) for p in parts]
                    + [torch.zeros(N * HW, Cpad - written, dtype=torch.float16, device="cuda")], dim=1)
    guard = torch.randn(1, Cpad, device="cuda", generator=g).half()
    out = torch.cat([torch.full((N * HW, Cpad), float("nan"), dtype=torch.float16, device="cuda"), guard])
    ctr = torch.full((N * HW + 40,), -1, dtype=torch.int32, device="cuda")
    nz = min(N * HW, 37)
    a.x, a.Cx = x.data_ptr(), Cx
    if scaled:
        a.scale_tab, a.scale_n, a.scale_idx = scale_tab.data_ptr(), 5, 3
    a.lq_nchw, a.Cl, a.mask_nchw = _lib.ptr(lq), Cl, _lib.ptr(mask)
    a.out, a.Cpad, a.N, a.HW = out.data_ptr(), Cpad, N, HW
    a.counters, a.n_counters = ctr.data_ptr(), nz
    _lib.check(_lib.lib.rs_op_pack_input(C.byref(a), G.stream()))
    torch.cuda.synchronize()
    assert torch.equal(G.bits(out[:N * HW]), G.bits(ref)), form
    assert torch.equal(G.bits(out[N * HW:]), G.bits(guard)), "guard row"
    assert (ctr[:nz] == 0).all() and (ctr[nz:] == -1).all()


@pytest.mark.parametrize("Cb", [0, 1])
@pytest.mark.parametrize("extra", [0, 5])
def test_pack_image_bit_identical_to_torch(Cb, extra):
    g = torch.Generator(device="cuda").manual_seed(17 + Cb + extra)
    N, H, W = 3, 7, 9
    a = torch.randn(N, 3, H, W, device="cuda", generator=g) * 4
    b = torch.rand(N, Cb, H, W, device="cuda", generator=g) if Cb else None
    Cpad = 3 + Cb + extra
    ref = torch.cat([a] + ([b] if Cb else []), dim=1).half().permute(0, 2, 3, 1).reshape(N * H * W, 3 + Cb)
    ref = torch.cat([ref, torch.zeros(N * H * W, extra, dtype=torch.float16, device="cuda")], dim=1)
    out = torch.full((N * H * W + 1, Cpad), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(_lib.lib.rs_op_pack_image(a.data_ptr(), 3, _lib.ptr(b), Cb, out.data_ptr(), Cpad, N, H * W, G.stream()))
    torch.cuda.synchronize()
    assert torch.equal(G.bits(out[:-1]), G.bits(ref))
    assert torch.isnan(out[-1]).all()


def test_pack_refusals():
    x = torch.zeros(1, 3, 4, 4, device="cuda")
    lq = torch.zeros(1, 3, 8, 8, device="cuda")
    out = torch.zeros(16, 32, dtype=torch.float16, device="cuda")
    nh = torch.zeros(16, 8, dtype=torch.float16, device="cuda")

    def args(**kw):
        a = _lib.PackInputArgsC()
        a.x, a.Cx, a.out, a.Cpad, a.N, a.HW = x.data_ptr(), 3, out.data_ptr(), 8, 1, 16
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    cases = [
        (args(lq_nchw=lq.data_ptr(), Cl=3, mask_nchw=x.data_ptr(), Cpad=6), "Cpad must be at least the 7 channels"),
        (args(lq_nchw=lq.data_ptr(), Cl=6, lq_unshuffle=1, W=4), "needs Cl % 4 == 0"),
        (args(lq_nchw=lq.data_ptr(), Cl=12, lq_unshuffle=1, W=4, mask_nchw=x.data_ptr(), Cpad=16), "a mask goes with"),
        (args(lq_nhwc=nh.data_ptr(), Cl=4, lq_ld=8, mask_nchw=x.data_ptr()), "mask_nchw follows lq_nchw"),
        (args(lq_nhwc=nh.data_ptr(), Cl=4, lq_ld=3), "lq_ld must be at least Cl"),
        (args(scale_tab=x.data_ptr(), scale_n=4, scale_idx=4), "scale_idx must be in [0, scale_n = 4)"),
        (args(lq_nchw=lq.data_ptr(), lq_nhwc=nh.data_ptr(), Cl=3, lq_ld=8), "give one"),
    ]
    for a, what in cases:
        _refused(_lib.lib.rs_op_pack_input(C.byref(a), G.stream()), what)
    _refused(_lib.lib.rs_op_pack_image(x.data_ptr(), 3, x.data_ptr(), 1, out.data_ptr(), 3, 1, 16, G.stream()),
             "Cpad must be at least Ca + Cb")


# ------------------------------------------------------------------------------------------------ embedding / FiLM

def _unetmodel(case):
    from oracle.make_golden_unetmodel import case_config
    from resshift_b200.models.unet import UNetModel
    ucfg, dcfg, hw = case_config(case)
    m = UNetModel(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 11), strict=True)
    return ucfg, dcfg, hw, m.cuda().eval()


def _unetconv(case):
    from oracle.make_golden_unetconv import case_config
    from resshift_b200.models.unet import UNetModelConv
    ucfg, dcfg, hw = case_config(case)
    m = UNetModelConv(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 12), strict=True)
    return ucfg, dcfg, hw, m.cuda().eval()


def _swin(name):
    from resshift_b200.config import preset
    from resshift_b200.models.unet import UNetModelSwin
    ucfg, dcfg = preset(name)
    dcfg.sf = 1
    m = UNetModelSwin(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 13), strict=True)
    return ucfg, dcfg, (64, 64), m.cuda().eval()


def _model(family, case):
    return {"swin": _swin, "unetmodel": _unetmodel, "unetconv": _unetconv}[family](case)


def _param_names(m):
    h = m._engine
    buf = C.create_string_buffer(256)
    shape = (C.c_int32 * 4)()
    nd, isb = C.c_int32(), C.c_int32()
    names = []
    for i in range(_lib.lib.rs_unet_param_count(h)):
        _lib.check(_lib.lib.rs_unet_param_info(h, i, buf, 256, shape, C.byref(nd), C.byref(isb)))
        names.append(buf.value.decode())
    return names


def _silu_bound(v):
    """|silu_f(v) - silu(v)| for the fp32 value v (float64 tensor), module docstring."""
    return (9 + 2.32 * v.abs()) * U * (v * torch.sigmoid(v)).abs() + 1e-30


def _linear_check(tag, x, Wt, b, got, silu_in, silu_out):
    """got = act_out(b + W act_in(x)) against float64 on the fp32 input x and fp16-rounded W."""
    xd = x.double()
    K = xd.shape[1]
    w = Wt.half().double()
    xin = F.silu(xd) if silu_in else xd
    pre = xin @ w.t() + b.double()
    mag = xin.abs() @ w.abs().t() + b.double().abs()
    err = (math.ceil(K / 32) + 6) * U * mag
    if silu_in:
        err = err + _silu_bound(xd) @ w.abs().t()
    if silu_out:
        return _check(tag, got, F.silu(pre), 1.1 * err + _silu_bound(pre))
    return _check(tag, got, pre, err)


def _embedding(m, plan, ts, film_rows):
    mc, K = m.cfg.model_channels, 4 * m.cfg.model_channels
    R = ts.numel()
    outs = [torch.full((R, n), float("nan"), device="cuda") for n in (mc, K, K, film_rows)]
    _lib.check(_lib.lib.rs_plan_embedding(plan.handle, ts.data_ptr(), R, *(o.data_ptr() for o in outs), G.stream()))
    torch.cuda.synchronize()
    return outs


EMB_MODELS = [("unetmodel", "legacy", True), ("unetmodel", "new_order", False), ("unetconv", "defaults", False)]


@pytest.mark.parametrize("family,case,ss", EMB_MODELS)
def test_embedding_and_film_vs_float64(family, case, ss):
    ucfg, _, (H, W), m = _model(family, case)
    assert bool(ucfg.use_scale_shift_norm) == ss, f"{family} {case}: scale-shift norm is {ucfg.use_scale_shift_norm}"
    COVERED["family"].add(family)
    plan = m.plan(1, H, W)
    names = _param_names(m)
    P = dict(m.named_parameters())
    emb = [n for n in names if n.endswith(".emb_layers.1.weight")]
    blocks = [n[:-len(".emb_layers.1.weight")] for n in emb]
    in_bias = ".in_layers.1.bias" if family == "unetconv" else ".in_layers.2.bias"
    film_rows = sum(P[n].shape[0] for n in emb)
    ts = torch.tensor([0.0, 1.0, 3.0, 37.0, 500.0, 999.0], device="cuda")
    sin, mid, vec, film = _embedding(m, plan, ts, film_rows)
    # sinusoid
    mc = m.cfg.model_channels
    half = mc // 2
    freq = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float64, device="cuda") / half)
    arg = ts.double()[:, None] * freq[None]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], dim=1)
    _check(f"sinusoid {family} {case}", sin, ref, torch.cat([34 * U * arg] * 2, dim=1) + 4 * U * ref.abs())
    _linear_check(f"time_embed.0 + SiLU {family} {case}", sin, P["time_embed.0.weight"], P["time_embed.0.bias"], mid, 0, 1)
    _linear_check(f"time_embed.2 {family} {case}", mid, P["time_embed.2.weight"], P["time_embed.2.bias"], vec, 0, 0)
    Wf = torch.cat([P[n] for n in emb])

    def fb():
        return torch.cat([P[b + ".emb_layers.1.bias"] + (0 if ss else P[b + in_bias]) for b in blocks])
    _linear_check(f"FiLM {family} {case}", vec, Wf, fb(), film, 1, 0)
    if ss:
        return
    # the fold survives reloading either bias alone (rs_unet_load_param)
    g = torch.Generator(device="cuda").manual_seed(5)
    for which in (in_bias, ".emb_layers.1.bias"):
        with torch.no_grad():
            for b in blocks:
                p = P[b + which]
                p.copy_(torch.randn(p.shape, device="cuda", generator=g) * 3 + 2)
                _lib.check(_lib.lib.rs_unet_load_param(m._engine, (b + which).encode(), p.data_ptr(), G.stream()))
        torch.cuda.synchronize()
        *_, vec2, film2 = _embedding(m, plan, ts, film_rows)
        _linear_check(f"FiLM after reloading {which} {family} {case}", vec2, Wf, fb(), film2, 1, 0)


def test_embedding_refusals():
    m = _tiny_model()
    plan = m.plan(1, 64, 64)
    ts = torch.zeros(80, device="cuda")
    for rows in (0, 65):
        _refused(_lib.lib.rs_plan_embedding(plan.handle, ts.data_ptr(), rows, None, None, None, None, G.stream()),
                 "rows must be in [1, 64]")


# ------------------------------------------------------------------------------------------------ the loop

LOOP_CASES = [("swin", "tiny", None), ("swin", "tiny_inpaint", None), ("swin", "tiny_faceir", None),
              ("unetmodel", "legacy", None), ("unetmodel", "lq2x", None), ("unetconv", "defaults", None),
              ("unetconv", "lq2x", None), ("swin", "tiny", (50, 4))]


def _loop_inputs(m, ucfg, B, H, W, g):
    Cc = ucfg.in_channels if hasattr(ucfg, "swin_depth") else ucfg.out_channels
    zy = torch.randn(B, Cc, H, W, device="cuda", generator=g)
    lq_shape = m.lq_shape(B, H, W)
    lq = torch.rand(*lq_shape, device="cuda", generator=g) * 2 - 1
    mask = None
    if getattr(ucfg, "cond_mask", False):
        mask = (torch.rand(B, 1, *lq_shape[2:], device="cuda", generator=g) > 0.5).float()
    return zy, lq, mask


def _run_loop(diff, m, zy, lq, mask, noises):
    B, Cc, H, W = zy.shape
    T = diff.num_timesteps
    s = diff.native_sampler(m, B, H, W)
    preds = torch.full((T, B, Cc, H, W), float("nan"), device="cuda")
    samples = torch.full_like(preds, float("nan"))
    final = torch.empty_like(zy)
    _lib.check(_lib.lib.rs_sampler_set_taps(s, preds.data_ptr(), samples.data_ptr()))
    try:
        _lib.check(_lib.lib.rs_sampler_run(s, zy.data_ptr(), noises.data_ptr(), lq.data_ptr(), _lib.ptr(mask),
                                           final.data_ptr(), 0, G.stream()))
    finally:
        _lib.check(_lib.lib.rs_sampler_set_taps(s, None, None))
    torch.cuda.synchronize()
    assert torch.equal(G.bits(final), G.bits(samples[-1]))
    return preds, samples


@pytest.mark.parametrize("family,case,respace", LOOP_CASES)
def test_loop_is_forwards_and_steps(family, case, respace):
    ucfg, dcfg, (H, W), m = _model(family, case)
    COVERED["family"].add(family)
    if respace is None:
        diff = _diffusion(dcfg.steps, dcfg.min_noise_level, dcfg.kappa)
    else:
        diff = _diffusion(respace[0], dcfg.min_noise_level, dcfg.kappa, respace[1])
        assert diff.timestep_map != list(range(diff.num_timesteps))
    T, B = diff.num_timesteps, 2
    tt = diff.step_tables()
    ref64 = _tables64(diff)
    g = torch.Generator(device="cuda").manual_seed(4242)
    zy, lq, mask = _loop_inputs(m, ucfg, B, H, W, g)
    noises = torch.randn(T + 1, *zy.shape, device="cuda", generator=g)
    noises[0].zero_()
    preds, samples = _run_loop(diff, m, zy, lq, mask, noises)

    def forward(x, i):
        xin = x * torch.tensor(tt["in_scale"][i], device="cuda")
        ts = torch.full((B,), float(tt["tsteps"][i]), device="cuda")
        return m._run_forward(xin, ts, lq, mask)

    worst = 0.0
    for k in range(T):
        t = T - 1 - k
        x_t = zy if k == 0 else samples[k - 1]
        assert torch.equal(G.bits(preds[k]), G.bits(forward(x_t, t))), f"preds[{k}] is not the forward of its input"
        worst = max(worst, _check(f"loop {family} {case} step k={k}", samples[k], step_ref(x_t, preds[k], noises[k + 1], t, ref64),
                                  step_bound(x_t, preds[k], noises[k + 1], t, ref64)))
    # a random prior noise: samples[0] against the float64 prior followed by the float64 step
    noises[0] = torch.randn(zy.shape, device="cuda", generator=g)
    preds, samples = _run_loop(diff, m, zy, lq, mask, noises)
    pc = diff.kappa * float(diff.sqrt_etas[-1])
    x64 = zy.double() + pc * noises[0].double()
    prior_err = U * (pc * noises[0].double()).abs() + 2 * U * (zy.double().abs() + (pc * noises[0].double()).abs())
    t = T - 1
    bound = step_bound(x64.float(), preds[0], noises[1], t, ref64) + float(ref64["coef1"][t]) * prior_err
    _check(f"loop {family} {case} prior + first step", samples[0], step_ref(x64, preds[0], noises[1], t, ref64), bound)


# ------------------------------------------------------------------------------------------------ first stage

def _fp16_weights(O, I, ld, g, scale=0.5):
    w = torch.randn(O, I, device="cuda", generator=g) * scale
    buf = torch.zeros(O, ld, dtype=torch.float16, device="cuda")
    buf[:, :I] = w.half()
    return buf, buf[:, :I].double()


@pytest.mark.parametrize("Cin,Cout,N,HW", [(3, 3, 2, 256), (8, 8, 1, 256), (8, 8, 2, 999), (5, 7, 1, 300)])
def test_pointwise_conv_vs_float64(Cin, Cout, N, HW):
    g = torch.Generator(device="cuda").manual_seed(Cin * 100 + HW)
    x = torch.randn(N, Cin, HW, device="cuda", generator=g) * 3
    wbuf, w = _fp16_weights(Cout, Cin, 8, g)
    b = torch.randn(Cout, device="cuda", generator=g)
    y = torch.full((N, Cout, HW), float("nan"), device="cuda")
    _lib.check(_lib.lib.rs_op_pointwise_conv(x.data_ptr(), wbuf.data_ptr(), 8, b.data_ptr(), Cin, Cout, N, HW, y.data_ptr(),
                                             G.stream()))
    torch.cuda.synchronize()
    ref = torch.einsum("oc,nch->noh", w, x.double()) + b.double()[None, :, None]
    mag = torch.einsum("oc,nch->noh", w.abs(), x.double().abs()) + b.double().abs()[None, :, None]
    _check(f"pointwise conv Cin={Cin} Cout={Cout} HW={HW}", y, ref, Cin * U * mag)


LOGVARS = [-40.0, -30.0, 20.0, 25.0, float(np.nextafter(np.float32(-30), np.float32(0))),
           float(np.nextafter(np.float32(-30), np.float32(-100))), float(np.nextafter(np.float32(20), np.float32(0))),
           float(np.nextafter(np.float32(20), np.float32(100)))]


def posterior_ref(m64, noise, E):
    mean, lv = m64[:, :E], m64[:, E:].clamp(-30.0, 20.0)
    sn = torch.exp(0.5 * lv) * noise.double()
    return mean + sn, 5 * U * sn.abs() + U * (mean + sn).abs()


@pytest.mark.parametrize("Cin,E,N,HW", [(8, 4, 2, 256), (8, 4, 1, 1024), (16, 8, 2, 333), (16, 4, 1, 257)])
def test_kl_posterior_vs_float64(Cin, E, N, HW):
    g = torch.Generator(device="cuda").manual_seed(Cin * 1000 + E * 10 + HW)
    h = torch.randn(N, Cin, HW, device="cuda", generator=g) * 2
    wbuf, w = _fp16_weights(2 * E, Cin, 16, g, 0.3)
    b = torch.randn(2 * E, device="cuda", generator=g)
    # planted logvars: the rows of these channels have zero weights, so the moment is the bias exactly
    planted = [LOGVARS[(c + (4 if Cin == 16 and E == 4 else 0)) % len(LOGVARS)] for c in range(E)]
    for c in range(E):
        b[E + c] = planted[c]
        wbuf[E + c].zero_()
    w = wbuf[:, :Cin].double()
    noise = torch.randn(N, E, HW, device="cuda", generator=g)
    z = torch.full((N, E, HW), float("nan"), device="cuda")
    mom = torch.full((N, 2 * E, HW), float("nan"), device="cuda")
    _lib.check(_lib.lib.rs_op_kl_posterior(h.data_ptr(), wbuf.data_ptr(), 16, b.data_ptr(), Cin, E, noise.data_ptr(),
                                           z.data_ptr(), mom.data_ptr(), N, HW, G.stream()))
    torch.cuda.synchronize()
    ref = torch.einsum("oc,nch->noh", w, h.double()) + b.double()[None, :, None]
    mag = torch.einsum("oc,nch->noh", w.abs(), h.double().abs()) + b.double().abs()[None, :, None]
    _check(f"kl moments Cin={Cin} E={E} HW={HW}", mom, ref, Cin * U * mag)
    assert torch.equal(mom[:, E:], b[E:][None, :, None].expand(N, E, HW)), "planted logvars"
    zr, bound = posterior_ref(mom.double(), noise, E)
    _check(f"kl z Cin={Cin} E={E} HW={HW} (logvars {planted})", z, zr, bound)
    z0 = torch.full_like(z, float("nan"))
    _lib.check(_lib.lib.rs_op_kl_posterior(h.data_ptr(), wbuf.data_ptr(), 16, b.data_ptr(), Cin, E, None, z0.data_ptr(),
                                           None, N, HW, G.stream()))
    torch.cuda.synchronize()
    assert torch.equal(G.bits(z0), G.bits(mom[:, :E].contiguous())), "mode() is the mean"


def test_kl_encode_in_place_clamps_crafted_logvars():
    from resshift_b200.models.autoencoder import AutoencoderKLTorch
    from resshift_b200.vq_arch import kl_preset, random_kl_state_dict
    cfg = kl_preset("tiny")
    sd = random_kl_state_dict(cfg, 0)
    E = cfg.embed_dim
    sd["quant_conv.bias"] = sd["quant_conv.bias"].clone()
    sd["quant_conv.bias"][E:] = torch.tensor([-45.0, -31.0, 22.0, 30.0])[:E]
    m = AutoencoderKLTorch(**cfg.to_kwargs())
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    g = torch.Generator().manual_seed(3)
    x = (torch.rand(2, 3, 64, 64, generator=g) * 2 - 1).cuda()
    noise = torch.randn(2, E, 16, 16, generator=g)
    z, mom = m.encode(x, return_moments=True, posterior_noise=noise)
    lv = mom[:, E:]
    assert (lv < -30).any() and (lv > 20).any(), "the crafted bias must drive logvar past both clamp limits"
    zr, bound = posterior_ref(mom.double(), noise.cuda(), E)
    _check("kl encode in place (clamped)", z, zr, bound)


def test_first_stage_refusals():
    x = torch.zeros(1, 17, 4, device="cuda")
    w = torch.zeros(32, 32, dtype=torch.float16, device="cuda")
    _refused(_lib.lib.rs_op_pointwise_conv(x.data_ptr(), w.data_ptr(), 32, x.data_ptr(), 9, 3, 1, 4, x.data_ptr(),
                                           G.stream()), "Cin must be at most 8")
    _refused(_lib.lib.rs_op_kl_posterior(x.data_ptr(), w.data_ptr(), 32, x.data_ptr(), 17, 4, None, x.data_ptr(), None, 1, 4,
                                         G.stream()), "Cin must be at most 16")
    _refused(_lib.lib.rs_op_kl_posterior(x.data_ptr(), w.data_ptr(), 32, x.data_ptr(), 8, 9, None, x.data_ptr(), None, 1, 4,
                                         G.stream()), "2E must be at most 16")


def _bicubic64(x, sf):
    """F.interpolate(x, scale_factor=sf, mode='bicubic', align_corners=False) by ATen's formula in float64, plus the
    bound of the module docstring."""
    A = -0.75
    N, Cc, H, W = x.shape
    xd = x.double()

    def axis(n_in):
        o = torch.arange(n_in * sf, dtype=torch.float64, device=x.device)
        s = (o + 0.5) / sf - 0.5
        i0 = torch.floor(s)
        t = s - i0
        c1 = lambda v: ((A + 2) * v - (A + 3)) * v * v + 1
        c2 = lambda v: ((A * v - 5 * A) * v + 8 * A) * v - 4 * A
        w = torch.stack([c2(t + 1), c1(t), c1(1 - t), c2(2 - t)], dim=1)
        idx = (i0.long()[:, None] + torch.arange(-1, 3, device=x.device)[None]).clamp(0, n_in - 1)
        return w, idx, s

    wy, iy, sy = axis(H)
    wx, ix, sx = axis(W)
    patch = xd[:, :, iy][:, :, :, :, ix]                 # [N, C, OH, 4, OW, 4]
    wgt = wy[:, :, None, None] * wx[None, None]          # [OH, 4, OW, 4]
    ref = (patch * wgt).sum(dim=(3, 5))
    mag = (patch.abs() * wgt.abs()).sum(dim=(3, 5))
    mx = patch.abs().amax(dim=(3, 5))
    bound = 16 * U * (mag + (sy.abs()[:, None] + sx.abs()[None] + 2) * mx)
    return ref, bound


@pytest.mark.parametrize("sf", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("H,W", [(1, 6), (6, 1), (2, 3), (5, 7)])
def test_bicubic_vs_float64(sf, H, W):
    g = torch.Generator(device="cuda").manual_seed(sf * 100 + H * 10 + W)
    x = torch.randn(2, 3, H, W, device="cuda", generator=g)
    y = torch.full((2, 3, H * sf, W * sf), float("nan"), device="cuda")
    _lib.check(_lib.lib.rs_op_bicubic_upsample(x.data_ptr(), 2, 3, H, W, sf, y.data_ptr(), G.stream()))
    torch.cuda.synchronize()
    if sf == 1:
        assert torch.equal(G.bits(y), G.bits(x))
    ref, bound = _bicubic64(x, sf)
    _check(f"bicubic sf={sf} {H}x{W}", y, ref, bound)


# ------------------------------------------------------------------------------------------------ coverage

def test_every_form_class_and_family_ran():
    """Runs last in this module: every pack form, step class and model family listed above was exercised."""
    assert COVERED["pack"] == set(PACK_FORMS), COVERED["pack"]
    assert COVERED["t"] == {"0", "1", "T-1"}, COVERED["t"]
    assert COVERED["family"] == {"swin", "unetmodel", "unetconv"}, COVERED["family"]
