"""Every op of the plans the tasks run, replayed with synthetic operands through the single-operator entries and held to
float64: the face-restoration (faceir), inpainting and x2 denoisers, the realsr denoiser, the f8_face, f4 and KL f8 first
stages at the sizes the CLI runs them, and every UNetModel / UNetModelConv fixture model (the DDPM, DDIM and DDIM-
inversion samplers' denoisers), random weights.

Convs run with the epilogue their plan row describes (engine.cu collect_profile): per-image bias rows at the plan's row
stride (bsN), the plan's statistics sinks at its cstride / coff, the SiLU second output and FiLM rows per image.  Each
replay is unforced: the entry must report the plan's grid, channel tile, ring depth, CTA pairing, sub-tiles, split-K,
persistence and box; two launches must be bit-identical; the output is held to test_gpu_conv_instances.py's bound on
the rows band_rows() selects (every row of maps up to 256 rows, test_gpu_cli_tile.py's row bands above), and every
sink's (mean, M2) pairs to float64 statistics of the whole stored output (G.check_slot_pairs).  Where a sink's GroupNorm
reduces its pairs with gn_finalize_kernel (gstat bit set: more than 64 tile slots), a third launch passes gstat: the
channels of the consumer's tensor that this conv does not write get the pairs of a synthetic fp16 map, and the group
statistics are held to float64 statistics of the stored output beside that map with test_gpu_cli_tile.py's
count-dependent finalisation bound.  The SiLU output must lie within one fp16 ulp of SiLU of the stored output, FiLM
within test_gpu_unetconv.py's bound (test_gpu_unetconv._check).  Statistics sinks exist only on boxes of at most two
images (the launcher refuses them beyond), so those rows carry none.

The other ops go through the helpers of the modules that own their kernels, at the plan's shape: GroupNorm (Case, on the
plan's route and slots), window and fused Swin attention, the fused MLP, UNet attention (unet_case), the VQ-GAN
attention (vq_case), the row softmax (softmax_case, T rows), nearest upsample and 2x2 average pool with the SiLU output
(resample_case, at the plan's batch).  Every op row of a plan must be claimed by one of these, so an op kind a plan gains
later fails test_plan_replay until something checks it.

test_report prints the worst ratio of error to bound per check, the distinct ops replayed per plan and kind, how many
conv rows were replayed with sinks, gstat, per-image bias, the SiLU output and FiLM (each must be nonzero), the wall time
and the peak torch.cuda.max_memory_allocated.
"""
import gc
import re
import time
from contextlib import contextmanager

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from tests import gpu_util as G
    from resshift_b200 import _lib
    from tests import test_gpu_attention as TA
    from tests import test_gpu_cli_tile as CT
    from tests import test_gpu_first_stage_kernels as FS
    from tests import test_gpu_groupnorm as GN
    from tests.test_gpu_cli_tile import band_rows, check_finalize_gstat
    from tests.test_gpu_conv_instances import Conv, _box, _conv_rows, _desc_rows, _first_stage_rows, _run, conv_env
    from tests.test_gpu_unetconv import _check as silu_film_check
    from tests.test_gpu_unetconv import resample_case

OBS = {}              # check -> worst ratio of error to bound
REPLAYED = {}         # plan -> {op kind: distinct ops replayed}
EPILOGUE = {"sinks": 0, "gstat": 0, "per-image bias": 0, "silu": 0, "film": 0}   # conv rows replayed with each feature
_T0 = []

_SOFTMAX = re.compile(r"softmax (\d+)$")
_RESAMPLE = re.compile(r"(upsample|avgpool) (\d+)x(\d+) C=(\d+)(?: silu=1)?$")


def _note(check, ratio):
    OBS[check] = max(OBS.get(check, 0.0), float(ratio))


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _free():
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _clock():
    torch.cuda.reset_peak_memory_stats()
    _T0.append(time.time())
    yield


@contextmanager
def _observed(prefix, *modules):
    """The worst ratios the helpers of `modules` record (their module-level OBS) and every G.assert_within bound met
    meanwhile, gathered into this module's OBS under `prefix`."""
    saved = [m.OBS for m in modules]
    for m in modules:
        m.OBS = {}
    within = G.assert_within

    def assert_within(tag, got, ref, mag, kappa, *a, **kw):
        r = within(tag, got, ref, mag, kappa, *a, **kw)
        _note(f"{prefix}: |d| vs bound", r / kappa)
        return r
    G.assert_within = assert_within
    try:
        yield
    finally:
        G.assert_within = within
        for m, s in zip(modules, saved):
            for k, v in m.OBS.items():          # {check: ratio}, {(kernel, class): ratio} or {route: {check: ratio}}
                name = " ".join(map(str, k)) if isinstance(k, tuple) else str(k)
                for sub, r in (v.items() if isinstance(v, dict) else [("", v)]):
                    _note(f"{prefix}: {name} {sub}".rstrip(), r)
            m.OBS = s


# ---------------------------------------------------------------------------------------------- plans and their op rows

def _swin_rows(name, B, H, W):
    """A UNetModelSwin task denoiser at batch B on an H x W latent (LQ, and the mask where the task takes one, at the
    size the feature extractor wants)."""
    from resshift_b200.config import preset
    from resshift_b200.models.unet import UNetModelSwin
    from resshift_b200.weights import random_state_dict
    ucfg, _ = preset(name)
    m = UNetModelSwin(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 0))
    m = m.cuda().eval()
    g = _gen(1)
    x = torch.randn(B, ucfg.in_channels, H, W, device="cuda", generator=g)
    lq = torch.rand(*m.lq_shape(B, H, W), device="cuda", generator=g) * 2 - 1
    mask = None
    if ucfg.cond_mask:
        mask = (torch.rand(B, 1, *lq.shape[2:], device="cuda", generator=g) < 0.3).float()
    t = torch.arange(B, device="cuda").float() + 2
    m(x, t, lq=lq, mask=mask)
    return _desc_rows(_lib.lib.rs_plan_profile_ops, m.plan(B, H, W).handle, x.data_ptr(), t.data_ptr(), lq.data_ptr(),
                      _lib.ptr(mask))


def _unetconv_rows(name, B=2):
    from oracle.make_golden_unetconv import case_config, case_inputs
    from resshift_b200.models.unet import UNetModelConv
    from resshift_b200.weights import random_state_dict
    ucfg, _, (h, w) = case_config(name)
    m = UNetModelConv(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 0), strict=True)
    m = m.cuda().eval()
    x, lq = (t.cuda() for t in case_inputs(ucfg, B, h, w, 7))
    t = torch.arange(B, device="cuda").float() + 1
    m(x, t, lq=lq)
    return _desc_rows(_lib.lib.rs_plan_profile_ops, m.plan(B, h, w).handle, x.data_ptr(), t.data_ptr(), lq.data_ptr(), None)


def _plans():
    """plan -> (batch, rows builder)."""
    from oracle.make_golden_unetconv import CASES as CONV_CASES
    from oracle.make_golden_unetmodel import CASES as MODEL_CASES
    plans = {}
    for B in (1, 3):
        plans[f"faceir_denoiser_b{B}_64x64"] = (B, lambda B=B: _swin_rows("faceir", B, 64, 64))
        plans[f"inpaint_denoiser_b{B}_64x64"] = (B, lambda B=B: _swin_rows("inpaint", B, 64, 64))
    plans["realsr_x2_denoiser_b1_64x64"] = (1, lambda: _swin_rows("realsr_x2", 1, 64, 64))
    plans["realsr_denoiser_b16_64x64"] = (16, lambda: _swin_rows("realsr", 16, 64, 64))
    plans["realsr_denoiser_b1_512x512"] = (1, lambda: _swin_rows("realsr", 1, 512, 512))
    for which, op in ((0, "encode"), (1, "decode")):
        plans[f"vq_f8_face_{op}_512"] = (1, lambda w=which: _first_stage_rows("vq", "f8_face", w, 1, 512, 512))
        plans[f"vq_f4_{op}_256"] = (1, lambda w=which: _first_stage_rows("vq", "f4", w, 1, 256, 256))
        plans[f"kl_f8_{op}_256"] = (1, lambda w=which: _first_stage_rows("kl", "f8", w, 1, 256, 256))
    for name in MODEL_CASES:
        plans[f"unetmodel_{name}_b3"] = (3, lambda n=name: TA._unetmodel_rows(n, *MODEL_CASES[n][1:]))
    for name in CONV_CASES:
        plans[f"unetconv_{name}_b2"] = (2, lambda n=name: _unetconv_rows(n))
    return plans


PLAN_NAMES = (["faceir_denoiser_b1_64x64", "faceir_denoiser_b3_64x64", "inpaint_denoiser_b1_64x64",
               "inpaint_denoiser_b3_64x64", "realsr_x2_denoiser_b1_64x64", "realsr_denoiser_b16_64x64",
               "realsr_denoiser_b1_512x512"] +
              [f"{fs}_{op}_{s}" for fs, s in (("vq_f8_face", 512), ("vq_f4", 256), ("kl_f8", 256)) for op in ("encode", "decode")] +
              [f"unetmodel_{n}_b3" for n in ("legacy", "new_order", "lq2x", "nonsquare")] +
              [f"unetconv_{n}_b2" for n in ("defaults", "ss_updown", "lq2x", "uneven")])


def plan_rows(plan):
    batch, fn = _plans()[plan]
    with conv_env():
        rows = fn()
    _free()
    return batch, rows


# ---------------------------------------------------------------------------------------------- convs, full epilogue

def _pairs_beside(out, d, k):
    """Sink k of conv row d as the consumer sees it: (float64 [N, Ho, Wo, cstride] map whose channels [coff, coff +
    Cout) are the stored output `out` and the rest a synthetic fp16 map, the pair buffer holding that map's (mean, M2)
    pairs outside the conv's slice and NaN inside it)."""
    cs, co = d[f"cs{k}"], d[f"co{k}"]
    N, Ho, Wo, Co = out.shape
    bw, bh, _, slots = _box(Ho, Wo)
    full = (torch.randn(N, Ho, Wo, cs, device="cuda", generator=_gen(900 + cs + co)) * 1.5 + 0.25).half().double()
    full[..., co:co + Co] = out.double()
    pairs = GN._pairs(GN._boxes(full, bh, bw))
    pairs[:, :, co:co + Co] = float("nan")
    part = torch.full((N * slots * cs * 2 + 64,), float("nan"), device="cuda")
    part[:N * slots * cs * 2] = pairs.reshape(-1)
    return full, part, slots


def _check_gstat(tag, L, d, k, out, kw):
    """Third launch with gstat on sink k (module docstring)."""
    full, part, slots = _pairs_beside(out, d, k)
    gs = torch.full((L.N, 32, 2), float("nan"), device="cuda")
    again, _ = L.run(sinks=[(part, d[f"cs{k}"], d[f"co{k}"])], gstat=gs, **kw)
    assert torch.equal(G.bits(again), G.bits(out)), f"{tag}: output with gstat differs"
    S = GN.Case.__new__(GN.Case)        # the statistics side of a GroupNorm case: its input is the consumer's tensor
    S.N, S.H, S.W, S.C, S.eps, S.x64, S._stats = L.N, L.Ho, L.Wo, d[f"cs{k}"], 1e-5, full, None
    with _observed("conv gstat", CT):
        check_finalize_gstat(f"{tag} gstat sink {k}", S, gs, slots)
    del full, part, S


def replay_conv(plan, i, d):
    """One conv row d (_conv_rows(..., epilogue=True)) with its plan's epilogue (module docstring)."""
    L = Conv(d["N"], d["Ho"] * d["s"], d["Wo"] * d["s"], d["Cin"], d["Cout"], d["k"], stride=d["s"], pad_lo=d["pad"],
             act=d["act"], res=bool(d["res"]), seed=i)
    if d["bsN"]:                        # one bias row per image, bsN apart (the plan's FiLM-table row stride)
        L.bias_sN = d["bsN"]
        L.bbuf = torch.randn(d["N"], d["bsN"], device="cuda", generator=_gen(500 + i)) * 0.5
        L.brows = L.bbuf[:, :d["Cout"]]
        EPILOGUE["per-image bias"] += 1
    want = {k: d[k] for k in ("grid", "BN", "stages", "cg", "msub", "splitk", "persist", "bw", "bh", "box_n")}
    kw = {"out_f32": bool(d["f32"]), "splitk": d["splitk"] > 1}
    tag = f"{plan} {d}"
    if d["silu"] or d["film"]:
        assert not d["sinks"] and not d["f32"] and d["Ho"] <= 256, tag
        with conv_env(), _observed("conv silu/film"):
            got, s = silu_film_check(tag, L, "image" if d["film"] else "none", 600 + i, want=want, splitk=kw["splitk"])
        sref = F.silu(got.double())
        _note("conv silu output: |d| / ulp16", ((s.double() - sref).abs() / G.ulp16(sref)).max().item())
        EPILOGUE["silu"] += d["silu"]
        EPILOGUE["film"] += d["film"]
        return
    spec = [(d[f"cs{k}"], d[f"co{k}"]) for k in range(d["sinks"])]
    with conv_env(), _observed("conv"):
        out, _, _ = _run(tag, L, want=want, rows=band_rows(d["Ho"]), sink_spec=spec, **kw)
    EPILOGUE["sinks"] += d["sinks"] > 0
    for k in range(d["sinks"]):
        if d["gstat"] >> k & 1:
            with conv_env():
                _check_gstat(tag, L, d, k, out, kw)
            EPILOGUE["gstat"] += 1
    del L, out
    _free()


def _replay_convs(plan, rows, batch):
    convs = _conv_rows(rows, epilogue=True)
    for i, d in enumerate(convs):
        replay_conv(plan, i, d)
    return len(convs)


# ---------------------------------------------------------------------------------------------- the other op kinds

def _replay_gns(plan, rows, batch):
    with _observed("gn", GN):
        return CT._replay_gns(plan, rows)


def _replay_windows(plan, rows, batch):
    with _observed("window attention", CT):
        return CT._replay_windows(plan, rows)


def _replay_swins(plan, rows, batch):
    with _observed("fused Swin attention", CT):
        return CT._replay_swins(plan, rows)


def _replay_mlps(plan, rows, batch):
    with _observed("fused MLP", CT):
        return CT._replay_mlps(plan, rows)


def _replay_unet_attn(plan, rows, batch):
    ops = CT._distinct(rows, TA._UNET)
    with _observed("unet attention", TA):
        for i, d in enumerate(ops):
            T, heads, D, N = map(int, d[:4])
            for cls in ("randn", "peaked"):
                TA.unet_case(cls, N, T, heads, D, d[4] == "new", seed=i, tag=f"{plan} unet_attn {d} {cls}")
            _free()
    return len(ops)


def _replay_vq_attn(plan, rows, batch):
    ops = CT._distinct(rows, TA._VQ)
    with _observed("vq attention", TA):
        for i, d in enumerate(ops):
            T, Cc, N = map(int, d)
            for cls in ("randn", "peaked"):
                TA.vq_case(cls, N, T, Cc, seed=i)
            _free()
    return len(ops)


def _replay_softmax(plan, rows, batch):
    ops = CT._distinct(rows, _SOFTMAX)
    with _observed("row softmax", FS):
        for (cols,) in ops:
            FS.softmax_case(int(cols), int(cols), int(cols))         # the T x T scores of one image
            _free()
    return len(ops)


def _replay_resample(plan, rows, batch):
    ops = CT._distinct(rows, _RESAMPLE)
    for kind, H, W, Cc in ops:
        resample_case(batch, int(H), int(W), int(Cc), kind == "avgpool")
        _free()
    return len(ops)


KINDS = {"conv": (_replay_convs, re.compile(r"conv")), "gn": (_replay_gns, re.compile(r"gn ")),
         "attn": (_replay_windows, re.compile(r"attn ")), "swin_attn": (_replay_swins, re.compile(r"swin_attn ")),
         "mlp": (_replay_mlps, re.compile(r"mlp ")), "unet_attn": (_replay_unet_attn, re.compile(r"unet_attn ")),
         "vq_attn": (_replay_vq_attn, re.compile(r"vq_attn ")), "softmax": (_replay_softmax, _SOFTMAX),
         "resample": (_replay_resample, _RESAMPLE)}


def _claims(r):
    """The op-row parsers of the replays that claim row r."""
    from tests.test_gpu_conv_instances import _DESC
    return [rx for rx in (_DESC, GN._GN, TA._ATTN, TA._SWIN, CT._MLP, TA._UNET, TA._VQ, _SOFTMAX, _RESAMPLE) if rx.match(r)]


@pytest.mark.parametrize("plan", PLAN_NAMES)
def test_plan_replay(plan):
    batch, rows = plan_rows(plan)
    assert rows
    assert all(len(r) < 255 for r in rows), "an op description filled its buffer (truncated)"
    unclaimed = sorted({r for r in rows if not _claims(r)})
    assert not unclaimed, f"{plan}: op rows no check claims: {unclaimed}"
    done = {}
    for kind, (fn, rx) in KINDS.items():
        if any(rx.match(r) for r in rows):
            done[kind] = fn(plan, rows, batch)
            _free()
    REPLAYED[plan] = done
    print(f"[plan] {plan}: " + ", ".join(f"{n} distinct {k}" for k, n in done.items()))


# ---------------------------------------------------------------------------------------------- report

def test_report():
    """Run with the rest of the module: worst ratio of error to bound per check, ops per plan, the conv rows replayed
    with each epilogue feature (each must be nonzero), wall time, memory."""
    if not REPLAYED:
        pytest.skip("run with the rest of the module")
    for k, r in sorted(OBS.items()):
        print(f"[observed] {k}: worst ratio {r:.3g}")
    for plan, d in REPLAYED.items():
        print(f"[replayed] {plan}: " + ", ".join(f"{n} {k}" for k, n in d.items()))
    print("[conv epilogue] rows replayed with " + ", ".join(f"{k}: {n}" for k, n in EPILOGUE.items()))
    props = torch.cuda.get_device_properties(0)
    print(f"[task plans] wall time {time.time() - _T0[0]:.1f} s, peak max_memory_allocated "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB on {props.name}")
    if set(REPLAYED) == set(PLAN_NAMES):
        assert all(EPILOGUE.values()), EPILOGUE
