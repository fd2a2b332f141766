"""Every op of the plans the tasks run, replayed with synthetic operands through the single-operator entries and held to
float64: the face-restoration (faceir), inpainting and x2 denoisers, the realsr denoiser, the f8_face, f4 and KL f8 first
stages at the sizes the CLI runs them, and every UNetModel / UNetModelConv fixture model (the DDPM, DDIM and DDIM-
inversion samplers' denoisers), random weights.

Convs run with the epilogue their plan row describes (engine.cu collect_profile): per-image bias rows at the plan's row
stride (bsN), the plan's statistics sinks at its cstride / coff, the SiLU second output and FiLM rows per image.  Each
replay is unforced: the entry must report the plan's grid, channel tile, ring depth, CTA pairing, sub-tiles, split-K,
persistence and box; two launches must be bit-identical; the output is held to test_gpu_conv_instances.py's bound on the
rows plan_ops.band_rows() selects (every row of maps up to 256 rows, test_gpu_cli_tile.py's row bands above), and every
sink's (mean, M2) pairs to float64 statistics of the whole stored output (G.check_slot_pairs).  Where a sink's GroupNorm
reduces its pairs with gn_finalize_kernel (gstat bit set: more than 64 tile slots), a third launch passes gstat: the
channels of the consumer's tensor that this conv does not write get the pairs of a synthetic fp16 map, and the group
statistics are held to float64 statistics of the stored output beside that map with test_gpu_cli_tile.py's
count-dependent finalisation bound (gn_ref.check_finalize_gstat).  The SiLU output must lie within one fp16 ulp of SiLU
of the stored output, FiLM within test_gpu_unetconv.py's bound (conv_ref.check_silu_film).  Statistics sinks exist only
on boxes of at most two images (the launcher refuses them beyond), so those rows carry none.

The other ops go through the support modules of their kernels, at the plan's shape: GroupNorm, window and fused Swin
attention and the fused MLP through plan_ops' replays (which test_gpu_cli_tile.py runs too), UNet attention
(attn_ref.unet_case), the VQ-GAN attention (attn_ref.vq_case), the row softmax (first_stage_ref.softmax_case, T rows),
nearest upsample and 2x2 average pool with the SiLU output (plan_ops.replay_resamples, at the plan's batch).  Every op
row of a plan must be claimed by one of these, so an op kind a plan gains later fails test_plan_replay until something
checks it.

test_report prints the worst ratio of error to bound per check, the distinct ops replayed per plan and kind, how many
conv rows were replayed with sinks, gstat, per-image bias, the SiLU output and FiLM (each must be nonzero), the wall time
and the peak torch.cuda.max_memory_allocated.
"""
import time

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from tests import gpu_util as G
    from tests import plan_ops
    from tests.attn_ref import unet_case, vq_case
    from tests.conv_ref import KAPPA, check_silu_film, conv_env, run_conv
    from tests.first_stage_ref import softmax_case
    from tests.gn_ref import boxes, check_finalize_gstat, pairs
    from tests.gpu_util import module_clock  # noqa: F401  (the module's wall-time fixture)

OBS = {}              # check -> worst ratio of error to bound
REPLAYED = {}         # plan -> {op kind: distinct ops replayed}
EPILOGUE = {"sinks": 0, "gstat": 0, "per-image bias": 0, "silu": 0, "film": 0}   # conv rows replayed with each feature


def _note(check, ratio):
    G.note(OBS, check, ratio)


# ---------------------------------------------------------------------------------------------- plans and their op rows

def _plans():
    """plan -> (batch, rows builder)."""
    from oracle.make_golden_unetconv import CASES as CONV_CASES
    from oracle.make_golden_unetmodel import CASES as MODEL_CASES
    plans = {}
    for B in (1, 3):
        plans[f"faceir_denoiser_b{B}_64x64"] = (B, lambda B=B: plan_ops.swin_rows("faceir", B, 64, 64))
        plans[f"inpaint_denoiser_b{B}_64x64"] = (B, lambda B=B: plan_ops.swin_rows("inpaint", B, 64, 64))
    plans["realsr_x2_denoiser_b1_64x64"] = (1, lambda: plan_ops.swin_rows("realsr_x2", 1, 64, 64))
    plans["realsr_denoiser_b16_64x64"] = (16, lambda: plan_ops.swin_rows("realsr", 16, 64, 64))
    plans["realsr_denoiser_b1_512x512"] = (1, lambda: plan_ops.swin_rows("realsr", 1, 512, 512))
    for which, op in ((0, "encode"), (1, "decode")):
        plans[f"vq_f8_face_{op}_512"] = (1, lambda w=which: plan_ops.first_stage_rows("vq", "f8_face", w, 1, 512, 512))
        plans[f"vq_f4_{op}_256"] = (1, lambda w=which: plan_ops.first_stage_rows("vq", "f4", w, 1, 256, 256))
        plans[f"kl_f8_{op}_256"] = (1, lambda w=which: plan_ops.first_stage_rows("kl", "f8", w, 1, 256, 256))
    for name in MODEL_CASES:
        plans[f"unetmodel_{name}_b3"] = (3, lambda n=name: plan_ops.unetmodel_rows(n, *MODEL_CASES[n][1:]))
    for name in CONV_CASES:
        plans[f"unetconv_{name}_b2"] = (2, lambda n=name: plan_ops.unetconv_rows(n))
    return plans


PLAN_NAMES = (["faceir_denoiser_b1_64x64", "faceir_denoiser_b3_64x64", "inpaint_denoiser_b1_64x64",
               "inpaint_denoiser_b3_64x64", "realsr_x2_denoiser_b1_64x64", "realsr_denoiser_b16_64x64",
               "realsr_denoiser_b1_512x512"] +
              [f"{fs}_{op}_{s}" for fs, s in (("vq_f8_face", 512), ("vq_f4", 256), ("kl_f8", 256)) for op in ("encode", "decode")] +
              [f"unetmodel_{n}_b3" for n in ("legacy", "new_order", "lq2x", "nonsquare")] +
              [f"unetconv_{n}_b2" for n in ("defaults", "ss_updown", "lq2x", "uneven")])


# ---------------------------------------------------------------------------------------------- convs, full epilogue

def _pairs_beside(out, d, k):
    """Sink k of conv row d as the consumer sees it: (float64 [N, Ho, Wo, cstride] map whose channels [coff, coff +
    Cout) are the stored output `out` and the rest a synthetic fp16 map, the pair buffer holding that map's (mean, M2)
    pairs outside the conv's slice and NaN inside it)."""
    cs, co = d[f"cs{k}"], d[f"co{k}"]
    N, Ho, Wo, Co = out.shape
    bw, bh, _, slots = G.box128(Ho, Wo)
    full = (torch.randn(N, Ho, Wo, cs, device="cuda", generator=G.gen(900 + cs + co)) * 1.5 + 0.25).half().double()
    full[..., co:co + Co] = out.double()
    p = pairs(boxes(full, bh, bw))
    p[:, :, co:co + Co] = float("nan")
    part = torch.full((N * slots * cs * 2 + 64,), float("nan"), device="cuda")
    part[:N * slots * cs * 2] = p.reshape(-1)
    return full, part, slots


def _check_gstat(tag, L, d, k, out, kw):
    """Third launch with gstat on sink k (module docstring); the consumer's tensor is the map beside the output."""
    full, part, slots = _pairs_beside(out, d, k)
    gs = torch.full((L.N, 32, 2), float("nan"), device="cuda")
    again, _ = L.run(sinks=[(part, d[f"cs{k}"], d[f"co{k}"])], gstat=gs, **kw)
    assert torch.equal(G.bits(again), G.bits(out)), f"{tag}: output with gstat differs"
    e_mu, e_r = check_finalize_gstat(f"{tag} gstat sink {k}", full, 1e-5, gs, slots)
    _note("conv gstat: gn finalize outlier: mean", e_mu)
    _note("conv gstat: gn finalize outlier: rstd", e_r)
    del full, part


def replay_conv(plan, i, d):
    """One conv row d (plan_ops.conv_rows(..., epilogue=True)) with its plan's epilogue (module docstring)."""
    L = plan_ops.conv_of(d, seed=i)
    if d["bsN"]:                        # one bias row per image, bsN apart (the plan's FiLM-table row stride)
        L.bias_sN = d["bsN"]
        L.bbuf = torch.randn(d["N"], d["bsN"], device="cuda", generator=G.gen(500 + i)) * 0.5
        L.brows = L.bbuf[:, :d["Cout"]]
        EPILOGUE["per-image bias"] += 1
    want = {k: d[k] for k in plan_ops.CONV_WANT}
    kw = {"out_f32": bool(d["f32"]), "splitk": d["splitk"] > 1}
    tag = f"{plan} {d}"
    if d["silu"] or d["film"]:
        assert not d["sinks"] and not d["f32"] and d["Ho"] <= 256, tag
        with conv_env():
            got, s, ratio = check_silu_film(tag, L, "image" if d["film"] else "none", 600 + i, want=want,
                                            splitk=kw["splitk"])
        _note("conv silu/film: |d| vs bound", ratio / KAPPA)
        sref = F.silu(got.double())
        _note("conv silu output: |d| / ulp16", ((s.double() - sref).abs() / G.ulp16(sref)).max().item())
        EPILOGUE["silu"] += d["silu"]
        EPILOGUE["film"] += d["film"]
        return
    spec = [(d[f"cs{k}"], d[f"co{k}"]) for k in range(d["sinks"])]
    with conv_env():
        out, _, _, ratio = run_conv(tag, L, want=want, rows=plan_ops.band_rows(d["Ho"]), sink_spec=spec, **kw)
    _note("conv: |d| vs bound", ratio / KAPPA)
    EPILOGUE["sinks"] += d["sinks"] > 0
    for k in range(d["sinks"]):
        if d["gstat"] >> k & 1:
            with conv_env():
                _check_gstat(tag, L, d, k, out, kw)
            EPILOGUE["gstat"] += 1
    del L, out
    G.free()


def _replay_convs(plan, rows, batch):
    convs = plan_ops.conv_rows(rows, epilogue=True)
    for i, d in enumerate(convs):
        replay_conv(plan, i, d)
    return len(convs), {}


# ---------------------------------------------------------------------------------------------- the other op kinds

def _replay_unet_attn(plan, rows, batch):
    ops, obs = plan_ops.distinct(rows, "unet_attn"), {}
    for i, d in enumerate(ops):
        T, heads, D, N = map(int, d[:4])
        for cls in ("randn", "peaked"):
            worst = unet_case(cls, N, T, heads, D, d[4] == "new", seed=i, tag=f"{plan} unet_attn {d} {cls}")[1]
            G.note(obs, "|d| vs bound", worst)
            G.note(obs, f"unet<{D}> {cls}", worst)
        G.free()
    return len(ops), obs


def _replay_vq_attn(plan, rows, batch):
    ops, obs = plan_ops.distinct(rows, "vq_attn"), {}
    for i, d in enumerate(ops):
        T, Cc, N = map(int, d)
        for cls in ("randn", "peaked"):
            worst = vq_case(cls, N, T, Cc, seed=i)
            G.note(obs, "|d| vs bound", worst)
            G.note(obs, f"vq<{Cc}> {cls}", worst)
        G.free()
    return len(ops), obs


def _replay_softmax(plan, rows, batch):
    ops, obs = plan_ops.distinct(rows, "softmax"), {}
    for (cols,) in ops:
        worst, per_class = softmax_case(int(cols), int(cols), int(cols))         # the T x T scores of one image
        G.note(obs, "|d| vs bound", worst)
        for cls, r in per_class.items():
            G.note(obs, f"softmax {cls}", r)
        G.free()
    return len(ops), obs


# kind -> (replay, name of its checks in the report)
KINDS = {"conv": (_replay_convs, None),
         "gn": (lambda plan, rows, batch: plan_ops.replay_gns(plan, rows), "gn"),
         "attn": (lambda plan, rows, batch: plan_ops.replay_windows(plan, rows), None),
         "swin_attn": (lambda plan, rows, batch: plan_ops.replay_swins(plan, rows), None),
         "mlp": (lambda plan, rows, batch: plan_ops.replay_mlps(plan, rows), None),
         "unet_attn": (_replay_unet_attn, "unet attention"), "vq_attn": (_replay_vq_attn, "vq attention"),
         "softmax": (_replay_softmax, "row softmax"),
         "resample": (lambda plan, rows, batch: plan_ops.replay_resamples(rows, batch), None)}


@pytest.mark.parametrize("plan", PLAN_NAMES)
def test_plan_replay(plan):
    batch, fn = _plans()[plan]
    rows = plan_ops.unforced(fn)
    assert rows
    unclaimed = sorted({r for r in rows if not plan_ops.claimed(r)})
    assert not unclaimed, f"{plan}: op rows no check claims: {unclaimed}"
    done = {}
    for kind, (replay, prefix) in KINDS.items():
        if plan_ops.distinct(rows, kind):
            done[kind], obs = replay(plan, rows, batch)
            for k, r in obs.items():
                _note(f"{prefix}: {k}" if prefix else k, r)
            G.free()
    REPLAYED[plan] = done
    print(f"[plan] {plan}: " + ", ".join(f"{n} distinct {k}" for k, n in done.items()))


# ---------------------------------------------------------------------------------------------- report

def test_report(module_clock):
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
    print(f"[task plans] wall time {time.time() - module_clock:.1f} s, peak max_memory_allocated "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB on {props.name}")
    if set(REPLAYED) == set(PLAN_NAMES):
        assert all(EPILOGUE.values()), EPILOGUE
