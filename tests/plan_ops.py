"""The test side of a plan's op profile (rs_plan_profile_ops / rs_vq_profile_ops; engine.cu collect_profile writes one
description row per op): reading the rows, parsing each op kind, building the rows of each model family with random
weights, and replaying the GroupNorm, window attention, fused Swin attention, fused MLP and resample rows through their
single-operator entries against float64.  Each replay returns how many distinct ops it replayed and the worst ratio of
error to bound per check."""
import ctypes as C
import re

import torch

from resshift_b200 import _lib
from tests import gpu_util as G
from tests.attn_ref import SwinCase, WindowCase, run_window
from tests.conv_ref import Conv, conv_env, resample_case
from tests.gn_ref import Case
from tests.mlp_ref import KAPPA as MLP_KAPPA
from tests.mlp_ref import mlp, reference as mlp_reference

# ---------------------------------------------------------------------------------------------- reading and parsing

def read_rows(fn, *args):
    """The op descriptions a profile entry writes; none may have filled its buffer (truncated)."""
    cap, stride = 2048, 256
    ms = (C.c_double * cap)()
    desc = C.create_string_buffer(cap * stride)
    n = C.c_int32()
    _lib.check(fn(*args, ms, desc, stride, cap, C.byref(n), _lib.current_stream()))
    rows = [desc.raw[i * stride:(i + 1) * stride].split(b"\0")[0].decode() for i in range(n.value)]
    assert all(len(r) < stride - 1 for r in rows), "an op description filled its buffer (truncated)"
    return rows


def plan_rows(plan, x, t, lq, mask=None):
    """The op rows of a denoiser plan, run on x, t, lq (and mask)."""
    return read_rows(_lib.lib.rs_plan_profile_ops, plan.handle, x.data_ptr(), t.data_ptr(), lq.data_ptr(),
                     _lib.ptr(mask))


def vq_rows(plan):
    """The op rows of a first-stage plan (rs_vq_profile_ops re-runs them on the inputs the last call left)."""
    return read_rows(_lib.lib.rs_vq_profile_ops, plan.handle)


OPS = {
    "conv": re.compile(r"conv(\d)x\d s(\d) (\d+)x(\d+) Cin=(\d+) Cout=(\d+) grid=(\d+) BN=(\d+) st=(\d+) \S* cg=(\d+) "
                       r"ms=(\d+) sk=(\d+) box=(\d+)x(\d+)x(\d+) N=(\d+) persist=(\d+) pad=(\d+) act=(\d+) res=(\d+) "
                       r"f32=(\d+)(?: silu=(\d) film=(\d) bsN=(\d+) sinks=(\d) cs=(\d+),(\d+) co=(\d+),(\d+) "
                       r"gstat=(\d)$)?"),
    "gn": re.compile(r"gn (\d+)x(\d+) C=(\d+) N=(\d+) route=(\w+) slots=(\d+) eps=(\S+) silu=(\d) film=(\w+)@(-?\d+) "
                     r"apply=(\d+) rows=(\d+) csplit=(\d+) "),
    "attn": re.compile(r"attn (\d+)x(\d+) window=(\d+) shift=(\d+) N=(\d+) heads=(\d+) head_dim=(\d+) hpc=(\d+) "
                       r"simt=(\d)"),
    "swin_attn": re.compile(r"swin_attn (\d+)x(\d+) shift=(\d+) grid=(\d+) N=(\d+) E=(\d+) heads=(\d+) slots=(\d+)"),
    "mlp": re.compile(r"mlp (\d+)x(\d+) E=(\d+) Hd=(\d+) grid=(\d+)"),
    "unet_attn": re.compile(r"unet_attn T=(\d+) heads=(\d+) D=(\d+) N=(\d+) order=(\w+)"),
    "vq_attn": re.compile(r"vq_attn T=(\d+) C=(\d+) N=(\d+)"),
    "softmax": re.compile(r"softmax (\d+)$"),
    "resample": re.compile(r"(upsample|avgpool) (\d+)x(\d+) C=(\d+)(?: silu=1)?$"),
}
_CONV_KEYS = ("k", "s", "Ho", "Wo", "Cin", "Cout", "grid", "BN", "stages", "cg", "msub", "splitk", "bw", "bh", "box_n",
              "N", "persist", "pad", "act", "res", "f32")
_EPI_KEYS = ("silu", "film", "bsN", "sinks", "cs0", "cs1", "co0", "co1", "gstat")
# the launch an unforced replay of a conv row must report
CONV_WANT = ("grid", "BN", "stages", "cg", "msub", "splitk", "persist", "bw", "bh", "box_n")


def claimed(row):
    """Whether some op kind's parser takes the row."""
    return any(rx.match(row) for rx in OPS.values())


def distinct(rows, kind):
    """The distinct field tuples of the rows of one op kind, sorted."""
    return sorted({tuple(OPS[kind].match(r).groups()) for r in rows if OPS[kind].match(r)})


def conv_rows(rows, epilogue=False):
    """Distinct conv launches of an op list, as dicts of the description's fields; with epilogue, also of the fields
    that describe the epilogue (SiLU output, FiLM, per-image bias row stride, statistics sinks, gstat bits)."""
    keys = _CONV_KEYS + _EPI_KEYS
    seen = {}
    for r in rows:
        if r.startswith("conv"):
            m = OPS["conv"].match(r)
            assert m and (m.group(len(keys)) is not None or not epilogue), r
            d = dict(zip(keys, (None if v is None else int(v) for v in m.groups())))
            if not epilogue:
                d = {k: d[k] for k in _CONV_KEYS}
            seen.setdefault(tuple(d.values()), d)
    return list(seen.values())


def gn_rows(rows):
    """Distinct GroupNorms of an op list, as dicts of the description's fields."""
    keys = ("H", "W", "C", "N", "route", "slots", "eps", "silu", "film", "film_off", "apply", "rows", "csplit")
    seen = {}
    for r in rows:
        if r.startswith("gn "):
            m = OPS["gn"].match(r)
            assert m, r
            d = dict(zip(keys, m.groups()))
            for k in keys:
                if k not in ("route", "eps", "film"):
                    d[k] = int(d[k])
            d["eps"] = float(d["eps"])
            seen.setdefault(tuple(d.values()), d)
    return list(seen.values())


def conv_of(d, seed):
    """A random Conv layer of conv row d."""
    return Conv(d["N"], d["Ho"] * d["s"], d["Wo"] * d["s"], d["Cin"], d["Cout"], d["k"], stride=d["s"], pad_lo=d["pad"],
                act=d["act"], res=bool(d["res"]), seed=seed)


def band_rows(H):
    """BAND_ROWS(H) of test_gpu_cli_tile.py's module docstring (None: every row)."""
    if H <= 256:
        return None
    r = {0, 1, H - 2, H - 1}
    for j in range(1, 8):
        r |= {j * H // 8 - 1, j * H // 8}
    s = H // 32
    r |= {j * s + (5 * j) % s for j in range(32)}
    return torch.tensor(sorted(r), device="cuda")


# ---------------------------------------------------------------------------------------------- rows of each model
# family (random weights; the rows depend on the shapes only, not on the input values)

def _loaded(cls, ucfg):
    from resshift_b200.weights import random_state_dict
    m = cls(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 0), strict=True)
    return m.cuda().eval()


def _forward_rows(m, B, H, W, x, lq, mask=None):
    t = torch.arange(B, device="cuda").float() + 2
    m(x, t, lq=lq, **({} if mask is None else {"mask": mask}))
    return plan_rows(m.plan(B, H, W), x, t, lq, mask)


def swin_rows(ucfg, B, H, W):
    """A UNetModelSwin (a task preset's name, or a config) at batch B on an H x W latent, with the LQ and, where the
    model takes one, the mask at the size the feature extractor wants."""
    from resshift_b200.config import preset
    from resshift_b200.models.unet import UNetModelSwin
    if isinstance(ucfg, str):
        ucfg = preset(ucfg)[0]
    m = _loaded(UNetModelSwin, ucfg)
    g = G.gen(1)
    x = torch.randn(B, ucfg.in_channels, H, W, device="cuda", generator=g)
    lq = torch.rand(*m.lq_shape(B, H, W), device="cuda", generator=g) * 2 - 1
    mask = None
    if ucfg.cond_mask:
        mask = (torch.rand(B, 1, *lq.shape[2:], device="cuda", generator=g) < 0.3).float()
    return _forward_rows(m, B, H, W, x, lq, mask)


def unetmodel_rows(name, H, W, B=3):
    """The UNetModel fixture `name` of oracle/make_golden_unetmodel.py."""
    from oracle.make_golden_unetmodel import case_config, case_inputs
    from resshift_b200.models.unet import UNetModel
    ucfg = case_config(name)[0]
    x, lq = (t.cuda() for t in case_inputs(ucfg, B, H, W, 5))
    return _forward_rows(_loaded(UNetModel, ucfg), B, H, W, x, lq)


def unetconv_rows(name, B=2):
    """The UNetModelConv fixture `name` of oracle/make_golden_unetconv.py, at its own size."""
    from oracle.make_golden_unetconv import case_config, case_inputs
    from resshift_b200.models.unet import UNetModelConv
    ucfg, _, (h, w) = case_config(name)
    x, lq = (t.cuda() for t in case_inputs(ucfg, B, h, w, 7))
    return _forward_rows(_loaded(UNetModelConv, ucfg), B, h, w, x, lq)


def first_stage_rows(kind, name, which, batch, h, w):
    """The encode (which 0) or decode (1) plan of a VQ-GAN ("vq") or KL ("kl") first-stage preset on h x w images."""
    from resshift_b200.models.autoencoder import AutoencoderKLTorch, VQModelTorch
    from resshift_b200.vq_arch import kl_preset, random_kl_state_dict, random_vq_state_dict, vq_preset
    cfg = (vq_preset if kind == "vq" else kl_preset)(name)
    sd = (random_vq_state_dict if kind == "vq" else random_kl_state_dict)(cfg, 0)
    m = (VQModelTorch if kind == "vq" else AutoencoderKLTorch)(**cfg.to_kwargs())
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    g = G.gen(2)
    f = 2 ** (len(cfg.ch_mult) - 1)
    if which == 0:
        m.encode(torch.rand(batch, 3, h, w, device="cuda", generator=g) * 2 - 1)
    else:
        z = torch.randn(batch, cfg.embed_dim, h // f, w // f, device="cuda", generator=g) * 0.6
        m.decode(z, force_not_quantize=True) if kind == "vq" else m.decode(z)
    return vq_rows(m.plan(which, batch, h, w))


# the shipped plans several kernel families replay
SHIPPED = {
    "realsr_denoiser_b16_64x64": lambda: swin_rows("realsr", 16, 64, 64),
    "vq_f4_encode_256": lambda: first_stage_rows("vq", "f4", 0, 1, 256, 256),
    "vq_f4_decode_256": lambda: first_stage_rows("vq", "f4", 1, 1, 256, 256),
    "vq_f8_face_decode_512": lambda: first_stage_rows("vq", "f8_face", 1, 1, 512, 512),
    "kl_tiny_encode": lambda: first_stage_rows("kl", "tiny", 0, 2, 64, 96),
    "kl_tiny_decode": lambda: first_stage_rows("kl", "tiny", 1, 2, 64, 96),
}


# ---------------------------------------------------------------------------------------------- replays
# Each runs every distinct op of its kind in a plan's rows unforced at the plan's shape, on the row bands of maps taller
# than 256 rows: the entry must report the plan's configuration and two launches must be bit-identical.

def replay_gns(plan, rows):
    """GroupNorms on the plan's route, slots, eps and SiLU, FiLM rows per image and shared where the plan has FiLM.
    Worst ratios per "route check"."""
    gns, obs = gn_rows(rows), {}
    for i, d in enumerate(gns):
        films = [None] if d["film"] == "none" else ["image", "shared"]
        print(f"[gn route] {plan} {d['H']}x{d['W']} C={d['C']}: route={d['route']} slots={d['slots']} "
              f"K={d['slots'] * d['C'] // 32} items per group")
        for film in films:
            L = Case(d["N"], d["H"], d["W"], d["C"], eps=d["eps"], silu=d["silu"], film=film, seed=i, device="cuda")
            slots = d["slots"] if d["route"].startswith("stats") else None
            out = L.run(d["route"], slots=slots)
            again = L.run(d["route"], slots=slots)
            assert torch.equal(G.bits(out[0]), G.bits(again[0])), f"{plan} {d}: two launches differ"
            if out[2] is not None:
                assert torch.equal(G.bits(out[2]), G.bits(again[2])), f"{plan} {d}: gstat of two launches differ"
            del again
            info = out[1]
            assert (info["slots"], info["apply_ctas"], info["apply_rows"], info["csplit"]) == \
                (d["slots"], d["apply"], d["rows"], d["csplit"]), f"{plan} {d}: launched {info}"
            for k, r in L.check(f"{plan} {d} film={film}", d["route"], out, rows=band_rows(d["H"])).items():
                G.note(obs, f"{d['route']} {k}", r)
            del L, out
            G.free()
    return len(gns), obs


def replay_windows(plan, rows):
    """Window attentions on randn operands; worst ratio as "window attention"."""
    attn, obs = distinct(rows, "attn"), {}
    for i, d in enumerate(attn):
        H, W, ws, shift, N, heads, hd, hpc, simt = map(int, d)
        assert not simt
        L = WindowCase("randn", N, H // ws, W // ws, heads, ws, hd, shift, seed=i)
        out, info, ratio = L.check(f"{plan} attn {d}", hpc=0)
        assert info["hpc"] == hpc, (d, info)
        again, _ = run_window(L.qkv, L.dense, heads, ws, hd, shift, 0, False)
        assert torch.equal(G.bits(out), G.bits(again)), f"{plan} attn {d}: two launches differ"
        G.note(obs, "window attention", ratio)
        del L
        G.free()
    return len(attn), obs


def replay_swins(plan, rows):
    """Fused Swin attention halves on randn operands; worst ratio as "fused Swin attention"."""
    swin, obs = distinct(rows, "swin_attn"), {}
    for i, d in enumerate(swin):
        H, W, shift, grid, N, E, heads, slots = map(int, d)
        L = SwinCase("randn", N, H, W, E, shift, slots, seed=i)
        y, pout, info = L.run(0)
        assert info["grid"] == grid, (d, info)
        y2, pout2, _, ratio = L.check(f"{plan} swin_attn {d}")
        assert torch.equal(G.bits(y), G.bits(y2)) and torch.equal(G.bits(pout), G.bits(pout2)), f"{plan} swin {d}: differ"
        G.note(obs, "fused Swin attention", ratio)
        del L, y, y2
        G.free()
    return len(swin), obs


def replay_mlps(plan, rows, N=1):
    """Fused MLPs at batch N; worst ratio to mlp_ref.KAPPA as "fused MLP"."""
    mlps, obs = distinct(rows, "mlp"), {}
    for i, d in enumerate(mlps):
        H, W, E, Hd, _grid = map(int, d)
        g = G.gen(100 + i)
        x = (torch.randn(N, H, W, E, device="cuda", generator=g) * 1.5 + 0.3).half()
        res = torch.randn(N, H, W, E, device="cuda", generator=g).half()
        w1 = torch.randn(Hd, E, device="cuda", generator=g) / E ** 0.5
        b1 = torch.randn(Hd, device="cuda", generator=g) * 0.5
        w2 = torch.randn(E, Hd, device="cuda", generator=g) / Hd ** 0.5
        b2 = torch.randn(E, device="cuda", generator=g) * 0.5
        w1p, _ = G.pack_weight(w1)
        w2p, _ = G.pack_weight(w2)
        out, _ = mlp(x, res, w1p, b1, w2p, b2, E, Hd)
        out2, _ = mlp(x, res, w1p, b1, w2p, b2, E, Hd)
        assert torch.equal(G.bits(out), G.bits(out2)), f"{plan} mlp {d}: two launches differ"
        sel = band_rows(H)
        xs, rs, os_ = (t if sel is None else t[:, sel] for t in (x, res, out))
        ref, mag, slack = mlp_reference(xs.reshape(-1, E), rs.reshape(-1, E), w1, b1, w2, b2)
        r = G.assert_within(f"{plan} mlp {d}", os_.reshape(-1, E), ref, mag, MLP_KAPPA, slack=slack)
        G.note(obs, "fused MLP", r / MLP_KAPPA)
        G.free()
    return len(mlps), obs


def replay_resamples(rows, N):
    """Nearest upsamples and 2x2 average pools with the SiLU output, at batch N (conv_ref.resample_case)."""
    ops = distinct(rows, "resample")
    for kind, H, W, Cc in ops:
        resample_case(N, int(H), int(W), int(Cc), kind == "avgpool")
        G.free()
    return len(ops), {}


def unforced(fn):
    """The rows of a builder, built with no conv override set."""
    with conv_env():
        rows = fn()
    G.free()
    return rows
