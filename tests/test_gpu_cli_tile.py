"""The default CLI tile: one 512x512 LQ tile at x4 (inference_resshift.py --chop_size 512), i.e. a bicubic x4 to
2048x2048, an f4 VQ-GAN encode at 2048x2048 (bottleneck attention over T = 262144 positions at C = 512), the realsr
denoiser on a 512x512 latent at batch 1, an f4 decode back to 2048x2048 and the overlap-average of such tiles, held to
float64 references and to the fp32 oracle at that size.  The smaller sizes are held by test_gpu_conv_instances.py,
test_gpu_groupnorm.py, test_gpu_attention.py, test_gpu_mlp_instances.py and test_gpu_vq_attention.py, whose references
this one runs from the support modules (conv_ref, gn_ref, attn_ref, mlp_ref, plan_ops); their bounds apply unchanged.

Row bands.  Where a float64 reference of a whole 2048x2048 map costs too much (convs, GroupNorm applies, the fused MLP),
it is computed on the output rows BAND_ROWS(H) of every image of an H-row map, H > 256:
    rows 0, 1, H - 2, H - 1;
    rows j H/8 - 1 and j H/8 for j = 1 .. 7 (both sides of those boundaries between 128-pixel conv boxes: at W = 2048 a
    box is 128x1, 16 per row, so row H/2 = 1024 is where tile index 16384 starts);
    rows j H/32 + (5 j mod H/32) for j = 0 .. 31 (an even spread at shifting offsets).
Maps of at most 256 rows are checked on every row.  Convs and GroupNorm applies are local, so banding loses only the
rows it skips; GroupNorm statistics are always checked in full.

Attention rows.  T = 262144 is 4096 query tiles of 64 rows.  ATTN_ROWS checks one row of every tile (row 64 t +
(37 t mod 64)) and all 64 rows of tile 0, tile 4095 and the tiles 132 j - 1 and 132 j (j = 1 .. 31) on both sides of
each 132-CTA wave boundary: 8128 rows.  The float64 reference of all 262144 rows was not run, to keep the file's time.

a. Plan replays (vq_f4_encode_2048, vq_f4_decode_2048, realsr_denoiser_b1_512x512, random weights): every distinct conv,
   GroupNorm, window attention, fused Swin attention and fused MLP through its _ex entry point, unforced: the entry
   reports the plan's configuration, two launches are bit-identical, every checked element is within its module's
   float64 bound; the decoder's nearest upsamples through rs_op_upsample2x_ex with the SiLU output
   (conv_ref.resample_case).  Every op row of each plan is claimed by a replay here or by b (vq_attn), so an
   op kind a plan gains later fails test_plan_replay until something checks it.

b. vq_attn_sm90_kernel<512> at N = 1, T = 262144 against float64 in the classes of test_gpu_attention.py (randn, peaked,
   equal, large) and "needle": q and k rows are +-2 sign codes (a matching scaled logit is 90.5, others have standard
   deviation 4), q_r = k_j(r) with j(r) = 16 (r mod 16384) + (r div 16384) mod 16, so every key block and every position
   in a block is some row's needle and the output row must equal v_j(r).  kP at T = 262144 is 3.9e-3 while one 16-key
   block of a randn row carries about 6e-5 of the softmax mass: only the needle class turns a lost, repeated or
   misordered key block into an O(1) error.  Eight row ranges (rs_op_vq_attention_rows, an 8-member attention team's
   split) equal the full launch bit for bit.  encoder.mid.attn_1 and decoder.mid.attn_1 of the 2048 plans, probed
   under RS_NO_REUSE=1: `.attn` against float64 attention of the plan's own fp16 q, k, v, and the block output against
   x + proj_out(attn) (bound of test_gpu_first_stage_kernels.py b).

c. GroupNorm at 32768 slots per image: each plan GroupNorm on the finalisation route (gn_finalize_kernel, K = slots *
   C/32 items per group) with an "outlier slot" class: in group g one 128-pixel box is offset by +50.  Group g's box
   holds the items that unrolled load g mod 4 of warp g div 4 reads (group 0 takes slot 0 and group 31 the last slot
   in the first placement); a second placement moves every group's box.  A skipped or double-counted slot moves that
   group's mean by about 50 * 128 / (H W) = 1.5e-3, some 600 times the bound.  The statistics bound adds the
   count-dependent term of the kernel's per-thread fp32 sum of K / 256 items to test_gpu_groupnorm.py's constants
   (gn_ref.check_finalize_gstat): at K = 262144 the decoder's rstd error (843 U in one H100 run) exceeds K_R = 512 U
   alone.

d. End to end against the fp32 oracle on the GPU, TF32 off (max|d| <= 1e-2, mean <= 2e-3; the denoiser forward
   test_gpu_unet.py's 1e-2 / 2.5e-3): f4 encode of the bicubic x4 of a 512x512 LQ, f4 decode of a 512x512 latent
   (force_not_quantize; quantised with the code agreement bounded), decode at batch 2 (image 1 bit-identical when
   image 0 changes, and within tolerance of the oracle), the realsr denoiser at 512x512 b1 at two timesteps, one CLI
   unit through ResShiftSampler (realsr_journal, T = 4) stage by stage, and rs_op_tile_gather of two 2048x2048 tiles
   at output columns 0 and 1792 against float64.

test_report prints the worst ratio of error to bound per check, the ops replayed per plan, the wall time and the peak
torch.cuda.max_memory_allocated.
"""
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from tests import gpu_util as G
    from tests import plan_ops
    from tests.gpu_util import module_clock  # noqa: F401  (the module's wall-time fixture)
    from resshift_b200 import _lib
    from tests.attn_ref import kappas, online_qkv, vq_check
    from tests.conv_ref import KAPPA, conv_env, run_conv
    from tests.first_stage_ref import no_reuse, tokens, w16
    from tests.gn_ref import Case, check_finalize_gstat

TOL_MAX, TOL_MEAN = 1e-2, 2e-3
T_CLI, C_CLI = 262144, 512
OBS = {}              # check -> worst ratio of error to bound
REPLAYED = {}         # plan -> {op kind: distinct ops replayed}


def _note(check, ratio):
    G.note(OBS, check, ratio)


def attn_rows(T=T_CLI):
    """ATTN_ROWS of the module docstring."""
    tiles = T // 64
    one = torch.arange(tiles) * 64 + (torch.arange(tiles) * 37) % 64
    full = {0, tiles - 1} | {t for j in range(1, tiles // 132 + 1) for t in (132 * j - 1, 132 * j) if t < tiles}
    rows = set(one.tolist()) | {64 * t + i for t in full for i in range(64)}
    return torch.tensor(sorted(rows), device="cuda")


# ---------------------------------------------------------------------------------------------- plans and their op rows

PLANS = {
    "vq_f4_encode_2048": lambda: plan_ops.first_stage_rows("vq", "f4", 0, 1, 2048, 2048),
    "vq_f4_decode_2048": lambda: plan_ops.first_stage_rows("vq", "f4", 1, 1, 2048, 2048),
    "realsr_denoiser_b1_512x512": lambda: plan_ops.swin_rows("realsr", 1, 512, 512),
}
_ROWS = {}


def plan_rows(plan):
    if plan not in _ROWS:
        _ROWS[plan] = plan_ops.unforced(PLANS[plan])
    return _ROWS[plan]


# ---------------------------------------------------------------------------------------------- a. plan replays

def _replay_convs(plan, rows):
    """Each distinct conv without statistics sinks, on the row bands."""
    convs = plan_ops.conv_rows(rows)
    for i, d in enumerate(convs):
        L = plan_ops.conv_of(d, seed=i)
        want = {k: d[k] for k in plan_ops.CONV_WANT}
        with conv_env():
            out, _, _, ratio = run_conv(f"{plan} {d}", L, stats=False, want=want, out_f32=bool(d["f32"]),
                                        splitk=d["splitk"] > 1, rows=plan_ops.band_rows(d["Ho"]))
        _note("conv", ratio / KAPPA)
        del L, out
        G.free()
    return len(convs), {}


# op kinds checked elsewhere in this module: the T = 262144 attention by b
CHECKED_BY = {"vq_attn": "test_vq_attention_* (b)"}


@pytest.mark.parametrize("plan", list(PLANS))
def test_plan_replay(plan):
    rows = plan_rows(plan)
    assert rows
    replays = {"conv": lambda: _replay_convs(plan, rows), "gn": lambda: plan_ops.replay_gns(plan, rows),
               "attn": lambda: plan_ops.replay_windows(plan, rows),
               "swin_attn": lambda: plan_ops.replay_swins(plan, rows), "mlp": lambda: plan_ops.replay_mlps(plan, rows),
               "upsample": lambda: plan_ops.replay_resamples(rows, 1)}
    done = {}
    for kind, replay in replays.items():
        done[kind], obs = replay()
        for k, r in obs.items():
            _note(f"gn {k}" if kind == "gn" else k, r)
    for r in plan_ops.distinct(rows, "vq_attn"):
        assert tuple(map(int, r)) == (T_CLI, C_CLI, 1), r          # the shape b holds to float64
    REPLAYED[plan] = done
    print(f"[plan] {plan}: " + ", ".join(f"{n} distinct {k}" for k, n in done.items()))
    unclaimed = [r for r in rows if not plan_ops.claimed(r)]
    assert not unclaimed, f"{plan}: op rows no check claims: {sorted(set(unclaimed))}"
    assert not plan_ops.distinct(rows, "unet_attn")


# ---------------------------------------------------------------------------------------------- b. T = 262144 attention

def needle_qkv(T=T_CLI, Cc=C_CLI, seed=0):
    """fp16 q, k, v [1, T, C] of the needle class and j(r)."""
    g = G.gen(seed)
    k = torch.where(torch.rand(1, T, Cc, device="cuda", generator=g) < 0.5, -2.0, 2.0).half()
    r = torch.arange(T, device="cuda")
    j = 16 * (r % 16384) + (r // 16384) % 16
    q = k[:, j].contiguous()
    v = torch.randn(1, T, Cc, device="cuda", generator=g).half()
    return q, k, v, j


def _vq_op(q, k, v, rows=None, out=None):
    N, T, Cc = q.shape
    if out is None:
        out = torch.full((N, T, Cc), float("nan"), dtype=torch.float16, device="cuda")
    rb, re_ = rows or (0, T)
    _lib.check(_lib.lib.rs_op_vq_attention_rows(q.data_ptr(), k.data_ptr(), v.data_ptr(), N, T, Cc, Cc, rb, re_,
                                                out.data_ptr(), G.stream()))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("cls", ["needle", "randn", "peaked", "equal", "large"])
def test_vq_attention_262144(cls):
    rows = attn_rows()
    if cls == "needle":
        q, k, v, j = needle_qkv(seed=3)
        # the class as built: on the checked rows the needle's scaled logit exceeds every other by at least 40
        for i in range(0, rows.numel(), 512):
            r = rows[i:i + 512]
            s = torch.mm(q[0, r].float(), k[0].float().t()) * C_CLI ** -0.5
            top = s[torch.arange(r.numel(), device="cuda"), j[r]]
            s[torch.arange(r.numel(), device="cuda"), j[r]] = -1e9
            assert (top - s.amax(1)).min().item() >= 40
    else:
        q, k, v = (t[:, 0].half().contiguous() for t in online_qkv(cls, 1, 1, T_CLI, C_CLI, G.gen(7 + len(cls))))
    out = _vq_op(q, k, v)
    assert torch.isfinite(out).all()
    _note(f"vq<512> T=262144 {cls}", vq_check(cls, q, k, v, out, rows=rows))
    if cls == "needle":
        # every output row equals its needle's v row: 1/2 ulp16 + the accumulation part of kP
        kp = kappas("vq", T_CLI, C_CLI)[0]
        want = v[0, j].double()
        err = (out[0].double() - want).abs()
        allow = 0.5 * G.ulp16(want) + kp * want.abs() + 2.0 ** -25
        ratio = (err / allow).max().item()
        _note("vq<512> T=262144 needle = v row (all rows)", ratio)
        bad = (err > allow).any(1).nonzero()[:, 0]
        assert bad.numel() == 0, (f"{bad.numel()} rows differ from their needle's v row; first rows {bad[:8].tolist()} "
                                  f"(key blocks {(j[bad[:8]] // 16).tolist()}, query tiles {(bad[:8] // 64).tolist()})")
        # 8 query-row ranges, an 8-member attention team's split, equal the full launch bit for bit
        parts = torch.full_like(out, float("nan"))
        step = T_CLI // 8
        for i in range(8):
            _vq_op(q, k, v, rows=(i * step, (i + 1) * step), out=parts)
        assert torch.equal(G.bits(parts), G.bits(out)), "8 row ranges differ from the full launch"


def _vq_model(seed=0):
    from resshift_b200.models.autoencoder import VQModelTorch
    from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
    cfg = vq_preset("f4")
    sd = random_vq_state_dict(cfg, seed)
    m = VQModelTorch(**cfg.to_kwargs())
    m.load_state_dict(sd, strict=True)
    return cfg, sd, m.cuda().eval()


@pytest.mark.parametrize("which", [0, 1])
def test_vq_attention_plan_mid_blocks(which):
    """encoder.mid.attn_1 (which 0) / decoder.mid.attn_1 (which 1) of the 2048 plans, probed under RS_NO_REUSE=1."""
    p = ("encoder", "decoder")[which] + ".mid.attn_1"
    with no_reuse():
        cfg, sd, m = _vq_model()
        g = G.gen(40 + which)
        if which == 0:
            m.encode(torch.rand(1, 3, 2048, 2048, device="cuda", generator=g) * 2 - 1)
        else:
            m.decode(torch.randn(1, cfg.embed_dim, 512, 512, device="cuda", generator=g) * 0.6, force_not_quantize=True)
        torch.cuda.synchronize()
        pr = {s: m.probe(which, 1, 2048, 2048, p + s) for s in (".in", ".q", ".k", ".v", ".attn", "")}
    del m
    G.free()
    q, k, v, a = (pr[s].flatten(2).transpose(1, 2).half().contiguous() for s in (".q", ".k", ".v", ".attn"))
    assert q.shape == (1, T_CLI, C_CLI)
    assert torch.equal(pr[".v"].half().float(), pr[".v"]), "the .v probe is not the fp16 tensor the kernel read"
    rows = attn_rows()
    _note(f"plan {p}.attn", vq_check("plan", q, k, v, a, rows=rows))
    x, out, at = (tokens(pr[s])[0] for s in (".in", "", ".attn"))
    wp, bp = w16(sd, f"{p}.proj_out.weight", C_CLI), sd[f"{p}.proj_out.bias"].cuda().double()
    x, out, at = x[rows], out[rows], at[rows]
    ref = x + at @ wp.t() + bp
    mag = at.abs() @ wp.abs().t() + bp.abs() + x.abs()
    U32 = 2.0 ** -23
    _note(f"plan {p} output", G.assert_within(f"{p} block output", out, ref, (C_CLI + 2) * U32 * mag, 1.0))
    del pr
    G.free()


# ---------------------------------------------------------------------------------------------- c. GroupNorm, 32768 slots

def outlier_slots(slots, cpg, seed):
    """One slot per group (module docstring, c): group g's box holds items read by unrolled load g % 4 of warp g // 4."""
    K = slots * cpg
    assert 1024 % cpg == 0 and K >= 1024
    g = torch.Generator().manual_seed(seed)
    out = []
    for grp in range(32):
        u, w = grp % 4, grp // 4
        it = int(torch.randint(K // 1024, (1,), generator=g))
        lane = int(torch.randint(max(1, 32 // cpg), (1,), generator=g))
        item = it * 1024 + u * 256 + w * 32 + lane * cpg
        out.append(item // cpg)
    if seed == 0:
        out[0], out[31] = 0, slots - 1               # items 0 .. cpg-1 (load 0, warp 0), K-cpg .. K-1 (load 3, warp 7)
    if K % 1024:                                     # the remainder loop's items
        out[5] = (K // 1024 * 1024 + (K % 1024) // 2) // cpg
    return out


@pytest.mark.parametrize("plan", ["vq_f4_encode_2048", "vq_f4_decode_2048"])
def test_groupnorm_outlier_slots(plan):
    rows = [d for d in plan_ops.gn_rows(plan_rows(plan)) if d["H"] == 2048]
    assert rows, "no GroupNorm at 2048x2048"
    fin = [d for d in rows if d["route"] == "finalize"]
    print(f"[gn route] {plan} 2048x2048: " + ", ".join(f"C={d['C']} route={d['route']} slots={d['slots']}" for d in rows))
    assert fin, "no 2048x2048 GroupNorm takes the finalisation route"
    for i, d in enumerate(fin):
        bw, bh, box_n, slots = G.box128(d["H"], d["W"])
        assert slots == d["slots"] == 32768 and box_n == 1
        cpg = d["C"] // 32
        print(f"[gn outlier] {plan} C={d['C']}: K = {slots * cpg} items per group, remainder {slots * cpg % 1024}")
        for placement in (0, 1):
            L = Case(d["N"], d["H"], d["W"], d["C"], eps=d["eps"], silu=d["silu"], seed=50 + i, device="cuda")
            per_row = d["W"] // bw
            for grp, s in enumerate(outlier_slots(slots, cpg, placement)):
                y0, x0 = (s // per_row) * bh, (s % per_row) * bw
                box = L.x64[:, y0:y0 + bh, x0:x0 + bw, grp * cpg:(grp + 1) * cpg]
                box.copy_((box + 50).half().double())
            L.xbuf[..., L.xc0:L.xc0 + d["C"]] = L.x64.half()
            out = L.run("finalize")
            assert out[1]["finalize"], out[1]
            tag = f"{plan} C={d['C']} outlier slots placement {placement}"
            e_mu, e_r = check_finalize_gstat(tag, L.x64, L.eps, out[2], slots)
            _note("gn finalize outlier: mean", e_mu)
            _note("gn finalize outlier: rstd", e_r)
            L.check_y(tag, out[0], rows=plan_ops.band_rows(d["H"]))
            del L, out
            G.free()


# ---------------------------------------------------------------------------------------------- d. end to end

@pytest.fixture
def fp32_reference():
    with G.fp32_matmuls():
        yield


def _report(tag, got, ref, tol_max=TOL_MAX, tol_mean=TOL_MEAN):
    d = (got.float() - ref.float().to(got.device)).abs()
    mx, mn = d.max().item(), d.mean().item()
    print(f"[cli tile] {tag}: max|d|={mx:.3e} mean|d|={mn:.3e}")
    _note(f"{tag} max", mx / tol_max)
    _note(f"{tag} mean", mn / tol_mean)
    return mx, mn


_ORACLE = {}


def _lq(seed=61):
    return torch.rand(1, 3, 512, 512, device="cuda", generator=G.gen(seed)) * 2 - 1


def _oracle_z_y():
    """The oracle's f4 latent of the bicubic x4 of _lq() (VQ weights of seed 0), computed once."""
    from oracle import vq_oracle as vo
    from oracle import vq_options_oracle as vx
    from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
    if "z_y" not in _ORACLE:
        cfg = vq_preset("f4")
        sd = {n: t.cuda() for n, t in random_vq_state_dict(cfg, 0).items()}
        x = vo.bicubic_upsample(_lq(), 4)
        with torch.no_grad():
            _ORACLE["x"], _ORACLE["z_y"] = x, vx.vq_encode(x, sd, cfg, chunk=2048)
    return _ORACLE["x"], _ORACLE["z_y"]


def test_encode_2048(fp32_reference):
    _, _, m = _vq_model()
    x, z_ref = _oracle_z_y()
    got = m.encode(x)
    assert got.shape == (1, 3, 512, 512) and torch.isfinite(got).all()
    mx, mn = _report("f4 encode 2048x2048 (bicubic x4 of a 512 LQ)", got, z_ref)
    assert mx <= TOL_MAX and mn <= TOL_MEAN


def test_decode_512_latent(fp32_reference):
    from oracle import vq_options_oracle as vx
    cfg, sd, m = _vq_model()
    sd = {n: t.cuda() for n, t in sd.items()}
    z = torch.randn(1, 3, 512, 512, device="cuda", generator=G.gen(62)) * 0.6
    got = m.decode(z, force_not_quantize=True)
    with torch.no_grad():
        ref = vx.vq_decode(z, sd, cfg, force_not_quantize=True, chunk=2048)
    assert got.shape == (1, 3, 2048, 2048) and torch.isfinite(got).all()
    mx, mn = _report("f4 decode 512x512 latent (force_not_quantize)", got, ref)
    assert mx <= TOL_MAX and mn <= TOL_MEAN
    # quantised, on the encoder's latent of a CLI input
    _, z_y = _oracle_z_y()
    with torch.no_grad():
        img_ref, idx_ref = vx.vq_decode(z_y, sd, cfg, return_indices=True, chunk=2048)
    img = m.decode(z_y)
    flips = (m.last_indices.to(idx_ref.device) != idx_ref).float().mean().item()
    mx, mn = _report(f"f4 decode(quantise(z)) 512x512, code flips {flips * 100:.4f} %", img, img_ref)
    assert flips <= 0.002 and mn <= TOL_MEAN
    if flips == 0:
        assert mx <= TOL_MAX


def test_decode_batch2(fp32_reference):
    """chop_bs = 2: 2^31-byte 128-channel and 2^32-byte 256-channel activations."""
    from oracle import vq_options_oracle as vx
    cfg, sd, m = _vq_model()
    g = G.gen(63)
    z = torch.randn(2, 3, 512, 512, device="cuda", generator=g) * 0.6
    a = m.decode(z, force_not_quantize=True)[1].clone()
    z2 = z.clone()
    z2[0] = torch.randn(3, 512, 512, device="cuda", generator=g) * 0.6
    b = m.decode(z2, force_not_quantize=True)[1].clone()
    assert torch.equal(G.bits(a), G.bits(b)), "image 1 changed with image 0"
    del m
    G.free()
    sd = {n: t.cuda() for n, t in sd.items()}
    with torch.no_grad():
        ref = vx.vq_decode(z[1:], sd, cfg, force_not_quantize=True, chunk=2048)[0]
    mx, mn = _report("f4 decode batch 2, image 1", a, ref)
    assert mx <= TOL_MAX and mn <= TOL_MEAN


def test_denoiser_512(fp32_reference):
    from oracle import unet_oracle as uo
    from resshift_b200.config import preset
    from resshift_b200.models.unet import UNetModelSwin
    from resshift_b200.weights import random_state_dict
    ucfg, _ = preset("realsr")
    sd = random_state_dict(ucfg, 0)
    m = UNetModelSwin(**ucfg.to_kwargs())
    m.load_state_dict(sd)
    m = m.cuda().eval()
    sdc = {n: t.cuda() for n, t in sd.items()}
    g = G.gen(64)
    x = torch.randn(1, 3, 512, 512, device="cuda", generator=g)
    lq = torch.rand(1, 3, 512, 512, device="cuda", generator=g) * 2 - 1
    for tt in (14, 2):
        t = torch.tensor([tt], device="cuda")
        got = m(x, t, lq=lq)
        with torch.no_grad():
            ref = uo.unet_forward(sdc, ucfg, x, t, lq=lq)
        mx, mn = _report(f"realsr denoiser 512x512 b1 t={tt}", got, ref, G.FWD_MAX, G.FWD_MEAN)
        assert mx <= G.FWD_MAX and mn <= G.FWD_MEAN


def test_cli_unit_sampler(fp32_reference):
    """One CLI unit: sf 4, chop 512 / stride 448, a 512x512 LQ, realsr_journal (T = 4), stage by stage."""
    from oracle import diffusion_oracle as do
    from oracle import unet_oracle as uo
    from oracle import vq_options_oracle as vx
    from resshift_b200.config import preset
    from resshift_b200.sampler import ResShiftSampler, make_configs
    from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
    from resshift_b200.weights import random_state_dict
    ucfg, dcfg = preset("realsr_journal")
    dcfg.sf = 4
    vcfg = vq_preset("f4")
    ae = {"target": "ldm.models.autoencoder.VQModelTorch", "params": vcfg.to_kwargs(), "ckpt_path": random_vq_state_dict(vcfg, 0)}
    configs = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    s = ResShiftSampler(configs, sf=4, use_amp=True, seed=123, chop_size=512, chop_stride=448, padding_offset=16)
    diff, aem, model = s.base_diffusion, s.autoencoder, s.model
    T = diff.num_timesteps
    assert T == 4
    y0 = _lq()
    g = G.gen(65)
    noises = torch.stack([torch.randn(1, 3, 512, 512, device="cuda", generator=g) for _ in range(T + 1)])
    sd_u = {n: t.cuda() for n, t in random_state_dict(ucfg, 0).items()}
    sd_v = {n: t.cuda() for n, t in random_vq_state_dict(vcfg, 0).items()}
    _, z_y_ref = _oracle_z_y()
    tabs = do.schedule_tables(do.eta_schedule(dcfg.steps, dcfg.min_noise_level, dcfg.etas_end, dcfg.kappa,
                                              dcfg.schedule_kwargs["power"]), dcfg.kappa)
    with torch.no_grad():
        z_ref = do.p_sample_loop(lambda xx, tt: uo.unet_forward(sd_u, ucfg, xx, tt, lq=y0), z_y_ref, list(noises), tabs,
                                 dcfg.kappa)
        img_ref, idx_ref = vx.vq_decode(z_ref, sd_v, vcfg, return_indices=True, chunk=2048)
    z_y = diff.encode_first_stage(y0, aem, up_sample=True)
    mx, mn = _report("CLI unit: z_y", z_y, z_y_ref)
    assert mx <= TOL_MAX and mn <= TOL_MEAN
    z = diff.sample_latent(z_y, model, {"lq": y0}, noises=noises)
    mx, mn = _report("CLI unit: final latent", z, z_ref, TOL_MAX, G.FWD_MEAN)
    assert mx <= TOL_MAX and mn <= G.FWD_MEAN
    img_same = aem.decode(z_ref)
    flips = (aem.last_indices.to(idx_ref.device) != idx_ref).float().mean().item()
    mx, mn = _report(f"CLI unit: decode(quantise(z_ref)), code flips {flips * 100:.4f} %", img_same, img_ref)
    assert flips <= 0.002 and mn <= TOL_MEAN
    if flips == 0:
        assert mx <= TOL_MAX
    diff.draw_noises = lambda z_y_, noise=None, noise_repeat=False: noises.to(z_y_.device)
    out = s.sample_func(y0, noise_repeat=False, mask=None).float()
    flips = (aem.last_indices.to(idx_ref.device) != idx_ref).float().mean().item()
    d = (out - img_ref.clamp(-1, 1)).abs()
    print(f"[cli tile] CLI unit end to end: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e} "
          f"code flips {flips * 100:.3f} %")
    assert out.shape == (1, 3, 2048, 2048) and torch.isfinite(out).all() and out.abs().max().item() <= 1.0
    assert flips <= 0.05 and d.mean().item() <= 5e-2         # test_gpu_vq.py's end-to-end bounds
    if flips == 0:
        assert d.max().item() <= TOL_MAX


def test_tile_gather_cli_geometry():
    """Two 2048x2048 tiles at output columns 0 and 1792 (stride 448 x 4) against float64."""
    g = G.gen(66)
    N, Cc, th, tw = 1, 3, 2048, 2048
    ys, xs = [0], [0, 1792]
    H, W = th, xs[-1] + tw
    tiles = torch.randn(2, N, Cc, th, tw, device="cuda", generator=g)
    acc = torch.zeros(N, Cc, H, W, device="cuda", dtype=torch.float64)
    mag = torch.zeros_like(acc)
    cnt = torch.zeros_like(acc)
    for ix, x0 in enumerate(xs):
        acc[..., x0:x0 + tw] += tiles[ix].double()
        mag[..., x0:x0 + tw] += tiles[ix].double().abs()
        cnt[..., x0:x0 + tw] += 1
    out = torch.full((N, Cc, H, W), float("nan"), device="cuda")
    ys_d = torch.tensor(ys, dtype=torch.int32, device="cuda")
    xs_d = torch.tensor(xs, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib.rs_op_tile_gather(tiles.data_ptr(), N, Cc, H, W, th, tw, len(ys), len(xs), ys_d.data_ptr(),
                                          xs_d.data_ptr(), out.data_ptr(), G.stream()))
    torch.cuda.synchronize()
    ref = acc / cnt
    allow = 2.0 ** -23 * mag / cnt                     # one fp32 sum rounding and the division, relative to the sum of |tiles|
    err = (out.double() - ref).abs()
    _note("tile gather", (err / allow.clamp(min=1e-30)).max().item())
    assert not (err > allow).any(), f"tile gather: {int((err > allow).sum())} elements outside the bound"


# ---------------------------------------------------------------------------------------------- report

def test_report(module_clock):
    """Run with the rest of the module: the worst ratio of error to bound per check, ops per plan, wall time, memory."""
    if not OBS:
        pytest.skip("run with the rest of the module")
    for k, r in sorted(OBS.items()):
        print(f"[observed] {k}: worst ratio {r:.3g}")
    for plan, d in REPLAYED.items():
        print(f"[replayed] {plan}: " + ", ".join(f"{n} {k}" for k, n in d.items()))
    props = torch.cuda.get_device_properties(0)
    print(f"[cli tile] wall time {time.time() - module_clock:.1f} s, peak max_memory_allocated "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB on {props.name}")
