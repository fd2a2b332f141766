"""GPU parity of first stages built with the Encoder / Decoder options — attention at any level, attn_type none, pooled
resampling, tanh_out — against the reference's own outputs (oracle/make_golden_vq_options.py) and the oracle run on the
GPU in fp32 (oracle/vq_options_oracle.py); passes with several fused attentions (attention blocks over more than 8192 positions): the segments between
them (rs_vq_run_between), attention teams that split each of them, and a device pool whose single tile forms a team.

Bounds as in test_gpu_vq.py: per-pixel |delta| <= 1e-2 and mean |delta| <= 2e-3 on the continuous parts; the quantised
decode is held to the code agreement (reported) and its mean."""
from dataclasses import replace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import vq_options_oracle as oo
from oracle.make_golden_vq_options import RUNS, configs, inputs
from resshift_b200 import _lib as L
from resshift_b200.parallel import attention_row_ranges
from resshift_b200.vq_arch import ldm_vq_preset, random_kl_state_dict, random_vq_state_dict, vq_preset

TOL_MAX, TOL_MEAN = 1e-2, 2e-3
RUN_IDS = [(name, r) for name, runs in RUNS.items() for r in range(len(runs))]


def _model(cfg, seed=0):
    from resshift_b200.models.autoencoder import AutoencoderKLTorch, VQModelTorch
    m = (AutoencoderKLTorch if cfg.kl else VQModelTorch)(**cfg.to_kwargs())
    sd = (random_kl_state_dict if cfg.kl else random_vq_state_dict)(cfg, seed)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval(), sd


def _report(tag, got, ref):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    print(f"[vq options] {tag}: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e} ref_std={ref.float().std().item():.3f}")
    return d.max().item(), d.mean().item()


@pytest.mark.parametrize("name,r", RUN_IDS)
def test_vs_reference_golden(golden_dir, name, r):
    cfg = configs()[name]
    key = f"{name}_{r}"
    gold = np.load(golden_dir / RUNS[name][r][3])
    m, sd = _model(cfg)
    x, z = inputs(name, r)
    x = x.cuda()
    if cfg.kl:
        zz, mom = m.encode(x, sample_posterior=False, return_moments=True)
        ref = torch.from_numpy(gold["moments"])
        for tag, got, want in (("moments", mom, ref), ("mode", zz, ref[:, :cfg.embed_dim])):
            mx, mn = _report(f"{key} {tag}", got, want)
            assert mx <= TOL_MAX and mn <= TOL_MEAN
        mx, mn = _report(f"{key} decode", m.decode(ref[:, :cfg.embed_dim].contiguous().cuda()), torch.from_numpy(gold["dec"]))
        assert mx <= TOL_MAX and mn <= TOL_MEAN
        return
    mx, mn = _report(f"{key} encode", m.encode(x), torch.from_numpy(gold["enc"]))
    assert mx <= TOL_MAX and mn <= TOL_MEAN
    z = z.cuda()
    mx, mn = _report(f"{key} decode (not quantised)", m.decode(z, force_not_quantize=True), torch.from_numpy(gold["dec_nq"]))
    assert mx <= TOL_MAX and mn <= TOL_MEAN
    # quantised: the code map against the reference's, the image against the oracle's decode of the same latent (the
    # oracle's quantised decode is pinned to the reference through the code map and dec_nq)
    dec = m.decode(z)
    flips = m.last_indices.cpu().numpy() != gold["idx"]
    print(f"[vq options] {key}: code flips {int(flips.sum())} / {flips.size}")
    assert flips.mean() <= 0.002
    mx, mn = _report(f"{key} decode (quantised) vs oracle", dec, oo.vq_decode(z.cpu(), sd, cfg))
    assert mn <= TOL_MEAN
    if not flips.any():
        assert mx <= TOL_MAX
    if cfg.tanh_out:
        assert dec.abs().max().item() <= 1.0


@pytest.mark.parametrize("name,r", RUN_IDS)
def test_vs_oracle(name, r):
    cfg = configs()[name]
    key = f"{name}_{r}"
    m, sd = _model(cfg)
    x, _ = inputs(name, r)
    if cfg.kl:
        _, mom = m.encode(x.cuda(), sample_posterior=False, return_moments=True)
        mx, mn = _report(f"{key} moments vs oracle", mom, oo.kl_moments(x, sd, cfg))
    else:
        mx, mn = _report(f"{key} encode vs oracle", m.encode(x.cuda()), oo.vq_encode(x, sd, cfg))
    assert mx <= TOL_MAX and mn <= TOL_MEAN


# (tag, config, batch, image H, W, fused attentions of encode, of decode)
LARGE = [("f4_attn_128_64", replace(vq_preset("f4"), attn_resolutions=(128, 64)), 1, 512, 512, 5, 7),
         ("ldm_f8_1024", ldm_vq_preset("vq-f8"), 1, 1024, 1024, 3, 4)]


@pytest.fixture(scope="module")
def large_models():
    return {tag: _model(cfg) for tag, cfg, *_ in LARGE}


@pytest.mark.parametrize("tag,cfg,b,hh,ww,n_enc,n_dec", LARGE, ids=[c[0] for c in LARGE])
def test_several_fused_attentions_vs_gpu_oracle(large_models, tag, cfg, b, hh, ww, n_enc, n_dec):
    """The oracle in fp32 on the GPU, its attention in 4096-row chunks (exact: each row's softmax is over all keys)."""
    m, sd = large_models[tag]
    sdg = {k: v.cuda() for k, v in sd.items()}
    g = torch.Generator(device="cuda").manual_seed(21)
    x = torch.rand(b, 3, hh, ww, device="cuda", generator=g) * 2 - 1
    enc = m.encode(x)
    assert len(m.plan(0, b, hh, ww).attentions) == n_enc and len(m.plan(1, b, hh, ww).attentions) == n_dec
    with torch.no_grad():
        ref = oo.vq_encode(x, sdg, cfg, chunk=4096)
    mx, mn = _report(f"{tag} encode vs GPU oracle", enc, ref)
    assert mx <= TOL_MAX and mn <= TOL_MEAN
    z = torch.randn(ref.shape, device="cuda", generator=g) * 0.6
    dec = m.decode(z, force_not_quantize=True)
    with torch.no_grad():
        ref = oo.vq_decode(z, sdg, cfg, force_not_quantize=True, chunk=4096)
    del sdg
    mx, mn = _report(f"{tag} decode vs GPU oracle", dec, ref)
    assert mx <= TOL_MAX and mn <= TOL_MEAN


def test_batch_independence_and_determinism():
    cfg = configs()["levels"]
    m, _ = _model(cfg)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.rand(3, 3, 96, 160, device="cuda", generator=g) * 2 - 1
    a = m.encode(x).clone()
    assert torch.equal(a, m.encode(x))
    x2 = torch.rand_like(x) * 2 - 1
    x2[1] = x[1]
    assert torch.equal(m.encode(x2)[1], a[1])
    z = torch.randn(3, 3, 24, 40, device="cuda", generator=g) * 0.6
    d = m.decode(z).clone()
    assert torch.equal(d, m.decode(z))
    z2 = torch.randn_like(z) * 0.6
    z2[2] = z[2]
    assert torch.equal(m.decode(z2)[2], d[2])
    # tanh_out and pooled resampling
    m, _ = _model(configs()["noattn_pool_tanh"])
    d = m.decode(z).clone()
    assert torch.equal(d, m.decode(z)) and d.abs().max().item() <= 1.0


def test_segments_equal_whole_pass_and_refuse_out_of_order(large_models):
    m, _ = large_models["ldm_f8_1024"]
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.rand(1, 3, 1024, 1024, device="cuda", generator=g) * 2 - 1
    ref = m.encode(x).clone()
    plan = m.plan(0, 1, 1024, 1024)
    n = len(plan.attentions)
    assert n == 3
    st = L.current_stream()
    out = torch.empty_like(ref)
    L.check(L.lib.rs_vq_encode_begin(plan.handle, x.data_ptr(), st))
    for a in range(1, n):
        L.check(L.lib.rs_vq_run_between(plan.handle, a, st))
    L.check(L.lib.rs_vq_encode_end(plan.handle, out.data_ptr(), st))
    assert torch.equal(out, ref)
    img = m.decode(ref).clone()
    dplan = m.plan(1, 1, 1024, 1024)
    idx = torch.empty_like(m.last_indices)
    dout = torch.empty_like(img)
    L.check(L.lib.rs_vq_decode_begin(dplan.handle, ref.data_ptr(), idx.data_ptr(), 0, st))
    for a in range(1, len(dplan.attentions)):
        L.check(L.lib.rs_vq_run_between(dplan.handle, a, st))
    L.check(L.lib.rs_vq_decode_end(dplan.handle, dout.data_ptr(), st))
    assert torch.equal(dout, img) and torch.equal(idx, m.last_indices)
    # out of order / out of range
    L.check(L.lib.rs_vq_encode_begin(plan.handle, x.data_ptr(), st))
    for a, msg in ((2, "out of order"), (0, "outside"), (3, "outside")):
        with pytest.raises(L.RsError, match=msg):
            L.check(L.lib.rs_vq_run_between(plan.handle, a, st))
    with pytest.raises(L.RsError, match="_end out of order"):
        L.check(L.lib.rs_vq_encode_end(plan.handle, out.data_ptr(), st))
    L.check(L.lib.rs_vq_run_between(plan.handle, 1, st))
    with pytest.raises(L.RsError, match="out of order"):
        L.check(L.lib.rs_vq_run_between(plan.handle, 1, st))
    L.check(L.lib.rs_vq_run_between(plan.handle, 2, st))
    L.check(L.lib.rs_vq_encode_end(plan.handle, out.data_ptr(), st))
    assert torch.equal(out, ref)
    with pytest.raises(L.RsError, match="out of order"):             # after _end, _begin comes next
        L.check(L.lib.rs_vq_run_between(plan.handle, 1, st))
    # the a = 0 calls keep their meaning, and the _at calls name the attention
    for a, view in enumerate(plan.attentions):
        assert view.shape == (1, 128 * 128, 512)
    with pytest.raises(L.RsError, match="outside"):
        L.check(L.lib.rs_vq_set_attention_rows_at(plan.handle, 3, 0, 64))


def _team_runs(m, call, members, which, n_attn):
    """Virtual members of a team, one after the other, with one exchange per fused attention of the pass.  A pass
    through a team of one (every row computed, the same segments) records each attention's full output; then each
    member runs with only its rows computed, checks them against that record bit for bit, and its exchange writes the
    other members' rows from it.  (Rows captured from the members themselves, as test_gpu_vq_attention_rows.py does
    with one attention, would be wrong from the second attention on: a member's input there depends on every row of
    the first.)  Returns the outputs of the members' runs."""
    full = []
    with m.attention_team(0, 1, lambda view, rb, re: full.append(view.clone())):
        call()
    assert len(full) == n_attn

    def fill(member):
        count = [0]

        def exchange(view, rb, re):
            a = count[0]
            assert (rb, re) != (0, view.shape[1]) and torch.equal(view[:, rb:re], full[a][:, rb:re])
            for m2, (b2, e2) in enumerate(attention_row_ranges(view.shape[1], members)):
                if m2 != member:
                    view[:, b2:e2] = full[a][:, b2:e2]
            count[0] += 1
        return exchange

    outs = []
    for member in range(members):
        with m.attention_team(member, members, fill(member)):
            outs.append(call())
            views = m.plan(which, *call.plan_key).attentions
            assert len(views) == n_attn
            assert m.attention_rows == [(which, *attention_row_ranges(v.shape[1], members)[member]) for v in views]
    return outs


@pytest.mark.parametrize("members", [2, 3])
def test_attention_teams_bit_identical(large_models, members):
    m, _ = large_models["f4_attn_128_64"]
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.rand(1, 3, 512, 512, device="cuda", generator=g) * 2 - 1
    ref = m.encode(x).clone()
    enc = lambda: m.encode(x).clone()
    enc.plan_key = (1, 512, 512)
    for got in _team_runs(m, enc, members, 0, 5):
        assert torch.equal(got, ref)
    z = torch.randn(1, 3, 128, 128, device="cuda", generator=g) * 0.6
    dref = m.decode(z).clone()
    dec = lambda: m.decode(z).clone()
    dec.plan_key = (1, 512, 512)
    for got in _team_runs(m, dec, members, 1, 7):
        assert torch.equal(got, dref)


def test_plan_refuses_fused_form_at_64_channels():
    m, _ = _model(replace(vq_preset("tiny"), attn_resolutions=(32,)))
    with pytest.raises(L.RsError, match=r"encoder\.down\.1\.attn\.0.*\{128, 256, 512\}"):
        m.encode(torch.zeros(1, 3, 192, 192, device="cuda"))


def test_device_pool_team_with_several_fused_attentions(tmp_path):
    """inference() of one 128x128 LQ tile (x4: 512x512, a 128x128 bottleneck) with a tiny first stage that has
    attention at resolution 16 (its bottleneck level): 3 fused attentions per encode, 4 per decode.  A pool of two
    replicas of this device runs the tile as one team; the PNGs equal the one-GPU run's."""
    import cv2
    from resshift_b200.config import preset
    from resshift_b200.sampler import ResShiftSampler, make_configs
    from resshift_b200.weights import random_state_dict
    ucfg, dcfg = preset("tiny")
    dcfg.sf = 4
    vcfg = replace(vq_preset("tiny"), attn_resolutions=(16,))
    ae = {"target": "ldm.models.autoencoder.VQModelTorch", "params": vcfg.to_kwargs(), "ckpt_path": random_vq_state_dict(vcfg, 0)}
    configs_ = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    chop = dict(chop_size=512, chop_stride=448, padding_offset=16)
    (tmp_path / "in").mkdir()
    cv2.imwrite(str(tmp_path / "in" / "t.png"), np.random.default_rng(7).integers(0, 256, (128, 128, 3), dtype=np.uint8))
    outs = {}
    for tag, devices in (("one", None), ("pool", "0,0")):
        s = ResShiftSampler(configs_, sf=4, use_amp=True, seed=123, devices=devices, **chop)
        s.setup_seed()
        s.inference(tmp_path / "in", tmp_path / tag, bs=1)
        outs[tag] = (tmp_path / tag / "t.png").read_bytes()
        if devices is not None:
            rows = [rep.autoencoder.attention_rows for rep in s.pool.replicas]
            for r in rows:
                assert [w for w, _, _ in r] == [0] * 3 + [1] * 4, r
            for k in range(7):                      # each attention's rows tile [0, T) across the two members
                (a0, a1), (b0, b1) = sorted((r[k][1], r[k][2]) for r in rows)
                assert a0 == 0 and a1 == b0 and b1 == 16384 and a1 > a0
    assert outs["pool"] == outs["one"]
