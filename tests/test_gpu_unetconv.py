"""GPU tests of the reference's UNetModelConv on the native kernels.

Epilogue: the conv's second, SiLU output (``rs_conv_args.silu_out``, a channel slice of a wider buffer) and its FiLM
after the activation (``film``, one row per image or one shared row), on every route the launcher can take — one tile,
CTA pair, persistent, persistent pair, split-K with the reduce kernel, the SIMT cross-check kernel, and RS_CONV_MSUB=2 /
RS_CONV_EPI=direct, which the launcher steers to one sub-tile / the staged epilogue for such convs — against float64
with the error model of test_gpu_conv_instances.py (tests/conv_ref.py).  silu_out must be within one fp16 ulp of SiLU of
the stored output, repeated launches bit-identical, the reported route the forced one, and nothing outside the views
written.  Resampling: pool / upsample with the SiLU output against torch.  Models: every fixture of
tests/golden/unetconv.npz against the reference and the fp32 oracle, a 64x128 latent, an image alone equal to the same
image in a batch, the fused 4-step loop (graph replay equal to eager enqueue) against the reference's trajectory,
ResShiftSampler end to end from a ``models.unet.UNetModelConv`` yaml, one GPU and a device pool."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import unetconv_oracle as uo
from oracle.make_golden_unetconv import CASES, OUT_STRIDE, case_config, case_inputs, trajectory_inputs
from resshift_b200.weights import random_state_dict

if torch.cuda.is_available():
    from resshift_b200 import _lib
    from tests import gpu_util as G
    from tests import plan_ops
    from tests.conv_ref import MODES, Conv, check_silu_film, conv_env, epi_bc, film_rows, launch_silu, resample_case

FWD_MAX, FWD_MEAN = 1e-2, 2.5e-3
LOOP_MAX, LOOP_MEAN = 1e-2, 3e-3


# ---------------------------------------------------------------------------------------------- epilogue

@pytest.mark.parametrize("form", ["none", "image", "shared"])
@pytest.mark.parametrize("bn", [16, 48, 64, 128, 256])
@pytest.mark.parametrize("mode", ["one_tile", "pair", "msub2", "persistent", "persistent_pair"])
def test_silu_output_and_film(mode, bn, form):
    """Forced channel tile x route, SiLU with a per-image bias (the in_layers conv folds emb_out into it), FiLM rows or a
    residual (the out_layers conv); Cout = 2 BN + 8 ends on a partial channel tile.  The SiLU output and FiLM run on
    one-sub-tile instances: RS_CONV_MSUB=2 is steered to one sub-tile, and requiring two is refused."""
    env, (cg, msub, persist) = MODES[mode]
    L = Conv(3, 16, 16, 72, 2 * bn + 8, 3, act=2, bias="row" if msub == 2 else "image", res=form == "none", seed=bn + len(form))
    if msub == 2:
        with conv_env(**env), pytest.raises(_lib.RsError, match="sub-tiles"):
            launch_silu(L, *film_rows(L, form, bn)[:2], bn=bn, msub=2)
        env = dict(env, RS_CONV_MSUB=2)
    with conv_env(**env):
        check_silu_film(f"silu BN={bn} {mode} film={form}", L, form, bn, bn=bn,
                        want={"BN": bn, "cg": cg, "msub": 1, "persist": persist, "splitk": 1, "epi_bc": epi_bc(bn)})


@pytest.mark.parametrize("form", ["none", "image", "shared"])
@pytest.mark.parametrize("route", ["split_k", "direct", "simt"])
def test_silu_output_and_film_other_routes(route, form):
    """Split-K (the reduce kernel writes both outputs), the SIMT cross-check kernel, and RS_CONV_EPI=direct, which the
    launcher steers to the staged epilogue (the direct epilogue has no SiLU output or FiLM)."""
    res = form == "none"
    if route == "split_k":
        L = Conv(3, 8, 8, 392, 104, 3, act=2, bias="image", res=res, seed=7 + len(form))
        with conv_env(RS_CONV_SPLITK=2, RS_CONV_PERSIST=0):
            check_silu_film(f"split-K film={form}", L, form, 11, splitk=True, want={"splitk": 2, "epi_bc": 0, "persist": 0})
    else:
        L = Conv(3, 16, 16, 72, 88, 3, act=2, bias="image", res=res, seed=9 + len(form))
        env = {"RS_CONV_EPI": "direct"} if route == "direct" else {"RS_CONV_IMPL": "simt"}
        want = {"epi_bc": "nonzero"} if route == "direct" else {"epi_bc": 0, "splitk": 1}
        with conv_env(**env):
            got, s, _ = check_silu_film(f"{route} film={form}", L, form, 13, want=want)
        if route == "direct":     # the staged epilogue it was steered to: the same launch as without the override
            with conv_env():
                got2, s2, _ = check_silu_film(f"staged film={form}", L, form, 13, want={"epi_bc": "nonzero"})
            assert torch.equal(G.bits(got), G.bits(got2)) and torch.equal(G.bits(s), G.bits(s2))


def test_silu_output_refusals():
    L = Conv(2, 16, 16, 64, 64, 3, act=2, res=True, seed=1)
    film = torch.zeros(1, 128, device="cuda")
    with conv_env():
        with pytest.raises(_lib.RsError, match="no residual"):
            launch_silu(L, film, 0)


# ---------------------------------------------------------------------------------------------- resampling

@pytest.mark.parametrize("pool", [False, True])
@pytest.mark.parametrize("shape", [(2, 8, 12, 64), (3, 16, 16, 8), (1, 40, 24, 96)])
def test_resample_with_silu_output(shape, pool):
    resample_case(*shape, pool)


# ---------------------------------------------------------------------------------------------- models

def _model(ucfg, seed=0):
    from resshift_b200.models.unet import UNetModelConv
    m = UNetModelConv(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, seed), strict=True)
    return m.cuda().eval()


def _cmp(tag, got, ref, bmax=FWD_MAX, bmean=FWD_MEAN):
    d = (got.float().cpu() - ref.float().cpu()).abs()
    print(f"[parity] {tag}: max|d|={d.max().item():.3e} mean|d|={d.mean().item():.3e}")
    assert not torch.isnan(got).any()
    assert d.max().item() <= bmax and d.mean().item() <= bmean, tag


@pytest.mark.parametrize("name", list(CASES))
def test_forward_vs_reference_golden(golden_dir, name):
    g = np.load(golden_dir / "unetconv.npz")
    ucfg, _, _ = case_config(name)
    seed, h, w = (int(v) for v in g[f"{name}/seed"])
    x, lq = case_inputs(ucfg, 2, h, w, seed)
    out = _model(ucfg)(x.cuda(), torch.from_numpy(g[f"{name}/t"]).cuda(), lq=lq.cuda())
    _cmp(f"golden {name}", out.reshape(-1)[::OUT_STRIDE], torch.from_numpy(g[f"{name}/out_sub"]))


@pytest.mark.parametrize("name,hw", [(n, CASES[n][1:]) for n in CASES] + [("defaults", (64, 128)), ("ss_updown", (64, 128))])
def test_forward_vs_oracle_fresh_inputs(name, hw):
    ucfg, _, _ = case_config(name)
    x, lq = case_inputs(ucfg, 2, hw[0], hw[1], 9200)
    t = torch.tensor([0, 3])
    ref = uo.unetconv_forward(random_state_dict(ucfg, 0), ucfg, x, t, lq=lq)
    _cmp(f"oracle {name} {hw}", _model(ucfg)(x.cuda(), t.cuda(), lq=lq.cuda()), ref)


@pytest.mark.parametrize("name", ["ss_updown", "uneven"])
def test_image_alone_equals_image_in_batch(name):
    ucfg, _, (h, w) = case_config(name)
    m = _model(ucfg)
    x, lq = case_inputs(ucfg, 3, h, w, 9300)
    t = torch.tensor([5, 2, 0])
    full = m(x.cuda(), t.cuda(), lq=lq.cuda())
    alone = m(x[1:2].cuda(), t[1:2].cuda(), lq=lq[1:2].cuda())
    assert torch.equal(full[1:2], alone)


def test_fused_loop_vs_reference_trajectory_and_graph_replay(golden_dir):
    from resshift_b200.models.script_util import create_gaussian_diffusion
    g = np.load(golden_dir / "unetconv.npz")
    ucfg, dcfg, hw = case_config("defaults")
    m = _model(ucfg)
    diff = create_gaussian_diffusion(**dcfg.to_kwargs())
    assert diff._native_ok(m, clip_denoised=False, denoised_fn=None, model_kwargs={"lq": None})
    y, noises = trajectory_inputs(2, dcfg.steps, hw)
    y, noises = y.cuda(), noises.cuda()
    finals = [diff.sample_latent(y, m, {"lq": y}, noises=noises).clone() for _ in range(2)]   # capture, then replay
    eager = diff.sample_latent(y, m, {"lq": y}, noises=noises, use_graph=False)
    assert torch.equal(finals[0], finals[1]) and torch.equal(finals[0], eager)
    _cmp("loop defaults", finals[0].reshape(-1)[::OUT_STRIDE], torch.from_numpy(g["loop/final_sub"]), LOOP_MAX, LOOP_MEAN)


def test_native_inputs_are_checked():
    from resshift_b200.models.script_util import create_gaussian_diffusion
    ucfg, dcfg, _ = case_config("lq2x")
    m = _model(ucfg)
    diff = create_gaussian_diffusion(**dcfg.to_kwargs())
    z = torch.zeros(1, 3, 32, 32, device="cuda")
    with pytest.raises(ValueError, match="lq must have shape"):
        diff.sample_latent(z, m, {"lq": torch.zeros(1, 3, 32, 32, device="cuda")})
    with pytest.raises(ValueError, match="no mask"):
        diff.sample_latent(z, m, {"lq": torch.zeros(1, 3, 64, 64, device="cuda"), "mask": torch.zeros(1, 1, 64, 64, device="cuda")})


def test_plan_profile_names_the_silu_outputs():
    """Every conv / resample whose output a ResBlockConv or the head reads writes its SiLU twin; the in_layers convs of the
    scale-shift model apply FiLM rows."""
    ucfg, _, (h, w) = case_config("ss_updown")
    m = _model(ucfg)
    x, lq = case_inputs(ucfg, 2, h, w, 1)
    m(x.cuda(), torch.tensor([1, 2]).cuda(), lq=lq.cuda())
    rows = plan_ops.plan_rows(m.plan(2, h, w), x.cuda(), torch.tensor([1.0, 2.0], device="cuda"), lq.cuda())
    assert not any(r.startswith("gn ") for r in rows)
    in_convs = [r for r in rows if ".in_layers.1." in r]
    out_convs = [r for r in rows if ".out_layers.1." in r]
    assert in_convs and all("silu=0 film=1" in r for r in in_convs)
    assert out_convs and all("silu=1" in r for r in out_convs)
    assert any(r.startswith("avgpool") for r in rows) and any(r.startswith("upsample") for r in rows)


# ---------------------------------------------------------------------------------------------- the whole pipeline

def _sampler(devices=None):
    from resshift_b200.sampler import ResShiftSampler, make_configs
    from resshift_b200.vq_arch import random_vq_state_dict, vq_preset
    ucfg, dcfg, _ = case_config("defaults")
    dcfg.sf = 4
    vcfg = vq_preset("tiny")
    ae = {"target": "ldm.models.autoencoder.VQModelTorch", "params": vcfg.to_kwargs(), "ckpt_path": random_vq_state_dict(vcfg, 0)}
    configs = make_configs(ucfg, dcfg, autoencoder=ae, state_dict=random_state_dict(ucfg, 0))
    configs.model.target = "models.unet.UNetModelConv"                   # the reference's yaml target string
    return ResShiftSampler(configs, sf=4, use_amp=True, seed=123, devices=devices, chop_size=64, chop_stride=48,
                           padding_offset=64)


def test_sampler_end_to_end_and_device_pool(tmp_path):
    import cv2
    from resshift_b200.models.unet import UNetModelConv
    s = _sampler()
    assert isinstance(s.model, UNetModelConv)
    assert s.base_diffusion._native_ok(s.model, clip_denoised=False, denoised_fn=None, model_kwargs={"lq": None})
    rng = np.random.default_rng(12)
    (tmp_path / "in").mkdir()
    for name, (h, w) in {"a": (90, 70), "b": (61, 47)}.items():     # odd sizes: reflect-padded to padding_offset
        cv2.imwrite(str(tmp_path / "in" / f"{name}.png"), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
    outs = []
    for smp, d in ((s, "ref"), (_sampler("0,0"), "pool")):
        smp.setup_seed()
        smp.inference(tmp_path / "in", tmp_path / d, bs=2)
        outs.append({p.name: p.read_bytes() for p in sorted((tmp_path / d).iterdir())})
    assert len(outs[0]) == 2 and outs[0] == outs[1]
    img = cv2.imread(str(tmp_path / "ref" / "b.png"))
    assert img.shape == (61 * 4, 47 * 4, 3)
