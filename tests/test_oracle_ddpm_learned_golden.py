"""Pins learned-variance DDPM models (learn_sigma=True: a 2 C head, LEARNED_RANGE) to the reference: the port's torch
route on each family's oracle UNet against the fixtures of oracle/make_golden_ddpm_learned.py, the param specs of the
widened models against the reference's inventories, the constructors' channel rule (x has out_channels, or
out_channels / 2 channels with a learned variance), and which calls the fused loop takes.  CPU only."""
import json

import numpy as np
import pytest
import torch

from oracle import unet_oracle, unetconv_oracle, unetmodel_oracle
from oracle.make_golden_ddpm_learned import CASES, OUT_STRIDE, case_inputs, diffusion_kwargs, model_config
from oracle.make_golden_ddpm import learned_range_model
from resshift_b200.arch import unet_param_spec, unetconv_param_spec, unetmodel_param_spec
from resshift_b200.config import UNetConfig, UNetModelConfig, UNetModelConvConfig
from resshift_b200.models import gaussian_diffusion as gd
from resshift_b200.models.script_util import create_gaussian_diffusion_ddpm
from resshift_b200.models.unet import UNetModel, UNetModelConv, UNetModelSwin
from resshift_b200.weights import random_state_dict

TOL = 2e-4   # fp32 CPU vs fp32 CPU, different op order inside the UNet; relative to the fixture's largest magnitude
V = gd.ModelVarTypeDDPM


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(golden_dir / "ddpm_learned.npz")


def _close(got, ref, what):
    err = np.abs(np.asarray(got) - ref).max()
    assert err < TOL * max(1.0, np.abs(ref).max()), f"{what}: max|d| {err:.3e} at max|ref| {np.abs(ref).max():.3e}"


@pytest.mark.parametrize("case", sorted(CASES))
def test_port_torch_route_matches_reference(gold, case, monkeypatch):
    """SpacedDiffusionDDPM's torch route (LEARNED_RANGE: the second half of the output interpolates the log variance),
    with the family's oracle UNet at out_channels = 2 C as the model"""
    family, _, loop, _, clip, eta, _ = CASES[case]
    ucfg, _ = model_config(case)
    sd = random_state_dict(ucfg, 0)
    fwd = {"unetmodel": unetmodel_oracle.unetmodel_forward, "unetconv": unetconv_oracle.unetconv_forward,
           "swin": unet_oracle.unet_forward}[family]
    lq, inputs = case_inputs(case)
    model = lambda x, t, lq=None: fwd(sd, ucfg, x, t, lq=lq)          # noqa: E731
    diff = create_gaussian_diffusion_ddpm(**diffusion_kwargs(case))
    assert diff.model_var_type == V.LEARNED_RANGE and not diff._native_ok(model, None, {"lq": lq})
    if loop == "reverse":
        rec = list(diff.ddim_reverse_sample_loop_progressive(model, inputs, clip_denoised=clip, model_kwargs={"lq": lq}))
    else:
        queue = list(inputs[1:])
        monkeypatch.setattr(torch, "randn_like", lambda ref: queue.pop(0))
        kw = dict(noise=inputs[0], clip_denoised=clip, model_kwargs={"lq": lq}, device="cpu")
        if loop == "ddim":
            rec = list(diff.ddim_sample_loop_progressive(model, tuple(inputs[0].shape), eta=eta, **kw))
        else:
            rec = list(diff.p_sample_loop_progressive(model, tuple(inputs[0].shape), **kw))
        monkeypatch.undo()
        assert not queue
    assert len(rec) == diff.num_timesteps
    _close(rec[-1]["sample"].numpy(), gold[f"{case}/final"], f"{case} final")
    for k, r in enumerate(rec):
        _close(r["sample"].reshape(-1)[::OUT_STRIDE].numpy(), gold[f"{case}/sample/{k}"], f"{case} sample {k}")
        _close(r["pred_xstart"].reshape(-1)[::OUT_STRIDE].numpy(), gold[f"{case}/pred_xstart/{k}"],
               f"{case} pred_xstart {k}")


@pytest.mark.parametrize("case", sorted(CASES))
def test_param_spec_matches_reference_inventory(golden_dir, case):
    ref = json.loads((golden_dir / "ddpm_learned_keys.json").read_text())[case]
    ucfg, _ = model_config(case)
    spec = {"unetmodel": unetmodel_param_spec, "unetconv": unetconv_param_spec, "swin": unet_param_spec}[CASES[case][0]]
    assert {n: list(s) for n, s, _ in spec(ucfg)} == ref


@pytest.mark.parametrize("cls", [UNetModelConfig, UNetModelConvConfig])
def test_constructor_channel_rule(cls):
    extra = dict(attention_resolutions=(), num_head_channels=32) if cls is UNetModelConfig else {}
    # (in, out) -> (channels of x, lq factor)
    for (i, o), (x, f) in {(6, 3): (3, 1), (15, 3): (3, 2), (6, 6): (3, 1), (15, 6): (3, 2), (11, 16): (8, 1),
                           (20, 16): (8, 2), (7, 4): (4, 1)}.items():
        cfg = cls(in_channels=i, out_channels=o, **extra)
        assert (cfg.x_channels, cfg.lq_factor) == (x, f), (i, o)
    # both readings fit (x 18 + lq 3, or x 9 + lq 12 at twice the size): the fixed-variance one wins
    cfg = cls(in_channels=21, out_channels=18, **extra)
    assert (cfg.x_channels, cfg.lq_factor) == (18, 1)
    for i, o in ((7, 3), (7, 6), (9, 5), (5, 3), (6, 2)):
        with pytest.raises(ValueError, match="in_channels"):
            cls(in_channels=i, out_channels=o, **extra)


def test_model_x_channels():
    small = dict(model_channels=32, num_res_blocks=1, channel_mult=(1, 2))
    assert UNetModel(image_size=32, in_channels=15, out_channels=6, attention_resolutions=(), **small).x_channels == 3
    assert UNetModel(image_size=32, in_channels=21, out_channels=18, attention_resolutions=(), **small).x_channels == 18
    assert UNetModelConv(in_channels=6, out_channels=6, **small).x_channels == 3
    swin = UNetConfig(model_channels=32, swin_embed_dim=64, out_channels=6)
    assert UNetModelSwin(**swin.to_kwargs()).x_channels == 3
    m = UNetModel(image_size=32, in_channels=6, out_channels=6, attention_resolutions=(), **small)
    with pytest.raises(ValueError, match="out_channels / 2 = 3"):
        m(torch.zeros(1, 6, 32, 32), torch.zeros(1), lq=torch.zeros(1, 3, 32, 32))
    with pytest.raises(ValueError, match="in_channels"):
        UNetModelConv(in_channels=7, out_channels=3, **small)


def _models():
    """(model, x channels, output channels) of every family, with a C and a 2 C head"""
    small = dict(model_channels=32, num_res_blocks=1, channel_mult=(1, 2))
    out = []
    for o in (3, 6):
        out.append(UNetModel(image_size=32, in_channels=6, out_channels=o, attention_resolutions=(), **small))
        out.append(UNetModelConv(in_channels=6, out_channels=o, **small))
        out.append(UNetModelSwin(**UNetConfig(model_channels=32, swin_embed_dim=64, out_channels=o).to_kwargs()))
    return out


def test_native_gate():
    kw = dict(beta_start=0.0015, beta_end=0.0155, timestep_respacing=8)
    lq = {"lq": torch.zeros(1)}
    for m in _models():
        assert m.x_channels == 3
        learned_head = m.cfg.out_channels == 6
        for var in (V.FIXED_LARGE, V.FIXED_SMALL, V.LEARNED, V.LEARNED_RANGE):
            diff = create_gaussian_diffusion_ddpm(**kw)
            diff.model_var_type = var
            want = (var in (V.LEARNED, V.LEARNED_RANGE)) == learned_head
            assert diff._native_ok(m, None, lq) is want, (type(m).__name__, m.cfg.out_channels, var)
            assert not diff._native_ok(m, lambda v: v, lq)            # denoised_fn stays on the torch route
            assert not diff._native_ok(m, None, {})
    diff = create_gaussian_diffusion_ddpm(learn_sigma=True, **kw)
    assert not diff._native_ok(learned_range_model, None, lq)
    # the nine rows of a LEARNED_RANGE sampler: the eight of ddpm_tables, then log(betas)
    tabs = diff.ddpm_learned_range_tables()
    assert tabs.shape == (9, 8) and diff.ddpm_tables().shape == (8, 8)
    np.testing.assert_array_equal(tabs[:8], diff.ddpm_tables())
    np.testing.assert_array_equal(tabs[8], np.log(diff.betas))
