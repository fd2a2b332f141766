"""Pins the oracle to the reference for the UNetModelSwin constructor options the shipped yaml files leave at one value
(use_scale_shift_norm=False, resblock_updown, conv_resample=False, patch_norm, cond_mask with lq_size == image_size,
dropout > 0), and the package's inventory to the reference's ``state_dict`` for each.  The fixtures were recorded from
the unmodified reference by oracle/make_golden_variants.py.  CPU only."""
import json

import numpy as np
import pytest
import torch

from oracle import diffusion_oracle as do
from oracle import unet_variants_oracle as uo
from oracle.make_golden_variants import (OUT_STRIDE, PROBE_STRIDE, VARIANTS, trajectory_inputs, variant_config,
                                         variant_inputs)
from resshift_b200.arch import unet_param_spec
from resshift_b200.weights import random_state_dict

TOL = 2e-4   # fp32 CPU vs fp32 CPU, different op order


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(golden_dir / "unet_variants.npz")


@pytest.mark.parametrize("tag", list(VARIANTS) + ["combined_64x128"])
def test_oracle_forward_matches_reference(gold, tag):
    name = tag.split("_64x128")[0]
    ucfg, _ = variant_config(name)
    sd = random_state_dict(ucfg, 0)
    seed, h, w = (int(v) for v in gold[f"{tag}/seed"])
    x, lq, mask = variant_inputs(ucfg, 2, h, w, seed)
    probes = {}
    out = uo.unet_forward(sd, ucfg, x, torch.from_numpy(gold[f"{tag}/t"]), lq=lq, mask=mask, probes=probes)
    assert np.abs(out.reshape(-1)[::OUT_STRIDE].numpy() - gold[f"{tag}/out_sub"]).max() < TOL
    keys = [k for k in gold.files if k.startswith(f"{tag}/probe_sub/")]
    assert len(keys) == len(probes)
    for k in keys:
        got = probes[k.split("/probe_sub/")[1]].reshape(-1)[::PROBE_STRIDE].numpy()
        assert np.abs(got - gold[k]).max() < TOL * max(1.0, np.abs(gold[k]).max()), k


def test_oracle_loop_matches_reference(gold):
    ucfg, dcfg = variant_config("combined")
    sd = random_state_dict(ucfg, 0)
    y, noises = trajectory_inputs(2, dcfg.steps)
    tabs = do.schedule_tables(do.eta_schedule(dcfg.steps, dcfg.min_noise_level, dcfg.etas_end, dcfg.kappa,
                                              dcfg.schedule_kwargs["power"]), dcfg.kappa)
    final = do.p_sample_loop(lambda xx, tt: uo.unet_forward(sd, ucfg, xx, tt, lq=y), y, list(noises), tabs, dcfg.kappa)
    assert np.abs(final.reshape(-1)[::OUT_STRIDE].numpy() - gold["loop/final_sub"]).max() < TOL


@pytest.mark.parametrize("name", ["tiny", "tiny_inpaint"])
def test_variants_oracle_equals_shipped_oracle_on_shipped_topologies(name):
    """For the shipped options the variants oracle computes exactly what oracle/unet_oracle.py does."""
    from oracle import unet_oracle
    from resshift_b200.config import preset
    ucfg, _ = preset(name)
    sd = random_state_dict(ucfg, 0)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 3, 64, 64, generator=g)
    hw = 64 << ucfg.fe_stages
    lq = torch.rand(2, 3, hw, hw, generator=g) * 2 - 1
    mask = torch.ones(2, 1, hw, hw) if ucfg.cond_mask else None
    t = torch.tensor([3, 1])
    assert torch.equal(uo.unet_forward(sd, ucfg, x, t, lq=lq, mask=mask),
                       unet_oracle.unet_forward(sd, ucfg, x, t, lq=lq, mask=mask))


@pytest.mark.parametrize("name", list(VARIANTS))
def test_param_spec_matches_reference_inventory(golden_dir, name):
    ref = json.loads((golden_dir / "unet_keys_variants.json").read_text())[name]
    ucfg, _ = variant_config(name)
    mine = {n: list(s) for n, s, _ in unet_param_spec(ucfg)}
    assert mine == ref


@pytest.mark.parametrize("kwargs,why", [
    (dict(cond_lq=False), "cond_lq"),
    (dict(dims=1), "dims"),
    (dict(window_size=4), "window_size"),
    (dict(num_head_channels=16), "head dim"),
])
def test_constructor_refuses_uncovered_options(kwargs, why):
    from resshift_b200.models.unet import UNetModelSwin
    ucfg, _ = variant_config("combined")
    args = {**ucfg.to_kwargs(), **kwargs}
    with pytest.raises(ValueError, match=why):
        UNetModelSwin(**args)
