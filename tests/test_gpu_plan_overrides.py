"""The kernel-choice overrides of the environment (INTEGRATION.md) are read once, when a plan is created: a plan bound
after the variable changed has the layout and the launches of a plan created and bound entirely under it.  Host-side
only: plans are created and bound (tensor maps, function attributes), no forward runs."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from resshift_b200 import _lib
from resshift_b200.config import preset

B, H, W = 16, 64, 64      # the benchmark's batch and latent size


@pytest.fixture(scope="module")
def engine():
    from resshift_b200.models.unet import UNetModelSwin
    ucfg, _ = preset("realsr")
    m = UNetModelSwin(**ucfg.to_kwargs())
    h = m._ensure_engine(torch.device("cuda", torch.cuda.current_device()))
    yield h
    del m


def _create(engine):
    h = C.c_void_p()
    _lib.check(_lib.lib.rs_plan_create(engine, B, H, W, C.byref(h)))
    return h


def _bind(h):
    """(workspace bytes, launches) of plan h bound on a fresh workspace."""
    nbytes = _lib.lib.rs_plan_workspace_bytes(h)
    ws = torch.empty(nbytes + 256, dtype=torch.uint8, device="cuda")
    _lib.check(_lib.lib.rs_plan_bind(h, (ws.data_ptr() + 255) // 256 * 256))
    return nbytes, _lib.lib.rs_plan_num_launches(h)


@pytest.mark.parametrize("var,value", [("RS_CONV_IMPL", "simt"), ("RS_CONV_SPLITK", "2"), ("RS_SWIN_FUSE_MIN_PAIRS", "1")])
def test_plan_keeps_the_overrides_it_was_created_with(engine, monkeypatch, var, value):
    monkeypatch.delenv(var, raising=False)
    plans = {"default": _create(engine)}
    try:
        default = _bind(plans["default"])
        monkeypatch.setenv(var, value)
        plans["whole"], plans["mixed"] = _create(engine), _create(engine)
        whole = _bind(plans["whole"])
        monkeypatch.delenv(var)
        mixed = _bind(plans["mixed"])
        assert whole != default, f"{var}={value} changes nothing at this shape"
        assert mixed == whole, (var, value, mixed, whole)
    finally:
        for h in plans.values():
            _lib.lib.rs_plan_destroy(h)
