"""Host-side pieces of the device pool (ResShiftSampler(devices=...) / RS_DEVICES): parsing the device list and the
refusals — a pool inside a multi-process run, a configuration that takes the generic per-step route, and devices that
differ in SM count or compute capability."""
from types import SimpleNamespace

import pytest

from resshift_b200.device_pool import check_identical_devices, parse_devices, pool_devices
from resshift_b200.sampler import ResShiftSampler

H100 = SimpleNamespace(name="NVIDIA H100 80GB HBM3", multi_processor_count=132, major=9, minor=0)
H100_PCIE = SimpleNamespace(name="NVIDIA H100 PCIe", multi_processor_count=114, major=9, minor=0)
A100 = SimpleNamespace(name="NVIDIA A100-SXM4-80GB", multi_processor_count=108, major=8, minor=0)


def _props(table):
    return lambda i: table[i]


@pytest.mark.parametrize("spec,count,expected", [
    ("all", 8, list(range(8))),
    ("ALL", 1, [0]),
    (" all ", 2, [0, 1]),
    ("0,2,3", 4, [0, 2, 3]),
    ("3, 1", 4, [3, 1]),
    ("0,0,0", 1, [0, 0, 0]),          # one replica per entry: a virtual pool on one GPU
    ("1", 2, [1]),
    (2, 3, [2]),
    ([1, 0], 2, [1, 0]),
    (("0", "1"), 2, [0, 1]),
])
def test_parse_devices(spec, count, expected):
    assert parse_devices(spec, count) == expected


@pytest.mark.parametrize("spec,count,match", [
    ("all", 0, "no CUDA device"),
    ("2", 2, "only 2 CUDA device"),
    ("-1", 2, "only 2 CUDA device"),
    ("0,x", 2, "comma-separated"),
    ("0;1", 2, "comma-separated"),
    ("0,,1", 2, "comma-separated"),
    ([], 2, "at least one"),
])
def test_parse_devices_rejects(spec, count, match):
    with pytest.raises(ValueError, match=match):
        parse_devices(spec, count)


def test_parse_devices_takes_torch_devices():
    import torch
    assert parse_devices([torch.device("cuda", 1), torch.device("cuda:0")], 2) == [1, 0]
    with pytest.raises(ValueError, match="CUDA device with an index"):
        parse_devices([torch.device("cpu")], 2)
    with pytest.raises(ValueError, match="CUDA device with an index"):
        parse_devices([torch.device("cuda")], 2)


def test_rs_devices_unset_or_empty_means_no_pool():
    props = _props([H100] * 8)
    assert pool_devices(None, environ={}, device_count=8, properties=props) is None
    assert pool_devices(None, environ={"RS_DEVICES": ""}, device_count=8, properties=props) is None
    assert pool_devices(None, environ={"RS_DEVICES": "  "}, device_count=8, properties=props) is None
    assert pool_devices([], environ={"RS_DEVICES": "all"}, device_count=8, properties=props) is None
    assert pool_devices("", environ={"RS_DEVICES": "all"}, device_count=8, properties=props) is None


def test_rs_devices_is_read_when_devices_is_none():
    props = _props([H100] * 8)
    assert pool_devices(None, environ={"RS_DEVICES": "all"}, device_count=8, properties=props) == list(range(8))
    assert pool_devices(None, environ={"RS_DEVICES": "0,2,3"}, device_count=8, properties=props) == [0, 2, 3]
    # an explicit argument wins over the variable
    assert pool_devices("5", environ={"RS_DEVICES": "all"}, device_count=8, properties=props) == [5]


def test_pool_refused_under_world_size_above_one():
    props = _props([H100] * 8)
    with pytest.raises(ValueError, match="WORLD_SIZE > 1"):
        pool_devices(None, environ={"RS_DEVICES": "all", "WORLD_SIZE": "2"}, device_count=8, properties=props)
    with pytest.raises(ValueError, match="WORLD_SIZE > 1"):
        pool_devices("0,1", environ={"WORLD_SIZE": "8"}, device_count=8, properties=props)
    # no pool asked for: nothing to refuse; WORLD_SIZE=1 is a one-process run
    assert pool_devices(None, environ={"WORLD_SIZE": "2"}, device_count=8, properties=props) is None
    assert pool_devices("0,1", environ={"WORLD_SIZE": "1"}, device_count=8, properties=props) == [0, 1]


def test_sampler_refuses_a_pool_under_torchrun_before_any_work(monkeypatch):
    """The refusal comes first in the constructor: no process group, no device and no model are touched."""
    monkeypatch.setenv("WORLD_SIZE", "2")
    monkeypatch.setenv("LOCAL_RANK", "0")
    with pytest.raises(ValueError, match="WORLD_SIZE > 1"):
        ResShiftSampler(None, devices="0,1")
    monkeypatch.setenv("RS_DEVICES", "all")
    with pytest.raises(ValueError, match="WORLD_SIZE > 1"):
        ResShiftSampler(None)


def test_mismatched_devices_are_refused():
    check_identical_devices([0, 1, 2], _props([H100, H100, H100]))
    check_identical_devices([1, 1], _props([A100, H100]))                  # only the listed devices count
    with pytest.raises(ValueError, match=r"identical devices.*132 SMs.*114 SMs"):
        check_identical_devices([0, 1], _props([H100, H100_PCIE]))
    with pytest.raises(ValueError, match=r"compute capability 9\.0.*compute capability 8\.0"):
        check_identical_devices([1, 0], _props([A100, H100]))
    with pytest.raises(ValueError, match="identical devices"):
        pool_devices("all", environ={}, device_count=3, properties=_props([H100, H100, H100_PCIE]))


def test_generic_route_is_refused_for_a_pool():
    """Without an autoencoder (or with a model other than this package's UNetModelSwin) the sampler takes the generic
    per-step route, whose noise is drawn inside the loop: it cannot be drawn ahead in one-GPU order."""
    from resshift_b200.config import preset
    from resshift_b200.models.script_util import create_gaussian_diffusion
    _, dcfg = preset("tiny")
    s = ResShiftSampler.__new__(ResShiftSampler)
    s.base_diffusion = create_gaussian_diffusion(**dcfg.to_kwargs())
    s.model, s.autoencoder, s.devices = object(), None, [0, 0]
    with pytest.raises(RuntimeError, match="a device pool needs the fused sampling loop.*generic per-step route"):
        s._build_pool()
