"""The first stage's row softmax (rs_op_softmax_rows) and the probes of its GEMM-form attention blocks as the GPU tests
drive them, with the row softmax's float64 reference and allowance (test_gpu_first_stage_kernels.py's module docstring,
a)."""
import os
from contextlib import contextmanager

import torch

from resshift_b200 import _lib
from tests import gpu_util as G

U16, U32, R32, S16 = 2.0 ** -11, 2.0 ** -23, 2.0 ** -24, 2.0 ** -25
FTZ = 2.0 ** -126
SM_CLASSES = ("randn", "uniform", "equal", "peaked", "gap")


def f32(x):
    """x rounded to fp32, as a Python float."""
    return torch.tensor(x, dtype=torch.float32).item()


def softmax_allowance(z, cols):
    """float64 softmax of the logits z [rows, cols] and its per-element allowance."""
    m = z.amax(-1, keepdim=True)
    d = z - m
    e = torch.exp(d)
    p = e / e.sum(-1, keepdim=True)
    rho = (z.abs() + d.abs()) * R32 + (2 + 1.173 * d.abs()) * U32
    n_l = 8 * -(-cols // 2048) + 12
    rel = torch.expm1(rho + (p * rho).sum(-1, keepdim=True) + (n_l + 2) * R32)
    return p, rel


def peak_columns(cols):
    """The first and last column, and one column in the range of every warp of every 16-byte vector a thread holds."""
    out = [0, cols - 1]
    for i in range(4):
        for w in range(8):
            start = 2048 * i + 256 * w
            if start < cols:
                out.append(min(start + (37 * (8 * i + w)) % 256, cols - 1))
    return out


def score_rows(rows, cols, scale, seed):
    """fp16 S [rows][cols] and the input class of each row."""
    g = G.gen(seed)
    z = torch.empty(rows, cols, device="cuda")
    peaks = peak_columns(cols)
    classes = ["peaked"] if rows == 1 else [SM_CLASSES[r % len(SM_CLASSES)] for r in range(rows)]
    counts = {"peaked": 0, "gap": 0}
    for cls in SM_CLASSES:
        idx = [r for r in range(rows) if classes[r] == cls]
        if not idx:
            continue
        sel = torch.tensor(idx, device="cuda")
        n = len(idx)
        if cls == "randn":
            z[sel] = 3 * torch.randn(n, cols, device="cuda", generator=g)
        elif cls == "uniform":
            z[sel] = 1e-3 * torch.randn(n, cols, device="cuda", generator=g)
        elif cls == "equal":
            z[sel] = 0.7
        else:
            lo, hi, top = (-40.0, 30.0, 40.0) if cls == "peaked" else (-55.0, -45.0, 50.0)
            z[sel] = lo + (hi - lo) * torch.rand(n, cols, device="cuda", generator=g)
            pos = torch.tensor([peaks[(counts[cls] + k) % len(peaks)] for k in range(n)], device="cuda")
            z[sel, pos] = top
            counts[cls] += n
    return (z / scale).half(), classes


def run_softmax(s, rows, cols, ld, scale):
    """rs_op_softmax_rows in place on the fp16 [rows][ld] buffer s."""
    _lib.check(_lib.lib.rs_op_softmax_rows(s.data_ptr(), rows, cols, ld, scale, G.stream()))
    torch.cuda.synchronize()


def softmax_case(rows, cols, ld):
    """rs_op_softmax_rows on rows x cols scores of every class in an fp16 [rows][ld] buffer, against float64.  Returns
    the worst ratio to the bound, and per input class the worst ratio of the accumulation error to the allowance."""
    scale = f32((64, 128, 512)[cols % 3] ** -0.5)
    s, classes = score_rows(rows, cols, scale, seed=cols * 7 + rows)
    sentinel = 1234.0
    buf = torch.full((rows, ld), sentinel, dtype=torch.float16, device="cuda")
    buf[:, :cols] = s
    run_softmax(buf, rows, cols, ld, scale)
    assert (buf[:, cols:] == sentinel).all(), "columns beyond cols were written"
    again = torch.full_like(buf, sentinel)
    again[:, :cols] = s
    run_softmax(again, rows, cols, ld, scale)
    assert torch.equal(G.bits(again), G.bits(buf)), "not bit-reproducible"
    step = max(1, (1 << 23) // cols)
    cls_t = torch.tensor([SM_CLASSES.index(c) for c in classes], device="cuda")
    worst, per_class = 0.0, {}
    for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        p, rel = softmax_allowance(s[r0:r1].double() * scale, cols)
        got = buf[r0:r1, :cols]
        allow = p * rel + FTZ
        tag = f"softmax cols={cols} rows={rows} ld={ld} rows {r0}:{r1}"
        worst = max(worst, G.assert_within(tag, got, p, allow, 1.0))
        for ci, cls in enumerate(SM_CLASSES):
            sel = cls_t[r0:r1] == ci
            if sel.any():
                G.note(per_class, cls, G.accumulation_ratio(got[sel], p[sel], allow[sel]))
    return worst, per_class


@contextmanager
def no_reuse():
    """Plans created inside keep every tensor alive for rs_plan_probe."""
    old = os.environ.get("RS_NO_REUSE")
    os.environ["RS_NO_REUSE"] = "1"
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("RS_NO_REUSE", None)
        else:
            os.environ["RS_NO_REUSE"] = old


def tokens(t):
    """[N, C, H, W] -> [N, T, C] float64."""
    return t.flatten(2).transpose(1, 2).double()


def w16(sd, name, cc):
    return sd[name].reshape(cc, -1).cuda().half().double()
