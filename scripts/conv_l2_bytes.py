"""L2 -> shared memory bytes of every conv launch of one denoiser forward at the benchmark shape, computed from the plan
geometry each launch reports (box, channel tile, CTA pairs, sub-tiles), next to its time (CUDA events around every
launch): the achieved operand byte rate per layer family.

A bytes: one 16 KB box per 128-pixel tile, channel tile, tap and 64-channel chunk.  B bytes: one weight tile per
k-block per CTA, per CTA pair (TMA multicast) or per msub sub-tiles.  Rows that TMA zero-fills are counted as loaded."""
import ctypes as C
import re
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch

from resshift_b200 import _lib
from resshift_b200.config import preset
from resshift_b200.models.unet import UNetModelSwin
from resshift_b200.weights import random_state_dict

PAT = re.compile(r"conv(\d)x\d s(\d) (\d+)x(\d+) Cin=(\d+) Cout=(\d+) grid=\d+ BN=(\d+) st=\d+ \S+ cg=(\d) ms=(\d) sk=(\d+) "
                 r"box=(\d+)x(\d+)x(\d+)")


def conv_bytes(desc, batch):
    k, s, H, W, cin, cout, BN, cg, ms, sk, bw, bh, bn = map(int, PAT.match(desc).groups())
    m_tiles = (W // bw) * (H // bh) * ((batch + bn - 1) // bn)
    n_tiles = -(-((cout + 15) // 16 * 16) // BN)
    kblocks = k * k * -(-cin // 64)
    a = m_tiles * n_tiles * kblocks * 128 * 128
    b = -(-m_tiles // (cg * ms)) * n_tiles * kblocks * BN * 128
    return f"conv{k}x{k} s{s} {H}x{W} Cin={cin} Cout={cout}", a, b, f"BN={BN} cg={cg} ms={ms} sk={sk} box={bw}x{bh}x{bn}"


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 16
    ucfg, _ = preset("realsr")
    m = UNetModelSwin(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 0))
    m = m.cuda().eval()
    x = torch.randn(B, 3, 64, 64, device="cuda")
    lq = torch.rand(B, 3, 64, 64, device="cuda") * 2 - 1
    t = torch.full((B,), 7.0, device="cuda")
    plan = m.plan(B, 64, 64)
    m(x, t, lq=lq)
    cap, stride = 1024, 160
    ms = (C.c_double * cap)()
    desc = C.create_string_buffer(cap * stride)
    n = C.c_int32()
    for _ in range(3):
        _lib.check(_lib.lib.rs_plan_profile_ops(plan.handle, x.data_ptr(), t.data_ptr(), lq.data_ptr(), None, ms, desc, stride,
                                                cap, C.byref(n), _lib.current_stream()))
    agg = {}
    for i in range(n.value):
        d = desc.raw[i * stride:(i + 1) * stride].split(b"\0")[0].decode()
        if not d.startswith("conv"):
            continue
        key, a, b, cfg = conv_bytes(d, B)
        e = agg.setdefault((key, cfg), [0, 0.0, 0, 0])
        e[0] += 1; e[1] += ms[i] * 1e3; e[2] += a; e[3] += b
    print(f"batch {B}: {sum(e[0] for e in agg.values())} conv launches, {sum(e[1] for e in agg.values()):.1f} us")
    print(f"{'us':>8} {'n':>3} {'A MB':>8} {'B MB':>8} {'GB/s':>7}  layer / config")
    for (key, cfg), (cnt, us, a, b) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"{us:8.1f} {cnt:3d} {a / 1e6:8.1f} {b / 1e6:8.1f} {(a + b) / us / 1e3:7.0f}  {key}  {cfg}")


if __name__ == "__main__":
    main()
