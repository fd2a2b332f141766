"""Measures a realsr-width UNetModelConv on the native kernels and the cost of the conv epilogue's SiLU output.
Prints the card's name, power limit and maximum SM clock first.

  * the per-launch table of one forward (rs_plan_profile_ops: CUDA events around every op) of a UNetModelConv with
    model_channels 160, channel_mult (1, 2, 2, 4), num_res_blocks 2, in 6 / out 3 (synthetic weights), batch 16, 64x64
    latent, and the ms per 15-step fused loop (CUDA graph replay) at the same shape;
  * the 64x64 160 -> 160 3x3 conv at batch 16 (the top level's out_layers conv: residual, fp16 output) launched by
    rs_op_conv2d_ex with and without silu_out, CUDA events around `reps` launches, median of 3 rounds.

    python scripts/profile_unetconv.py [reps]
"""
import ctypes as C
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch

from resshift_b200 import _lib
from resshift_b200.config import DiffusionConfig, UNetModelConvConfig
from resshift_b200.models.script_util import create_gaussian_diffusion
from resshift_b200.models.unet import UNetModelConv
from resshift_b200.weights import random_state_dict

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 50
B, HW, STEPS = 16, 64, 15


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                              # noqa: BLE001 — the name alone still identifies the card
        q = ""
    return q or torch.cuda.get_device_name(0)


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(3):
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / reps)
    return statistics.median(out)


def per_launch_table(m):
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(B, 3, HW, HW, device="cuda", generator=g)
    lq = torch.rand(B, 3, HW, HW, device="cuda", generator=g) * 2 - 1
    t = torch.full((B,), 7.0, device="cuda")
    m(x, t, lq=lq)
    plan = m.plan(B, HW, HW)
    cap, stride = 1024, 256
    ms, desc, n = (C.c_double * cap)(), C.create_string_buffer(cap * stride), C.c_int32()
    _lib.check(_lib.lib.rs_plan_profile_ops(plan.handle, x.data_ptr(), t.data_ptr(), lq.data_ptr(), None, ms, desc, stride, cap,
                                            C.byref(n), _lib.current_stream()))
    rows = [(ms[i], desc.raw[i * stride:(i + 1) * stride].split(b"\0")[0].decode()) for i in range(n.value)]
    total = sum(r[0] for r in rows)
    print(f"per-launch table of one forward (batch {B}, {HW}x{HW}): {len(rows)} ops, {total:.3f} ms summed")
    print(f"{'#':>4} {'ms':>8}  op")
    for i, (t_ms, d) in enumerate(rows):
        print(f"{i:>4} {t_ms:>8.4f}  {d}")
    kinds = {}
    for t_ms, d in rows:
        k = d.split()[0] + (" +silu" if "silu=1" in d else "") + (" +film" if "film=1" in d else "")
        kinds[k] = kinds.get(k, 0.0) + t_ms
    for k, v in sorted(kinds.items(), key=lambda kv: -kv[1]):
        print(f"  {k:<20} {v:8.3f} ms")


def loop_ms(m):
    diff = create_gaussian_diffusion(**DiffusionConfig(steps=STEPS).to_kwargs())
    g = torch.Generator(device="cuda").manual_seed(0)
    y = torch.rand(B, 3, HW, HW, device="cuda", generator=g) * 2 - 1
    noises = torch.randn(STEPS + 1, B, 3, HW, HW, device="cuda", generator=g)
    return timed(lambda: diff.sample_latent(y, m, {"lq": y}, noises=noises), max(2, REPS // 10)), m.num_launches(B, HW, HW)


def silu_out_cost():
    g = torch.Generator(device="cuda").manual_seed(1)
    Cc = 160
    x = torch.randn(B, HW, HW, Cc, device="cuda", generator=g).half()
    res = torch.randn(B, HW, HW, Cc, device="cuda", generator=g).half()
    w = torch.randn(Cc, Cc, 3, 3, device="cuda", generator=g) / (9 * Cc) ** 0.5
    wp = torch.empty(Cc * 9 * Cc, dtype=torch.float16, device="cuda")
    _lib.check(_lib.lib.rs_op_pack_conv_weight(w.data_ptr(), wp.data_ptr(), Cc, Cc, 3, 3, Cc, _lib.current_stream()))
    bias = torch.randn(Cc, device="cuda", generator=g)
    out, silu = torch.empty_like(x), torch.empty_like(x)
    info = (C.c_int32 * 12)()

    def args(with_silu):
        a = _lib.ConvArgsC()
        a.x, a.N, a.H, a.W, a.C, a.ld = x.data_ptr(), B, HW, HW, Cc, Cc
        a.w_packed, a.ipad, a.bias, a.cout, a.ksize, a.stride, a.pad_lo = wp.data_ptr(), Cc, bias.data_ptr(), Cc, 3, 1, 1
        a.residual, a.res_ld, a.out, a.out_ld = res.data_ptr(), Cc, out.data_ptr(), Cc
        if with_silu:
            a.silu_out, a.silu_ld = silu.data_ptr(), Cc
        return a

    st = _lib.current_stream()
    for with_silu in (False, True):
        a = args(with_silu)
        ms = timed(lambda: _lib.check(_lib.lib.rs_op_conv2d_ex(C.byref(a), info, st)), REPS)
        cfg = dict(zip(("grid", "BN", "msub", "stages", "cg", "splitk", "persist", "epi_bc"), list(info)[:8]))
        moved = B * HW * HW * Cc * 2 * (3 + int(with_silu))          # x, residual, out (+ silu_out) bytes, once each
        print(f"conv3x3 {HW}x{HW} {Cc}->{Cc} batch {B}, residual, silu_out={int(with_silu)}: {ms * 1e3:8.1f} us "
              f"({moved / ms / 1e6:.0f} GB/s of unique activation bytes), config {cfg}")


def main():
    print(f"card (name, power limit, max SM clock): {card()}")
    ucfg = UNetModelConvConfig(in_channels=6, model_channels=160, out_channels=3, num_res_blocks=2, channel_mult=(1, 2, 2, 4))
    m = UNetModelConv(**ucfg.to_kwargs())
    m.load_state_dict(random_state_dict(ucfg, 0))
    m = m.cuda().eval()
    per_launch_table(m)
    ms, n = loop_ms(m)
    print(f"UNetModelConv realsr width, batch {B}, {HW}x{HW} latent, {STEPS}-step fused loop: {ms:.2f} ms per loop, "
          f"{ms / STEPS:.3f} ms per denoise step, {n} launches per forward")
    silu_out_cost()


if __name__ == "__main__":
    main()
