"""Times the fused VQ-GAN attention kernel (rs_op_vq_attention, csrc/vq_attn.cuh) and puts it next to the GEMM +
row-softmax form the plans use up to 8192 positions and next to a whole large-image encode + decode.

    python scripts/profile_vq_attention.py [--iters 20]

Prints, with the card name and power limit of the run:
  * the fused kernel at C = 512, T in {4096, 16384, 65536}, batch 1 and 4: CUDA events over --iters launches after a
    warm-up, TFLOP/s from 4 T^2 C per image;
  * at T = 4096, the summed per-launch time of the current form's attention ops (the three per-image GEMMs and the row
    softmax between the GroupNorm and proj_out of the encoder's AttnBlock) of a 256x256 f4 encode plan
    (rs_vq_profile_ops);
  * f4 encode + decode of one 1024x1024 image (a 256x256 bottleneck, T = 65536) and the share of it spent in the two
    fused attention launches.
"""
import argparse
import ctypes as C
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch

from resshift_b200 import _lib
from resshift_b200.models.autoencoder import VQModelTorch
from resshift_b200.vq_arch import random_vq_state_dict, vq_preset


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        q = f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"
    return q


def events(fn, iters):
    fn(); fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def op_time(N, T, Cc, iters):
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, v = (torch.randn(N, T, Cc, device="cuda", generator=g).half() for _ in range(3))
    out = torch.empty_like(q)
    st = _lib.current_stream()
    f = lambda: _lib.check(_lib.lib.rs_op_vq_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), N, T, Cc, Cc, out.data_ptr(), st))
    return events(f, iters)


def profile_rows(plan):
    cap, stride = 1024, 160
    ms = (C.c_double * cap)()
    desc = C.create_string_buffer(cap * stride)
    n = C.c_int32()
    for _ in range(3):
        _lib.check(_lib.lib.rs_vq_profile_ops(plan.handle, ms, desc, stride, cap, C.byref(n), _lib.current_stream()))
    return [(ms[i], desc.raw[i * stride:(i + 1) * stride].split(b"\0")[0].decode()) for i in range(n.value)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profile_vq_attention.py needs a CUDA device")
    print(f"card: {card()}")
    Cc = 512
    print(f"== fused attention kernel, C = {Cc} (CUDA events, {a.iters} launches after warm-up)")
    for T in (4096, 16384, 65536):
        for N in (1, 4):
            ms = op_time(N, T, Cc, a.iters)
            print(f"vq_attn T={T:6d} N={N}: {ms:9.3f} ms  {4.0 * T * T * Cc * N / ms / 1e9:7.1f} TFLOP/s")

    cfg = vq_preset("f4")
    m = VQModelTorch(**cfg.to_kwargs())
    m.load_state_dict(random_vq_state_dict(cfg, 0), strict=True)
    m = m.cuda().eval()
    x = torch.rand(1, 3, 256, 256, device="cuda") * 2 - 1
    m.encode(x)
    rows = profile_rows(m.plan(0, 1, 256, 256))
    # the encoder's AttnBlock: after its GroupNorm "encoder.mid.attn_1.norm" come q, k, then per image V^T, S, softmax, PV
    i0 = next(i for i, (_, d) in enumerate(rows) if "encoder.mid.attn_1.norm" in d)
    i1 = next(i for i, (_, d) in enumerate(rows) if "encoder.mid.attn_1.proj_out" in d)
    attn = rows[i0 + 3:i1]
    print(f"== current form at T = 4096 (f4 256x256 encode plan, batch 1): {len(attn)} launches, "
          f"{sum(t for t, _ in attn):.3f} ms summed per-launch time (without the q / k convs)")
    for t, d in attn:
        print(f"   {t:8.3f} ms  {d}")

    x = torch.rand(1, 3, 1024, 1024, device="cuda") * 2 - 1
    z = m.encode(x)
    m.decode(z)
    enc = events(lambda: m.encode(x), 5)
    dec = events(lambda: m.decode(z), 5)
    att = sum(t for t, d in profile_rows(m.plan(0, 1, 1024, 1024)) + profile_rows(m.plan(1, 1, 1024, 1024)) if d.startswith("vq_attn"))
    print(f"== f4 1024x1024 (T = 65536): encode {enc:.3f} ms + decode {dec:.3f} ms = {enc + dec:.3f} ms; "
          f"the two fused attention launches {att:.3f} ms = {100 * att / (enc + dec):.1f} %")


if __name__ == "__main__":
    main()
