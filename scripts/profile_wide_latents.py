"""Measures first stages with wide latents and the denoiser on them (synthetic weights).  Prints the card's name and power
limit first.

  * AutoencoderKLTorch encode (posterior sampled with given noise) and decode of LDM's kl-f16 (16-channel latent) and
    kl-f32 (64-channel latent) at 256x256 batch 16 and at 1024x1024 batch 1: CUDA events around `reps` back-to-back
    calls after one warm-up call, median of 3 rounds;
  * the wide latent kernels on their own: pointwise_conv_wide_kernel and kl_posterior_wide_kernel through
    rs_op_pointwise_conv / rs_op_kl_posterior at batch 16, 64x64 latents (CUDA events around 50 x `reps` launches,
    median of 3 rounds), and every wide kernel inside the passes above and inside a VQ decode with a 64-dim, 16384-code
    codebook (torch.profiler's CUDA time per launch; launches overlap the tail of the kernel before them, whose
    remainder this time includes);
  * one denoiser forward (a denoise step) of the realsr UNetModelSwin at batch 16, 64x64 latent, with 16 latent
    channels against the same model with 3, CUDA events as above.

    python scripts/profile_wide_latents.py [reps]
"""
import statistics
import subprocess
import sys
import warnings
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch
from torch.profiler import ProfilerActivity, profile

from resshift_b200 import _lib
from resshift_b200.config import preset
from resshift_b200.models.autoencoder import AutoencoderKLTorch, VQModelTorch
from resshift_b200.models.unet import UNetModelSwin
from resshift_b200.vq_arch import VQConfig, kl_preset, random_kl_state_dict, random_vq_state_dict
from resshift_b200.weights import random_state_dict

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 10
ROUNDS = 3
WIDE = ("pointwise_conv_wide_kernel", "kl_posterior_wide_kernel", "vq_quantize_wide_kernel")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                              # noqa: BLE001 — the name alone still identifies the card
        q = ""
    return q or torch.cuda.get_device_name(0)


def timed(fn):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(ROUNDS):
        e0.record()
        for _ in range(REPS):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / REPS)
    return statistics.median(out)


def kernel_us(fn):
    """{wide kernel name: mean device microseconds per launch} over REPS calls of fn (after a warm-up call)."""
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(REPS):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if any(w in ev.key for w in WIDE):
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            out[ev.key.split("(")[0]] = (t / max(ev.count, 1), ev.count)
    return out


def kernels(tag):
    print(f"\n{tag} wide kernels on their own, batch 16, 64x64 latent positions, {50 * REPS} launches x {ROUNDS} rounds "
          "(median, us per launch)")
    N, HW = 16, 64 * 64
    st = _lib.current_stream()
    for cin, cout in ((16, 16), (64, 64)):
        x = torch.randn(N, cin, HW, device="cuda")
        w = (0.1 * torch.randn(cout, cin, device="cuda")).half()
        b = torch.randn(cout, device="cuda")
        y = torch.empty(N, cout, HW, device="cuda")
        us = 1e3 / 50 * timed(lambda: [_lib.check(_lib.lib.rs_op_pointwise_conv(x.data_ptr(), w.data_ptr(), cin, b.data_ptr(),
                                                                               cin, cout, N, HW, y.data_ptr(), st))
                                       for _ in range(50)])
        print(f"  pointwise_conv_wide_kernel  Cin {cin:>3} -> Cout {cout:>3}: {us:8.2f} us "
              f"({(x.numel() + y.numel()) * 4 / us / 1e3:.0f} GB/s of fp32 in + out)  {tag}")
    for cin, e in ((32, 16), (128, 64)):
        h = torch.randn(N, cin, HW, device="cuda")
        w = (0.1 * torch.randn(2 * e, cin, device="cuda")).half()
        b = torch.randn(2 * e, device="cuda")
        noise = torch.randn(N, e, HW, device="cuda")
        z = torch.empty(N, e, HW, device="cuda")
        mom = torch.empty(N, 2 * e, HW, device="cuda")
        us = 1e3 / 50 * timed(lambda: [_lib.check(_lib.lib.rs_op_kl_posterior(h.data_ptr(), w.data_ptr(), cin, b.data_ptr(), cin, e,
                                                                             noise.data_ptr(), z.data_ptr(), mom.data_ptr(), N,
                                                                             HW, st))
                                       for _ in range(50)])
        nbytes = (h.numel() + noise.numel() + z.numel() + mom.numel()) * 4
        print(f"  kl_posterior_wide_kernel    Cin {cin:>3} -> 2E {2 * e:>3}: {us:8.2f} us "
              f"({nbytes / us / 1e3:.0f} GB/s of fp32 h, noise, z, moments)  {tag}")


def first_stages(tag):
    print(f"\n{tag} KL first stages (synthetic weights), {REPS} calls x {ROUNDS} rounds (median)")
    print(f"{'model':>7} {'image':>10} {'batch':>5} {'latent':>12} {'encode ms':>10} {'decode ms':>10}   "
          "wide kernels in the passes (profiler us per launch)")
    for name in ("f16", "f32"):
        cfg = kl_preset(name)
        m = AutoencoderKLTorch(**cfg.to_kwargs())
        m.load_state_dict(random_kl_state_dict(cfg, 0))
        m = m.cuda().eval()
        f = cfg.downscale
        for hw, b in ((256, 16), (1024, 1)):
            x = torch.rand(b, 3, hw, hw, device="cuda") * 2 - 1
            noise = torch.randn(b, cfg.embed_dim, hw // f, hw // f, device="cuda")
            z = m.encode(x, posterior_noise=noise)
            t_enc = timed(lambda: m.encode(x, posterior_noise=noise))
            t_dec = timed(lambda: m.decode(z))
            k = kernel_us(lambda: (m.encode(x, posterior_noise=noise), m.decode(z)))
            ks = ", ".join(f"{n} {us:.2f}" for n, (us, _) in sorted(k.items()))
            print(f"{'kl-' + name:>7} {hw:>5}x{hw:<4} {b:>5} {cfg.embed_dim:>3}x{hw // f}x{hw // f:<5} {t_enc:>10.2f} "
                  f"{t_dec:>10.2f}   {ks}  {tag}")
            del x, z, noise
            m._plans.clear()
            torch.cuda.empty_cache()
        del m
    # the quantiser: a 64-dim VQ first stage with a 16384-code codebook, f4, 256x256 batch 16 (64x64 latent)
    cfg = VQConfig(embed_dim=64, n_embed=16384, z_channels=64, resolution=256, ch=128, ch_mult=(1, 2, 4), num_res_blocks=2)
    m = VQModelTorch(**cfg.to_kwargs())
    m.load_state_dict(random_vq_state_dict(cfg, 0))
    m = m.cuda().eval()
    z = torch.randn(16, 64, 64, 64, device="cuda") * 0.6
    t_dec = timed(lambda: m.decode(z))
    k = kernel_us(lambda: m.decode(z))
    ks = ", ".join(f"{n} {us:.2f}" for n, (us, _) in sorted(k.items()))
    print(f"{'vq-f4':>7} {'256x256':>10} {16:>5} {'64x64x64':>12} {'':>10} {t_dec:>10.2f}   {ks}  (E = 64, 16384 codes)  {tag}")
    del m, z
    torch.cuda.empty_cache()


def denoiser(tag):
    print(f"\n{tag} denoise step: realsr UNetModelSwin forward (synthetic weights), batch 16, 64x64 latent, "
          f"{REPS} calls x {ROUNDS} rounds (median)")
    base = None
    for c in (3, 16):
        ucfg, _ = preset("realsr")
        ucfg.in_channels = ucfg.out_channels = c
        m = UNetModelSwin(**ucfg.to_kwargs())
        m.load_state_dict(random_state_dict(ucfg, 0))
        m = m.cuda().eval()
        x = torch.randn(16, c, 64, 64, device="cuda")
        lq = torch.rand(16, 3, ucfg.lq_size, ucfg.lq_size, device="cuda") * 2 - 1
        t = torch.full((16,), 7, device="cuda")
        ms = timed(lambda: m(x, t, lq=lq))
        base = base or ms
        print(f"  latent channels {c:>2}: {ms:8.2f} ms per forward ({ms / base:.3f}x the 3-channel model)  {tag}")
        del m, x, lq
        torch.cuda.empty_cache()


def main():
    tag = f"[{card()}]"
    print(f"card: {tag[1:-1]}")
    warnings.filterwarnings("ignore", message=".*Profiler clears events.*")
    with torch.no_grad():
        kernels(tag)
        first_stages(tag)
        denoiser(tag)


if __name__ == "__main__":
    main()
