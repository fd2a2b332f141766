"""Times the KL first stage (AutoencoderKLTorch, the SD-style f8 configuration, synthetic weights) on one GPU: encode
(sampling the posterior with given noise) and decode at 256x256, 1024x1024 and 2048x2048, batch 1, CUDA events around
`reps` back-to-back calls after one warm-up call, median of `rounds`.  Prints the card's name and power limit first.

    python scripts/profile_kl.py [reps] [rounds]
"""
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch

from resshift_b200.models.autoencoder import AutoencoderKLTorch
from resshift_b200.vq_arch import kl_preset, random_kl_state_dict

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 5
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 3


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


def main():
    cfg = kl_preset("f8")
    m = AutoencoderKLTorch(**cfg.to_kwargs())
    m.load_state_dict(random_kl_state_dict(cfg, 0))
    m = m.cuda().eval()
    f = cfg.downscale
    print(f"card: {card()}; KL f8 (ch 128, ch_mult 1-2-4-4, z = embed = 4), batch 1, {REPS} calls x {ROUNDS} rounds (median)")
    print(f"{'image':>10} {'latent':>9} {'T':>6} {'attention':>9} {'encode ms':>10} {'decode ms':>10}")
    for hw in (256, 1024, 2048):
        x = torch.rand(1, 3, hw, hw, device="cuda") * 2 - 1
        noise = torch.randn(1, cfg.embed_dim, hw // f, hw // f, device="cuda")
        z = m.encode(x, posterior_noise=noise)
        t_enc = timed(lambda: m.encode(x, posterior_noise=noise))
        t_dec = timed(lambda: m.decode(z))
        fused = m.plan(0, 1, hw, hw).attention is not None
        print(f"{hw:>5}x{hw:<4} {hw // f:>4}x{hw // f:<4} {(hw // f) ** 2:>6} {'fused' if fused else 'gemm':>9} "
              f"{t_enc:>10.2f} {t_dec:>10.2f}")
        del x, z
        m._plans.clear()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
