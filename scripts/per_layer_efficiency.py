"""per-op table (scripts/profile_ops.py) -> per-layer efficiency table in markdown: algorithmic FLOPs / bytes of each layer
shape against the measured peaks (MEASURED_PEAKS.json).  usage: python scripts/per_layer_efficiency.py <per_op_table.log> [batch]"""
import json
import re
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
src = Path(sys.argv[1])
B = int(sys.argv[2]) if len(sys.argv) > 2 else 16
pk = json.loads((ROOT / "MEASURED_PEAKS.json").read_text()) if (ROOT / "MEASURED_PEAKS.json").exists() else {}
TF, GB = float(pk.get("bf16_tflops_sustained", 1427.5)), float(pk.get("hbm_gbs", 6582.5))
rows, total = [], None
for line in src.read_text().splitlines():
    m = re.match(r"ops\s+(\d+)\s+total\s+([\d.]+) ms", line)
    if m:
        total = float(m.group(2)) * 1e3
    m = re.match(r"\s+([\d.]+) us\s+([\d.]+)%\s+n=\s*(\d+)\s+avg\s+([\d.]+)\s+(.*)", line)
    if m:
        rows.append((float(m.group(1)), m.group(2), int(m.group(3)), float(m.group(4)), m.group(5).strip()))
print(f"# Per-layer efficiency, batch {B} (from `{src.name}`)\n")
print(f"Times are CUDA events around each launch of one un-graphed forward (serialised, launch gaps included: the sum is\n"
      f"{total / 1e3:.2f} ms), so the fractions are lower bounds.  GEMM layers: algorithmic FLOPs (real channels) against the measured\n"
      f"sustained bf16 peak ({TF} TFLOP/s).  GroupNorm / attention: algorithmic bytes (one read + one write) against the measured\n"
      f"HBM copy bandwidth ({GB:.0f} GB/s); these tensors are L2-resident, the figure only shows how far a pass is from being\n"
      f"bandwidth-limited at all.\n")
print("| total us | share | n | avg us | layer | TFLOP/s | frac of tensor peak | GB/s | frac of HBM peak |")
print("|---|---|---|---|---|---|---|---|---|")
for tot, share, n, avg, desc in rows:
    fl = by = None
    g = re.search(r"\s(\d+)x(\d+)(\s|$)", desc)
    H, W = (int(g.group(1)), int(g.group(2))) if g else (0, 0)
    px = B * H * W
    if desc.startswith("conv"):
        k = 9 if desc.startswith("conv3x3") else 1
        ci, co = int(re.search(r"Cin=(\d+)", desc).group(1)), int(re.search(r"Cout=(\d+)", desc).group(1))
        st = int(re.search(r"s(\d) ", desc).group(1))
        fl = 2.0 * (px / (st * st)) * k * ci * co
    elif desc.startswith("mlp"):
        E = int(re.search(r"E=(\d+)", desc).group(1))
        fl = 2.0 * px * E * 4 * E * 2
    elif desc.startswith("swin_attn"):
        E = int(re.search(r"E=(\d+)", desc).group(1))
        fl = px * (8.0 * E * E + 256.0 * E)
    elif desc.startswith("attn"):
        E = int(re.search(r"heads=(\d+)", desc).group(1)) * int(re.search(r"head_dim=(\d+)", desc).group(1))
        T = int(re.search(r"window=(\d+)", desc).group(1)) ** 2
        fl = px * 4.0 * T * E
        by = px * (3 * E + E) * 2.0
    elif desc.startswith("gn"):
        C = int(re.search(r"C=(\d+)", desc).group(1))
        by = px * C * 2.0 * 2
    tf = f"{fl / (avg * 1e-6) / 1e12:.0f}" if fl else ""
    ft = f"{fl / (avg * 1e-6) / 1e12 / TF:.2f}" if fl else ""
    gb = f"{by / (avg * 1e-6) / 1e9:.0f}" if by else ""
    fb = f"{by / (avg * 1e-6) / 1e9 / GB:.2f}" if by else ""
    print(f"| {tot:.1f} | {share}% | {n} | {avg:.1f} | {desc} | {tf} | {ft} | {gb} | {fb} |")
