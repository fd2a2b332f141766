"""Generate tests/golden/image_splitter.json by running the UNMODIFIED reference ImageSpliterTh.

    RESSHIFT_REFERENCE=<reference checkout> python -m oracle.make_golden_splitter

Records, for the (size, patch, stride) grid and the tiled-pass shapes tests/test_cpu_boundary.py checks, the tile starts
and the batches (tile origins and patch shapes) that iterating ImageSpliterTh(extra_bs=...) yields
(utils/util_image.py:889-979).  Nothing here copies reference source; it only imports and executes it.
"""
from __future__ import annotations

import json
import os
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
REF = Path(os.environ.get("RESSHIFT_REFERENCE", "/root/reference"))
GOLD = ROOT / "tests" / "golden"

SIZES = list(range(1, 70)) + [100, 127, 128, 129, 200, 255, 256, 257, 300, 448, 500, 592, 1000]
PATCH_STRIDES = [(16, 16), (16, 12), (32, 28), (64, 64), (128, 112), (256, 224)]
PLANS = [(75, 50, 32, 28, 4, 1), (148, 112, 128, 112, 4, 3), (64, 200, 64, 48, 4, 8),
         (40, 40, 64, 48, 4, 2), (592 // 4, 448 // 4, 128, 112, 4, 4), (512, 700, 256, 224, 1, 5)]


def main() -> None:
    sys.path[:0] = [str(ROOT / "oracle" / "_shims"), str(REF)]
    from utils.util_image import ImageSpliterTh                     # noqa: E402  (reference)
    starts = []
    for n in SIZES:
        for ps, st in PATCH_STRIDES:
            sp = ImageSpliterTh(torch.zeros(1, 1, n, max(n // 2, 1)), ps, st, sf=1)
            starts.append([n, ps, st, sp.height_starts_list, sp.width_starts_list])
    plans = []
    for (h, w, ps, st, sf, bs) in PLANS:
        sp = ImageSpliterTh(torch.zeros(2, 3, h, w), ps, st, sf=sf, extra_bs=bs)
        groups, shapes = [], []
        for pch, idx in sp:
            groups.append([[i[0] // sf, i[2] // sf] for i in idx])
            shapes.append([pch.shape[0], pch.shape[2], pch.shape[3]])
        plans.append({"args": [h, w, ps, st, sf, bs], "groups": groups, "shapes": shapes,
                      "height_starts": sp.height_starts_list, "width_starts": sp.width_starts_list})
    out = {"source": "utils/util_image.py ImageSpliterTh of zsyOAOA/ResShift @ 3ce1d81e", "starts": starts, "plans": plans}
    (GOLD / "image_splitter.json").write_text(json.dumps(out, separators=(",", ":")))


if __name__ == "__main__":
    main()
