"""Run an UNMODIFIED reference entry script (inference_resshift.py, app.py, ...) on the H100-native hot path:

    python -m resshift_b200.launch /path/to/ResShift/inference_resshift.py -i in -o out --task realsr --scale 4

It puts ``resshift_b200/overlay`` ahead of the script's directory on ``sys.path`` so that ``sampler``,
``models.unet`` and ``models.script_util`` resolve to this package (everything else — ldm, utils, datapipe,
basicsr, the rest of ``models`` — still comes from the reference tree), then executes the script as __main__.
The reference scripts open ``./configs/*.yaml`` and ``./weights`` relative to the working directory, so the script's
directory becomes the working directory (relative ``-i`` / ``-o`` paths are resolved against the original one first).
"""
import os
import runpy
import sys
from pathlib import Path


def main():
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    script = Path(sys.argv[1]).resolve()
    overlay = Path(__file__).resolve().parent / "overlay"
    repo = Path(__file__).resolve().parent.parent
    sys.path[:0] = [str(overlay), str(script.parent), str(repo)]
    args = sys.argv[2:]
    for i, a in enumerate(args[:-1]):                       # keep caller-relative paths valid after the chdir
        if a in ("-i", "--in_path", "-o", "--out_path", "--mask_path") and args[i + 1]:
            args[i + 1] = str(Path(args[i + 1]).resolve())
    sys.argv = [str(script)] + args
    os.chdir(script.parent)
    runpy.run_path(str(script), run_name="__main__")


if __name__ == "__main__":
    main()
