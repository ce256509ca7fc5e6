"""Write the LQ training set of the LQ-stage configs from an HQ folder, as the reference's generate_dataset.py does, with
degradation_bsrgan on the engine (femasr_b200.degrade):

    python scripts/generate_dataset.py --hq ../datasets/HQ_sub --out ../datasets/LQ_sub_X4 --scale 4 [--seed 123]

Images are taken in the reference's order (os.walk sorted by directory, file names in listing order, followlinks),
on one `random` / `np.random` stream seeded with --seed.  Each is read with cv2 as uint8 BGR, scaled by 1/255 in
float32, turned to RGB, degraded with use_crop=False, and saved as (lq BGR * 255) truncated to uint8.  The output path
is the input's relative path under --out with 'HR' replaced by 'LR' (the reference rewrites 'HQ_sub' to
'LQ_sub_X{scale}' and then 'HR' to 'LR' in the full path).
"""
from __future__ import annotations

import argparse
import os
import random
import sys

import cv2
import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from femasr_b200.degrade import degradation_bsrgan  # noqa: E402

EXTENSIONS = (".jpg", ".JPG", ".jpeg", ".JPEG", ".png", ".PNG", ".ppm", ".PPM", ".bmp", ".BMP", ".tif", ".TIF",
              ".tiff", ".TIFF")


def walk_images(root):
    """The reference's make_dataset order."""
    if not os.path.isdir(root):
        raise SystemExit(f"{root} is not a directory")
    out = []
    for d, _, names in sorted(os.walk(root, followlinks=True)):
        out += [os.path.join(d, n) for n in names if n.endswith(EXTENSIONS)]
    return out


def out_path(path, hq, out):
    return os.path.join(out, os.path.relpath(path, hq).replace("HR", "LR"))


def degrade_file(path, dst, scale):
    img = cv2.imread(path).astype(np.float32) / 255.
    lq, _ = degradation_bsrgan(img[:, :, [2, 1, 0]], sf=scale, use_crop=False)
    os.makedirs(os.path.dirname(dst) or ".", exist_ok=True)
    if not cv2.imwrite(dst, (lq[:, :, [2, 1, 0]] * 255).astype(np.uint8)):
        raise SystemExit(f"could not write {dst}")
    return lq.shape


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--hq", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--scale", type=int, choices=(2, 4), required=True)
    ap.add_argument("--seed", type=int, default=123)
    a = ap.parse_args(argv)
    random.seed(a.seed)
    np.random.seed(a.seed)
    for p in walk_images(a.hq):
        dst = out_path(p, a.hq, a.out)
        shape = degrade_file(p, dst, a.scale)
        print(f"Save {dst} {shape[0]}x{shape[1]}")


if __name__ == "__main__":
    main()
