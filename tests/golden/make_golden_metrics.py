"""Generate tests/golden/metrics/ (the PSNR / SSIM fixtures), offline.  Build container only (the Y conversion of the
ycbcr cases is the reference's own rgb2ycbcr):

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_metrics.py

pyiqa is not available offline, so the fixtures pin the definitions written in include/femasr_b200.h, computed
independently of the engine's oracle (tests/metrics_oracle.py):
- the Y channel: the reference's unmodified basicsr.utils.matlab_functions.rgb2ycbcr(img, y_only=True) for 'ycbcr', and
  the YIQ formula 0.299 R + 0.587 G + 0.114 B in float64 for 'yiq';
- SSIM: cv2.filter2D with the outer product of cv2.getGaussianKernel(11, 1.5), in float64, the 'valid' region cut out
  afterwards; PSNR: numpy float64.
Inputs are uint8 images / 255 (a smooth random field plus texture, tests/golden/make_golden_lpips.py); the second image
is the first plus small noise (SR-like) or an unrelated image.  SSIM rounds Y * 255; a pixel whose Y * 255 lies within
1e-4 of a rounding boundary (in either colour space) is redrawn, so that no fixture depends on how a tie rounds.
"""
from __future__ import annotations

import importlib.util
import os
import sys

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden_lpips import pair_u8  # noqa: E402
from oracle.ref_shim import REFERENCE_ROOT  # noqa: E402

OUT = os.path.join(HERE, "metrics")

# name, colour space ('rgb' = test_y_channel False), crop_border, B, H, W, per image: "sr" or "far"
CASES = [
    ("yiq_b3_37x53_crop0", "yiq", 0, 3, 37, 53, ("sr", "far", "sr")),
    ("yiq_b3_64x64_crop4", "yiq", 4, 3, 64, 64, ("sr", "sr", "far")),
    ("ycbcr_b1_256x256_crop4", "ycbcr", 4, 1, 256, 256, ("sr",)),
    ("ycbcr_b3_37x53_crop4", "ycbcr", 4, 3, 37, 53, ("far", "sr", "sr")),
    ("rgb_b3_64x64_crop4", "rgb", 4, 3, 64, 64, ("sr", "far", "sr")),
    ("rgb_b1_37x53_crop0", "rgb", 0, 1, 37, 53, ("sr",)),
]


def reference_rgb2ycbcr():
    spec = importlib.util.spec_from_file_location(
        "ref_matlab_functions", os.path.join(REFERENCE_ROOT, "basicsr", "utils", "matlab_functions.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.rgb2ycbcr


RGB2YCBCR = reference_rgb2ycbcr()


def y_of(img01: np.ndarray, space: str) -> np.ndarray:
    """[H,W,3] RGB float32 in [0, 1] -> [H,W] float64."""
    if space == "ycbcr":
        return RGB2YCBCR(img01, y_only=True).astype(np.float64)
    f = img01.astype(np.float64)
    return 0.299 * f[..., 0] + 0.587 * f[..., 1] + 0.114 * f[..., 2]


def near_ties(u8: np.ndarray) -> np.ndarray:
    """[3,H,W] uint8 -> [H,W] mask of pixels whose Y * 255 is within 1e-4 of a rounding boundary in either space."""
    img = (u8.transpose(1, 2, 0).astype(np.float32) / np.float32(255.0))
    mask = np.zeros(u8.shape[1:], dtype=bool)
    for space in ("yiq", "ycbcr"):
        v = y_of(img, space) * 255.0
        mask |= np.abs(v - np.floor(v) - 0.5) < 1e-4
    return mask


def untie(u8: np.ndarray, g: np.random.Generator) -> np.ndarray:
    u8 = u8.copy()
    for _ in range(100):
        m = near_ties(u8)
        if not m.any():
            return u8
        u8[2][m] = g.integers(0, 256, size=int(m.sum()), dtype=np.uint8)      # redraw the blue value of those pixels
    raise RuntimeError("could not remove the rounding ties")


def planes(u8: np.ndarray, space: str) -> list:
    """[3,H,W] uint8 -> the planes the metrics compare, float64 at data range 1."""
    img = u8.transpose(1, 2, 0).astype(np.float32) / np.float32(255.0)
    if space == "rgb":
        return [img[..., c].astype(np.float64) for c in range(3)]
    return [y_of(img, space)]


def crop(p: np.ndarray, c: int) -> np.ndarray:
    return p[c:p.shape[0] - c, c:p.shape[1] - c] if c else p


def psnr(px, py, c):
    mse = np.mean([np.mean((crop(a, c) - crop(b, c)) ** 2) for a, b in zip(px, py)])
    return 10.0 * np.log10(1.0 / (mse + 1e-8))


def ssim_plane(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    g = cv2.getGaussianKernel(11, 1.5)
    win = np.outer(g, g)

    def filt(t):
        return cv2.filter2D(t, -1, win)[5:-5, 5:-5]

    C1, C2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2
    mx, my = filt(a), filt(b)
    vx, vy, cxy = filt(a * a) - mx ** 2, filt(b * b) - my ** 2, filt(a * b) - mx * my
    cs = np.maximum((2 * cxy + C2) / (vx + vy + C2), 0.0)
    return (2 * mx * my + C1) / (mx ** 2 + my ** 2 + C1) * cs


def ssim(px, py, space, c):
    if space == "rgb":
        a, b = [p * 255.0 for p in px], [p * 255.0 for p in py]
    else:
        a, b = [np.round(p * 255.0) for p in px], [np.round(p * 255.0) for p in py]   # np.round: half to even
    return np.mean([ssim_plane(crop(u, c), crop(v, c)) for u, v in zip(a, b)])


def main():
    os.makedirs(OUT, exist_ok=True)
    for k, (name, space, c, B, H, W, kinds) in enumerate(CASES):
        u0, u1 = pair_u8(torch.Generator().manual_seed(700 + k), B, H, W, kinds)
        rng = np.random.default_rng(800 + k)
        u0 = np.stack([untie(u, rng) for u in u0.numpy()])
        u1 = np.stack([untie(u, rng) for u in u1.numpy()])
        p = np.array([psnr(planes(a, space), planes(b, space), c) for a, b in zip(u0, u1)])
        s = np.array([ssim(planes(a, space), planes(b, space), space, c) for a, b in zip(u0, u1)])
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, color_space=space, crop_border=c, x_u8=u0, y_u8=u1, psnr=p, ssim=s)
        print(f"{name}: psnr {np.round(p, 4).tolist()} ssim {np.round(s, 5).tolist()} -> {os.path.getsize(path) / 1e3:.0f} kB")


if __name__ == "__main__":
    main()
