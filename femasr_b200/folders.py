"""Folder pairing for the validation tools (scripts/validate.py, scripts/validate_lpips.py): LQ images pair with the GT
images of the same file name, and same-shape LQ images are grouped into batches for FeMaSRNet.sr_uint8."""
from __future__ import annotations

import glob
import os
from typing import List, Tuple

import numpy as np
import torch


def rgb01(bgr_u8: torch.Tensor) -> torch.Tensor:
    """uint8 BGR [B,h,w,3] -> fp32 RGB [B,3,h,w] / 255 (img2tensor(img) / 255).  On CUDA, torch computes a division by a
    Python scalar as a multiplication by its reciprocal, which differs from the reference's CPU division by 1 ulp for
    some values (DESIGN.md section 6, "PSNR / SSIM")."""
    return bgr_u8.flip(-1).permute(0, 3, 1, 2).float() / 255.0


def paired_batches(lq_dir: str, gt_dir: str, scale: int, batch: int) -> List[List[Tuple[str, np.ndarray, np.ndarray]]]:
    """Every image of lq_dir (sorted by name; files cv2 cannot read are skipped) with the GT of the same name, which must
    be `scale` times its size, as lists of at most `batch` (name, lq, gt) uint8 BGR HWC triples of one LQ shape: the
    shapes in order of first appearance.  Raises SystemExit naming the first LQ image without a matching GT."""
    import cv2
    groups = {}
    for path in sorted(glob.glob(os.path.join(lq_dir, "*"))):
        img = cv2.imread(path, cv2.IMREAD_COLOR)
        if img is None:
            continue
        gt = cv2.imread(os.path.join(gt_dir, os.path.basename(path)), cv2.IMREAD_COLOR)
        if gt is None or gt.shape[:2] != (img.shape[0] * scale, img.shape[1] * scale):
            raise SystemExit(f"{path}: no ground truth of {scale}x its size under {gt_dir}")
        groups.setdefault(img.shape[:2], []).append((os.path.basename(path), img, gt))
    return [items[i:i + batch] for items in groups.values() for i in range(0, len(items), batch)]
