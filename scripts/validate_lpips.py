#!/usr/bin/env python
"""LPIPS of a folder of super-resolved images against their ground truth, the way the training configs validate
(FeMaSRModel.nondist_validation, basicsr/models/femasr_model.py:255-292 of the reference: net_g.test -> tensor2img ->
img2tensor / 255 -> pyiqa's LPIPS against the GT in [0, 1]), with the generator and the metric both on the engine.

    python scripts/validate_lpips.py --lq DIR --gt DIR -w net_g.pth --lpips alex|vgg --lpips-weights FILE [FILE]

--lpips-weights: one file = a combined lpips state_dict (scaling_layer.*, net.slice*, lin*); two files = a torchvision
alexnet / vgg16 checkpoint and an lpips lin-weights file.  GT images pair with LQ images by file name.  Same-shape LQ
images are super-resolved and scored as one batch (FeMaSRNet.sr_uint8: identical per image to tensor2img(test(x))).
Prints one line per image and the mean."""
import argparse
import os
import sys
import warnings

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from basicsr.archs.femasr_arch import FeMaSRNet  # noqa: E402
from femasr_b200.folders import paired_batches, rgb01  # noqa: E402
from femasr_b200.lpips import LPIPS  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--lq", required=True)
    ap.add_argument("--gt", required=True)
    ap.add_argument("-w", "--weight", required=True, help="generator checkpoint {'params': state_dict}")
    ap.add_argument("--lpips", choices=("alex", "vgg"), default="alex", help="pyiqa 'lpips' = alex, 'lpips-vgg' = vgg")
    ap.add_argument("--lpips-weights", nargs="+", required=True)
    ap.add_argument("--scale", type=int, default=4)
    ap.add_argument("--codebook", default="32,1024,512", help="codebook_params row of the generator: scale,n_e,e_dim")
    ap.add_argument("--batch", type=int, default=8, help="most same-shape images per batch")
    a = ap.parse_args(argv)
    dev = torch.device("cuda")
    net = FeMaSRNet(codebook_params=[[int(v) for v in a.codebook.split(",")]], LQ_stage=True, scale_factor=a.scale)
    net.load_state_dict(torch.load(a.weight, map_location="cpu")["params"], strict=True)
    net = net.to(dev).eval()
    if len(a.lpips_weights) == 1:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")          # the file below replaces the untrained default tensors
            metric = LPIPS(a.lpips)
        metric.load_state_dict(torch.load(a.lpips_weights[0], map_location="cpu"), strict=True)
    else:
        metric = LPIPS(a.lpips, backbone_path=a.lpips_weights[0], lin_path=a.lpips_weights[1])
    metric = metric.to(dev)

    scores = {}
    with torch.no_grad():
        for chunk in paired_batches(a.lq, a.gt, a.scale, a.batch):
            lq = torch.from_numpy(np.stack([im for _, im, _ in chunk])).to(dev)
            sr = net.sr_uint8(lq)
            gt = torch.from_numpy(np.stack([g for _, _, g in chunk])).to(dev)
            d = metric(rgb01(sr), rgb01(gt), normalize=True).view(-1).cpu()
            for (name, _, _), v in zip(chunk, d.tolist()):
                scores[name] = v
    for name in sorted(scores):
        print(f"{name} {scores[name]:.6f}")
    print(f"mean lpips ({a.lpips}) over {len(scores)} images: {np.mean(list(scores.values())):.6f}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
