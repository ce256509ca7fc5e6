#!/usr/bin/env python
"""Folder / single-image super-resolution with the H100-native FeMaSRNet.

Same command line and behaviour as the reference's demo entry point (inference_femasr.py:19-69: -i/-w/-o/-s/
--suffix/--max_size; images below max_size^2 pixels go through `test`, larger ones through `test_tile`), written
against this repo's `basicsr` surface.  The reference's own script also runs unchanged with this repo on PYTHONPATH.
Weights: a checkpoint {'params': state_dict} as the reference saves them (-w); without -w the released weights
are fetched through load_file_from_url (needs network)."""
import argparse
import glob
import os
import sys

import cv2
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from basicsr.archs.femasr_arch import FeMaSRNet  # noqa: E402
from basicsr.utils import img2tensor, imwrite, tensor2img  # noqa: E402
from basicsr.utils.download_util import load_file_from_url  # noqa: E402

URLS = {s: f"https://github.com/chaofengc/FeMaSR/releases/download/v0.1-pretrain_models/FeMaSR_SRX{s}_model_g.pth"
        for s in (2, 4)}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("-i", "--input", default="inputs")
    ap.add_argument("-w", "--weight", default=None)
    ap.add_argument("-o", "--output", default="results")
    ap.add_argument("-s", "--out_scale", type=int, default=4)
    ap.add_argument("--suffix", default="")
    ap.add_argument("--max_size", type=int, default=600)
    ap.add_argument("--e_dim", type=int, default=512, help="codebook dim (released weights: 512)")
    ap.add_argument("--batch", type=int, default=0,
                    help="extension: >0 buckets same-shape images and super-resolves them N at a time with the uint8 "
                         "image boundary fused on the device (FeMaSRNet.sr_uint8); 0 = the reference's one-by-one loop")
    a = ap.parse_args(argv)
    dev = torch.device("cuda" if torch.cuda.is_available() else "cpu")
    wpath = a.weight or load_file_from_url(URLS[a.out_scale])
    net = FeMaSRNet(codebook_params=[[32, 1024, a.e_dim]], LQ_stage=True, scale_factor=a.out_scale).to(dev)
    net.load_state_dict(torch.load(wpath)["params"], strict=False)
    net.eval()
    os.makedirs(a.output, exist_ok=True)
    paths = [a.input] if os.path.isfile(a.input) else sorted(glob.glob(os.path.join(a.input, "*")))

    def save(path, img):
        name, ext = os.path.splitext(os.path.basename(path))
        imwrite(img, os.path.join(a.output, f"{name}{a.suffix}{ext}"))

    if a.batch > 0 and dev.type == "cuda":
        import numpy as np
        # same-shape buckets are flushed as soon as they hold `batch` images: at most (#distinct shapes x batch) decoded
        # images are alive at any time, instead of the whole folder
        buckets, rest = {}, []

        def flush(items):
            batch = torch.from_numpy(np.stack([im for _, im in items])).to(dev)
            for (path, _), o in zip(items, net.sr_uint8(batch).cpu().numpy()):
                save(path, o)

        for path in paths:
            img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
            if img is not None and img.ndim == 3 and img.shape[2] == 3 and img.dtype == "uint8" and \
                    img.shape[0] * img.shape[1] < a.max_size ** 2:
                items = buckets.setdefault(img.shape[:2], [])
                items.append((path, img))
                if len(items) == a.batch:
                    flush(items)
                    buckets[img.shape[:2]] = []
            else:
                rest.append(path)
        for items in buckets.values():
            if items:
                flush(items)
        paths = rest
    for path in paths:
        img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
        x = (img2tensor(img).to(dev) / 255.0).unsqueeze(0)
        h, w = x.shape[2:]
        out = net.test(x) if h * w < a.max_size ** 2 else net.test_tile(x)
        save(path, tensor2img(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
