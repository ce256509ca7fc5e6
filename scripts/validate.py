#!/usr/bin/env python
"""Validate a generator on a folder of LQ / GT pairs with a training config's own `val.metrics` block, the way
FeMaSRModel.nondist_validation scores it (basicsr/models/femasr_model.py:234-292 of the reference: net_g.test ->
tensor2img -> img2tensor / 255 -> every metric against the GT in [0, 1]), with the generator and every metric on the
engine.

    python scripts/validate.py -opt options/train_FeMaSR_LQ_stage.yml --lq DIR --gt DIR -w net_g.pth \\
        [--lpips-weights FILE [FILE]]

The generator is the config's `network_g` (basicsr.archs.build_network); each metric of `val.metrics` is built with
femasr_b200.metrics.create_metric(type, **options), `better` dropped as the model drops it.  --lpips-weights: one file =
a combined lpips state_dict, two files = a torchvision backbone checkpoint and an lpips lin-weights file (needed when the
block has an lpips metric; nothing is downloaded).  GT images pair with LQ images by file name; same-shape LQ images are
super-resolved and scored as one batch (FeMaSRNet.sr_uint8: identical per image to tensor2img(test(x))).
Prints one line per image with every metric, then the means and the key metric."""
import argparse
import os
import sys
import warnings

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from basicsr.archs import build_network  # noqa: E402
from femasr_b200.folders import paired_batches, rgb01  # noqa: E402
from femasr_b200.metrics import create_metric  # noqa: E402


def metric_plan(opt: dict):
    """(key_metric, [(name, type, options)]) of a parsed config's `val` block, in the block's order."""
    val = opt.get("val") or {}
    plan = []
    for name, mopt in (val.get("metrics") or {}).items():
        mopt = dict(mopt)
        mtype = mopt.pop("type", None)
        if mtype is None:
            raise SystemExit(f"val.metrics.{name}: no type")
        mopt.pop("better", None)
        plan.append((name, mtype, mopt))
    return val.get("key_metric"), plan


def load_options(path: str) -> dict:
    import yaml
    with open(path) as f:
        return yaml.safe_load(f)


def build_metrics(plan, lpips_weights, device):
    metrics = {}
    for name, mtype, mopt in plan:
        if mtype.startswith("lpips"):
            if not lpips_weights:
                raise SystemExit(f"val.metrics.{name} is {mtype!r}: give its weights with --lpips-weights")
            if len(lpips_weights) == 2:
                m = create_metric(mtype, backbone_path=lpips_weights[0], lin_path=lpips_weights[1], **mopt)
            else:
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")      # the file below replaces the untrained default tensors
                    m = create_metric(mtype, **mopt)
                m.net.load_state_dict(torch.load(lpips_weights[0], map_location="cpu"), strict=True)
        else:
            m = create_metric(mtype, **mopt)
        metrics[name] = m.to(device)
    return metrics


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("-opt", "--opt", required=True, help="training config (yaml) with network_g and val.metrics")
    ap.add_argument("--lq", required=True)
    ap.add_argument("--gt", required=True)
    ap.add_argument("-w", "--weight", required=True, help="generator checkpoint {'params': state_dict}")
    ap.add_argument("--lpips-weights", nargs="+", default=None)
    ap.add_argument("--batch", type=int, default=8, help="most same-shape images per batch")
    a = ap.parse_args(argv)
    if a.lpips_weights is not None and len(a.lpips_weights) > 2:
        ap.error("--lpips-weights takes one or two files")
    opt = load_options(a.opt)
    key, plan = metric_plan(opt)
    if not plan:
        raise SystemExit(f"{a.opt}: no val.metrics block")
    dev = torch.device("cuda")
    net = build_network(opt["network_g"])
    net.load_state_dict(torch.load(a.weight, map_location="cpu")["params"], strict=True)
    net = net.to(dev).eval()
    metrics = build_metrics(plan, a.lpips_weights, dev)

    scores = {}
    with torch.no_grad():
        for chunk in paired_batches(a.lq, a.gt, net.scale_factor, a.batch):
            lq = torch.from_numpy(np.stack([im for _, im, _ in chunk])).to(dev)
            sr = rgb01(net.sr_uint8(lq))
            gt = rgb01(torch.from_numpy(np.stack([g for _, _, g in chunk])).to(dev))
            vals = {name: m(sr, gt).view(-1).tolist() for name, m in metrics.items()}
            for i, (img, _, _) in enumerate(chunk):
                scores[img] = {name: v[i] for name, v in vals.items()}
    for img in sorted(scores):
        print(img + "".join(f" {name} {scores[img][name]:.6f}" for name in metrics))
    means = "".join(f" {name} {np.mean([s[name] for s in scores.values()]):.6f}" for name in metrics)
    print(f"mean over {len(scores)} images:{means}")
    print(f"key metric: {key}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
