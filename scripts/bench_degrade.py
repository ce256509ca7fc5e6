"""Throughput of degradation_bsrgan on the engine (femasr_b200.degrade), in images/s, for the reference's two callers:
generate_dataset.py (512x512 HR at sf 4 and sf 2) and BSRGANTrainDataset (a 256x256 crop, lq_patchsize 64), both with
use_crop=False.

    python scripts/bench_degrade.py [--images 40] [--warmup 5] [--out FILE.json]

Each image is one call on seeded streams; the timed window ends in a device synchronise.  Per image: the wall time,
and the device time per step kind from CUDA events around each step (a step's table or noise-field upload included).
The rest of the wall time is host work (the draws, numpy's noise fields, tap tables, launches).
"""
from __future__ import annotations

import argparse
import json
import os
import random
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from femasr_b200 import degrade as D  # noqa: E402

WORKLOADS = [("generate_dataset_512_sf4", 512, 4, 72), ("generate_dataset_512_sf2", 512, 2, 72),
             ("train_dataset_256_sf4", 256, 4, 64)]


class Timer:
    """CUDA events around each step (degradation_bsrgan's _timer hook)."""

    def __init__(self):
        self.events = []

    def begin(self):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return e

    def end(self, op, start):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.events.append((op, start, e))


def run(name, size, sf, lqp, n, warmup):
    g = np.random.default_rng(size * sf)
    imgs = [torch.from_numpy(g.random((size, size, 3), dtype=np.float32)).cuda() for _ in range(4)]
    random.seed(123)
    np.random.seed(123)
    for i in range(warmup):
        D.degradation_bsrgan(imgs[i % 4], sf, lqp, use_crop=False)
    timer = Timer()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        D.degradation_bsrgan(imgs[i % 4], sf, lqp, use_crop=False, _timer=timer)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    dev_ms = {}
    for op, s, e in timer.events:
        dev_ms[op] = dev_ms.get(op, 0.0) + s.elapsed_time(e) / n
    return dict(workload=name, images=n, images_per_s=n / wall, wall_ms_per_image=1e3 * wall / n,
                device_ms_per_image_by_step=dev_ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_degrade: needs a CUDA device (sm_90)")
    res = dict(device=torch.cuda.get_device_name(0), results=[run(*w, a.images, a.warmup) for w in WORKLOADS])
    for r in res["results"]:
        d = r["device_ms_per_image_by_step"]
        print(f"{r['workload']}: {r['images_per_s']:.1f} images/s, {r['wall_ms_per_image']:.2f} ms/image wall; device "
              f"ms/image: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(d.items())) + f" (sum {sum(d.values()):.3f})")
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
