"""Time of PSNR and SSIM (femasr_b200.metrics, Y channel, crop_border 4: the LQ config's val block) on the engine, at the
LPIPS bench's two workloads:
- batch 8 of 256 x 256 pairs (the training crops, batch_size_per_gpu 8, gt_size 256);
- one 1344 x 2032 pair (the gt_mod16 size class of DIV2K-val, which validation scores one image at a time).

    python scripts/bench_metrics.py [--steps 200] [--warmup 20] [--out DIR]

For each (metric, workload): microseconds per call of the public forward (CUDA events over --steps calls after --warmup
warm-up calls; each call allocates its output and scratch through the caching allocator, memsets the B arrival counters
and launches one kernel), the kernel's own time (torch.profiler, a separate run of --steps calls), and the bandwidth the
kernel achieves over the bytes the inputs require (both images, 3 channels of fp32: 24 B per cropped pixel) as a fraction
of the H100 SXM data sheet's 3.35 TB/s.  For context, the time of FeMaSRNet.sr_uint8
(x4, seeded weights, e_dim 512 as in the configs) producing the 1344 x 2032 image from its 336 x 508 LQ.  The card name
and power limit are read in the same run.  Writes nothing into the tree; --out DIR saves the JSON result there.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {"train_b8_256": (8, 256, 256), "val_b1_1344x2032": (1, 1344, 2032)}
HBM_PEAK = 3.35e12          # bytes/s, H100 SXM data sheet


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as ex:       # noqa: BLE001 - informational only
        return f"unknown ({ex})"


def time_us(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / steps


def kernel_us(fn, name, steps):
    """Mean device time of the kernels whose name contains `name`, from a separate torch.profiler run of `steps` calls."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    hits = [e for e in prof.key_averages() if name in e.key]
    if not hits:
        raise SystemExit(f"bench_metrics.py: no kernel named {name} in the profile")
    total = sum(getattr(e, "device_time_total", None) or e.cuda_time_total for e in hits)
    return total / sum(e.count for e in hits)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--sr-steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_metrics.py needs a CUDA sm_90 (H100) device")
    from femasr_b200.metrics import PSNR, SSIM

    dev = torch.device("cuda", 0)
    results = {"card": card(), "runs": []}
    print(f"card: {results['card']}")
    for wl, (B, H, W) in WORKLOADS.items():
        g = torch.Generator().manual_seed(1)
        x = torch.rand(B, 3, H, W, generator=g).to(dev)
        y = (x + 0.03 * torch.randn(B, 3, H, W, generator=g).to(dev)).clamp(0, 1)
        for m in (PSNR(test_y_channel=True, crop_border=4), SSIM(test_y_channel=True, crop_border=4)):
            us = time_us(lambda: m(x, y), args.steps, args.warmup)
            kus = kernel_us(lambda: m(x, y), f"{m._name}_kernel", args.steps)
            nbytes = 2 * B * 3 * (H - 8) * (W - 8) * 4
            gbs = nbytes / (kus * 1e-6) / 1e9
            r = {"metric": m._name, "workload": wl, "B": B, "H": H, "W": W, "us_per_call": us, "kernel_us": kus,
                 "bytes": nbytes, "kernel_GB_per_s": gbs, "hbm_fraction": gbs * 1e9 / HBM_PEAK,
                 "mean": m(x, y).mean().item()}
            results["runs"].append(r)
            print(f"{m._name:4s} {wl:17s} {us:8.2f} us/call, kernel {kus:8.2f} us: {gbs:7.1f} GB/s over the input "
                  f"bytes ({r['hbm_fraction']:.3f} of 3.35 TB/s)  mean {r['mean']:.4f}")

    from basicsr.archs.femasr_arch import FeMaSRNet
    from femasr_b200.spec import random_state_dict
    net = FeMaSRNet(codebook_params=[[32, 1024, 512]], LQ_stage=True, scale_factor=4)
    net.load_state_dict(random_state_dict(4, 512, seed=0, init="perturbed"), strict=True)
    net = net.to(dev).eval()
    lq = (torch.rand(1, 336, 508, 3, generator=torch.Generator().manual_seed(2)) * 255).to(torch.uint8).to(dev)
    assert tuple(net.sr_uint8(lq).shape) == (1, 1344, 2032, 3)
    sr_us = time_us(lambda: net.sr_uint8(lq), args.sr_steps, 2)
    results["sr_uint8_1344x2032_us"] = sr_us
    print(f"sr_uint8 336x508 -> 1344x2032: {sr_us / 1e3:9.2f} ms/image")
    for r in results["runs"]:
        if r["workload"] == "val_b1_1344x2032":
            print(f"  {r['metric']} at 1344x2032 is {r['us_per_call'] / sr_us:.2e} of that")
    print(json.dumps(results))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_metrics.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
