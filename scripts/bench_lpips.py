"""Throughput of LPIPS (femasr_b200.lpips.LPIPS, both nets) on the engine, on both GEMM paths, at two workloads:
- the training shape: batch 8 of 256 x 256 pairs (the perceptual loss of options/train_FeMaSR_*.yml: batch_size_per_gpu 8,
  gt_size 256);
- a validation shape: one 1344 x 2032 pair (the gt_mod16 size class of DIV2K-val, which validation scores one image at a
  time).

    python scripts/bench_lpips.py [--steps 10] [--warmup 3] [--nets alex,vgg] [--gemm-paths 0,1] [--out DIR]

For each (net, path, workload): pairs/s of the forward (CUDA events over --steps steps after --warmup warm-up steps), and
the algorithmic TF/s of the backbone convs from one separate profiled step.  The card name and power limit are read in
the same run.  The FLOP count is computed from shapes here and cross-checked against the engine's sizing-run count.
Writes nothing into the tree; --out DIR saves the JSON result there.
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


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as ex:       # noqa: BLE001 - informational only
        return f"unknown ({ex})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--nets", default="alex,vgg")
    ap.add_argument("--gemm-paths", default="0,1")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import warnings
    if not torch.cuda.is_available():
        raise SystemExit("bench_lpips.py needs a CUDA sm_90 (H100) device")
    from femasr_b200.lpips import LPIPS
    from femasr_b200.spec import random_lpips_state_dict
    from tests.test_lpips import lpips_flops_closed_form

    dev = torch.device("cuda", 0)
    results = {"card": card(), "runs": []}
    print(f"card: {results['card']}")
    for net in args.nets.split(","):
        for gp in (int(v) for v in args.gemm_paths.split(",")):
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                m = LPIPS(net, gemm_path=gp)
            m.load_state_dict(random_lpips_state_dict(net, 0), strict=True)
            m = m.to(dev)
            for wl, (B, H, W) in WORKLOADS.items():
                g = torch.Generator().manual_seed(1)
                x0 = torch.rand(B, 3, H, W, generator=g).to(dev)
                x1 = (x0 + 0.05 * torch.randn(B, 3, H, W, generator=g).to(dev)).clamp(0, 1)
                eng = m._native(dev)
                fl = lpips_flops_closed_form(net, B, H, W)
                assert eng.flops(B, H, W) == fl, (eng.flops(B, H, W), fl)
                for _ in range(args.warmup):
                    d = m(x0, x1, normalize=True)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    d = m(x0, x1, normalize=True)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / args.steps
                eng.set_profile(True)
                m(x0, x1, normalize=True)
                torch.cuda.synchronize()
                prof = eng.profile()
                eng.set_profile(False)
                conv = prof["lpips_conv"]
                assert abs(conv["flops"] - fl) <= 1e-6 * fl
                r = {"net": net, "gemm_path": gp, "workload": wl, "B": B, "H": H, "W": W, "ms_per_step": ms,
                     "pairs_per_s": B / (ms / 1e3), "gflop_per_pair": fl / B / 1e9,
                     "conv_tflops": fl / (conv["ms"] / 1e3) / 1e12, "launches": eng.last_launch_count(),
                     "d_mean": d.mean().item(), "profile": prof}
                results["runs"].append(r)
                print(f"{net:4s} gemm_path {gp} {wl:17s} {ms:9.2f} ms/step {r['pairs_per_s']:9.1f} pairs/s  "
                      f"convs {r['conv_tflops']:6.1f} TF/s algorithmic ({r['gflop_per_pair']:.1f} GFLOP/pair, "
                      f"{r['launches']} launches)")
                for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"]):
                    print(f"      {k:14s} launches {v['launches']:3d}  {v['ms']:9.3f} ms")
            m._engine.close()
            del m
            torch.cuda.empty_cache()
    print(json.dumps({k: v for k, v in results.items()}))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_lpips.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
