"""Throughput of UNetDiscriminatorSN (the training configs' network_d) on the engine, at the LQ stage's workload: the
discriminator scores batch 8 of 256 x 256 SR outputs (options/train_FeMaSR_LQ_stage.yml: batch_size_per_gpu 8,
gt_size 256).

    python scripts/bench_disc.py [--batch 8] [--size 256] [--steps 20] [--warmup 5] [--gemm-path 1] [--out DIR]

Prints the card name and power limit, images/s of the eval-mode forward (CUDA events over --steps steps after --warmup
warm-up steps), the per-kernel profile (a separate, profiled step) and the algorithmic TF/s of the discriminator's
convs.  The FLOP count (51.84 GFLOP per 256 x 256 image, conv0 at K = 27) is computed from shapes here and
cross-checked against the engine's sizing-run count and the profile's own FLOP counts.  Writes nothing into the tree;
--out DIR saves the JSON result there.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def disc_flops(H: int, W: int, F: int = 64) -> dict:
    """Algorithmic FLOPs (2 * MAC) of the disc_conv GEMMs (conv0 ... conv8) and the conv9 head on one H x W image."""
    f = H * W * F * 27                                                                       # conv0
    f += sum((H >> i) * (W >> i) * (F << i) * (F << (i - 1)) * 16 for i in (1, 2, 3))       # conv1 .. conv3
    f += sum((H >> lv) * (W >> lv) * (F << lv) * (F << (lv + 1)) * 9 for lv in (2, 1, 0))   # conv4 .. conv6
    f += 2 * H * W * F * F * 9                                                               # conv7, conv8
    return {"disc_conv": 2.0 * f, "disc_head": 2.0 * H * W * F * 9}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as ex:       # noqa: BLE001 - informational only
        return f"unknown ({ex})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--gemm-path", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert abs(sum(disc_flops(256, 256).values()) / 1e9 - 51.84) < 0.005

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_disc.py needs a CUDA sm_90 (H100) device")
    from basicsr.archs.discriminator_arch import UNetDiscriminatorSN
    from femasr_b200.spec import random_disc_state_dict

    dev = torch.device("cuda", 0)
    net = UNetDiscriminatorSN(3, gemm_path=args.gemm_path)
    net.load_state_dict(random_disc_state_dict(0), strict=True)
    net = net.to(dev).eval()
    eng = net._native(dev)
    B, S = args.batch, args.size
    x = torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(1)).to(dev)
    fl = {k: v * B for k, v in disc_flops(S, S).items()}
    total = sum(fl.values())
    assert eng.flops(B, S, S) == total, (eng.flops(B, S, S), total)

    with torch.no_grad():
        for _ in range(args.warmup):
            eng.forward(x)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            y = eng.forward(x)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        eng.set_profile(True)
        eng.forward(x)
        torch.cuda.synchronize()
        prof = eng.profile()
        eng.set_profile(False)
    for k, v in fl.items():
        assert abs(prof[k]["flops"] - v) <= 1e-6 * v, (k, prof[k]["flops"], v)
    conv_ms = prof["disc_conv"]["ms"]
    result = {
        "card": card(), "gemm_path": args.gemm_path, "batch": B, "size": S, "steps": args.steps,
        "images_per_s": B / (ms / 1e3), "ms_per_step": ms, "launches": eng.last_launch_count(),
        "gflop_per_image": total / B / 1e9, "disc_conv_tflops": fl["disc_conv"] / (conv_ms / 1e3) / 1e12,
        "output_max_abs": y.abs().max().item(), "profile": prof,
    }
    print(f"card: {result['card']}")
    print(f"UNetDiscriminatorSN, batch {B} x {S}x{S}, gemm_path {args.gemm_path}, {args.steps} steps after "
          f"{args.warmup} warm-up")
    print(f"  forward: {ms:8.2f} ms/step  {result['images_per_s']:8.1f} images/s  ({result['launches']} launches)")
    print("  kernels (one profiled step, CUDA events):")
    for k, r in sorted(prof.items(), key=lambda kv: -kv[1]["ms"]):
        tf = f"{r['flops'] / (r['ms'] / 1e3) / 1e12:7.1f} TF/s" if r["flops"] else ""
        print(f"    {k:14s} launches {r['launches']:3d}  {r['ms']:8.3f} ms  {tf}")
    print(f"  disc_conv: {fl['disc_conv'] / B / 1e9:.2f} GFLOP/image, {result['disc_conv_tflops']:.1f} TF/s algorithmic")
    print(json.dumps(result))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"bench_disc_gp{args.gemm_path}.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
