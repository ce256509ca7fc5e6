"""Throughput of the HQ-pretrain stage's forward with and without the semantic loss (use_semantic_loss=True), at that
configuration's own workload (options/train_FeMaSR_HQ_pretrain_stage.yml: batch_size_per_gpu 8, gt_size 256, HQ e512).

    python scripts/bench_semantic.py [--batch 8] [--size 256] [--steps 20] [--warmup 5] [--gemm-path 1] [--out DIR]

Prints the card name and power limit, images/s of `forward` without and with the loss (CUDA events over --steps
steps after --warmup warm-up steps, both through the engine's CUDA graph), the per-kernel profile of the semantic
branch (a separate, profiled step), and the algorithmic TF/s of the VGG convs.  The VGG FLOP count (46.13 GFLOP per
256 x 256 image) is computed from shapes here and cross-checked against the profile's own FLOP counts.
Writes nothing into the tree; --out DIR saves the JSON result there.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEM_KERNELS = ("vgg_im2col", "vgg_conv", "vgg_pool", "semantic_conv", "semantic_mse")


def vgg_flops(H: int, W: int) -> float:
    """Algorithmic FLOPs (2 * MAC) of VGG19 conv1_1 ... conv4_4 on one H x W image."""
    from femasr_b200.spec import VGG_CONVS
    f, h, w = 0.0, H, W
    for name, ci, co in VGG_CONVS:
        if name in ("conv2_1", "conv3_1", "conv4_1"):
            h, w = h // 2, w // 2
        f += 2.0 * h * w * co * ci * 9
    return f


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
    assert abs(vgg_flops(256, 256) / 1e9 - 46.13) < 0.005

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_semantic.py needs a CUDA sm_90 (H100) device")
    from basicsr.archs.femasr_arch import FeMaSRNet
    from femasr_b200.spec import random_state_dict

    dev = torch.device("cuda", 0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)       # the VGG weights come from the seeded state_dict
        net = FeMaSRNet(codebook_params=[[32, 1024, 512]], LQ_stage=False, use_semantic_loss=True,
                        gemm_path=args.gemm_path)
    net.load_state_dict(random_state_dict(1, 512, seed=0, semantic=True), strict=True)
    net = net.to(dev).eval()
    eng = net._native(dev)
    B, S = args.batch, args.size
    x = torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(1)).to(dev)

    def timed(want_sem):
        step = (lambda: eng.forward_graph(x, want_sem=want_sem)) if eng.use_graph else \
            (lambda: eng.forward(x, want_sem=want_sem))
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            res = step()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        return ms, res

    with torch.no_grad():
        ms_off, _ = timed(False)
        ms_on, res = timed(True)
        sem = res[3].item()
        eng.set_profile(True)
        eng.forward(x, want_sem=True)
        torch.cuda.synchronize()
        prof = eng.profile()
        eng.set_profile(False)
    rows = {k: prof[k] for k in SEM_KERNELS if k in prof}
    vgg_ms = rows["vgg_conv"]["ms"]
    vf = vgg_flops(S, S) * B
    assert abs(rows["vgg_conv"]["flops"] - vf) <= 1e-6 * vf, (rows["vgg_conv"]["flops"], vf)
    result = {
        "card": card(), "gemm_path": args.gemm_path, "batch": B, "size": S, "steps": args.steps,
        "images_per_s_without_sem": B / (ms_off / 1e3), "images_per_s_with_sem": B / (ms_on / 1e3),
        "ms_per_step_without_sem": ms_off, "ms_per_step_with_sem": ms_on, "semantic_loss": sem,
        "vgg_gflop_per_image": vgg_flops(S, S) / 1e9, "vgg_conv_tflops": vf / (vgg_ms / 1e3) / 1e12,
        "profile": rows,
    }
    print(f"card: {result['card']}")
    print(f"HQ e512, batch {B} x {S}x{S}, gemm_path {args.gemm_path}, {args.steps} steps after {args.warmup} warm-up")
    print(f"  forward without semantic loss: {ms_off:8.2f} ms/step  {result['images_per_s_without_sem']:8.1f} images/s")
    print(f"  forward with semantic loss:    {ms_on:8.2f} ms/step  {result['images_per_s_with_sem']:8.1f} images/s")
    print("  semantic-branch kernels (one profiled step, CUDA events):")
    for k, r in rows.items():
        tf = f"{r['flops'] / (r['ms'] / 1e3) / 1e12:7.1f} TF/s" if r["flops"] else ""
        print(f"    {k:14s} launches {r['launches']:3d}  {r['ms']:8.3f} ms  {tf}")
    print(f"  vgg_conv: {vgg_flops(S, S) / 1e9:.2f} GFLOP/image, {result['vgg_conv_tflops']:.1f} TF/s algorithmic")
    print(json.dumps(result))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"bench_semantic_gp{args.gemm_path}.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
