"""Per-shape timing of the tensor-core implicit GEMM through the C ABI (CUDA events, L2 flushed between reps).
Usage (GPU box): python scripts/microbench_tc.py > gpurun_out/microbench.txt"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import gpu_util as G  # noqa: E402

dev = torch.device("cuda", 0)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, reps=5):
    fn(); fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


ONLY = os.environ.get('MB_ONLY', '')        # substring filter on the case name ('|' separates alternatives)
F8 = int(os.environ.get('MB_F8', '0'))      # 1: the 3x3 convs in the F8 cross-term mode (layers behind the VQ)
GN = int(os.environ.get('MB_GN', '0'))      # 1: the 3x3 convs also emit GroupNorm partial sums (what most of them do in the network)


def conv_case(name, B, H, W, Cin, Cout, ksize=3, up=0, res=False, act=0, split=False, bias=True, slice_kb=0, inplace=False,
              res2=False):
    """inplace: the output overwrites the residual (y = res1), as proj, fc2 and the ResBlocks' second convs do in the
    network; res2: a second residual, as the last conv of decoder blocks 0 and 1 adds."""
    if ONLY and not any(o in name for o in ONLY.split('|')):
        return 0.0
    hi = (torch.randn(B, H, W, Cin, device=dev) * 0.5).half()
    lo = (torch.randn(B, H, W, Cin, device=dev) * 1e-4).half()
    w = torch.randn(Cout, Cin, ksize, ksize, device=dev) * 0.03
    blob = G.tc_pack_up2(w) if up else G.tc_pack(w)
    f8 = 1 if (F8 and ksize == 3 and not slice_kb) else 0
    if f8:
        hi, lo = G.tc_prepare_f8(torch.randn(B, H, W, Cin, device=dev) * 0.5)
        blob = G.tc_pack_f8(w, up2=bool(up))
    b = torch.randn(Cout, device=dev) if bias else None
    u = 2 if up else 1
    y = None if split else torch.empty(B, H * u, W * u, Cout, device=dev)
    r = torch.randn(B, H * u, W * u, Cout, device=dev) if res else None
    if inplace:
        y = r
    r2 = torch.randn(B, H * u, W * u, Cout, device=dev) if res2 else None
    gn = None
    if GN and ksize == 3 and not split:
        gn = torch.empty(B * G.tc_gn_rows(B, H, W, Cin, Cout, upsample=up, slice_kb=slice_kb) * 64, device=dev)
    fn = lambda: G.tc_igemm(hi, lo, blob, b, Cout, ksize, act=act, res1=r, res2=r2, y=y, upsample=up, split_out=split,
                            slice_kb=slice_kb, f8=f8, gn_partial=gn)
    ms = timeit(fn)
    flops = 2.0 * B * H * u * W * u * Cout * Cin * ksize * ksize
    execd = (2 if f8 else 3) * 2.0 * B * H * W * Cout * Cin * (4 * 4 if up else ksize * ksize)
    print(f"{name:34s} {ms:8.3f} ms  algorithmic {flops / ms / 1e9:7.1f} TF/s  executed {execd / ms / 1e9:7.1f} TF/s")
    return ms


print("# Swin linears, batch 32 @64x64 (tokens = 131072)")
conv_case("qkv 256->768", 32, 64, 64, 256, 768, 1)
conv_case("proj 256->256 +res", 32, 64, 64, 256, 256, 1, res=True)
conv_case("proj 256->256 +res in place", 32, 64, 64, 256, 256, 1, res=True, inplace=True)
conv_case("fc1 256->1024 gelu fp32 out", 32, 64, 64, 256, 1024, 1, act=1)
conv_case("fc1 256->1024 gelu split out", 32, 64, 64, 256, 1024, 1, act=1, split=True)
conv_case("fc1 256->1024 noact fp32 out", 32, 64, 64, 256, 1024, 1, act=0)
conv_case("fc2 1024->256 +res", 32, 64, 64, 1024, 256, 1, res=True)
print("# K-sliced accumulation (layers in front of the VQ): accumulator folded into an fp32 running sum every 256 of K")
conv_case("fc2 1024->256 +res sliced in place", 32, 64, 64, 1024, 256, 1, res=True, slice_kb=4, inplace=True)
conv_case("conv 256->256 @64x64 +res sliced", 32, 64, 64, 256, 256, res=True, slice_kb=4)
print("# 3x3 convs, batch 32")
conv_case("conv 256->256 @64x64 +res", 32, 64, 64, 256, 256, res=True)
conv_case("conv 256->256 @128x128", 32, 128, 128, 256, 256)
conv_case("conv 256->256 @128x128 +res", 32, 128, 128, 256, 256, res=True)
conv_case("conv 256->256 @128x128 +res in place", 32, 128, 128, 256, 256, res=True, inplace=True)
conv_case("conv 256->256 @128x128 +res in place +res2", 32, 128, 128, 256, 256, res=True, inplace=True, res2=True)
conv_case("conv 128->128 @256x256", 32, 256, 256, 128, 128)
conv_case("conv 128->128 @256x256 +res", 32, 256, 256, 128, 128, res=True)
conv_case("conv 128->128 @256x256 +res in place", 32, 256, 256, 128, 128, res=True, inplace=True)
conv_case("conv 128->128 @256x256 +res in place +res2", 32, 256, 256, 128, 128, res=True, inplace=True, res2=True)
conv_case("conv 64->64 @512x512 +res", 32, 512, 512, 64, 64, res=True)
conv_case("conv 64->64 @512x512", 32, 512, 512, 64, 64)
print("# upsample-fused (sub-pixel) convs, low-res input size given")
conv_case("up 256->256 @64->128", 32, 64, 64, 256, 256, up=1)
conv_case("up 256->128 @128->256", 32, 128, 128, 256, 128, up=1)
conv_case("up 128->64 @256->512", 32, 256, 256, 128, 64, up=1)


def prep_case(name, B, H, W, C, mode):
    if ONLY and not any(o in name for o in ONLY.split('|')):
        return
    from femasr_b200 import lib as L
    x = torch.randn(B, H, W, C, device=dev)
    sc, sh = torch.rand(B, C, device=dev) + 0.5, torch.randn(B, C, device=dev) * 0.1
    hi = torch.empty(B, H, W, C, dtype=torch.float16, device=dev); lo = torch.empty_like(hi)
    lib = L.load()
    fn = lambda: L.check(lib.femasr_tc_prepare(G.p(x), G.p(hi), G.p(lo), mode, G.p(sc), G.p(sh), None, None, B, H, W, C, 0, 1e-6, G.S()))
    if name.startswith("prep f8"):
        fn = lambda: L.check(lib.femasr_tc_prepare_f8(G.p(x), G.p(hi), G.p(lo), mode, G.p(sc), G.p(sh), B, H, W, C, G.S()))
    ms = timeit(fn)
    print(f"{name:34s} {ms:8.3f} ms  {x.numel() * 8 / ms / 1e6:7.1f} GB/s (4 B read + 4 B written per element)")


print("# operand staging (GN + SiLU + fp16 split), batch 32")
for mode, tag in ((1, "exact"), (3, "fast")):
    prep_case(f"prep {tag} 64ch @512x512", 32, 512, 512, 64, mode)
    prep_case(f"prep {tag} 128ch @256x256", 32, 256, 256, 128, mode)
    prep_case(f"prep {tag} 256ch @128x128", 32, 128, 128, 256, mode)
prep_case("prep none 256ch @64x64", 32, 64, 64, 256, 0)
prep_case("prep f8 fast 64ch @512x512", 32, 512, 512, 64, 3)
prep_case("prep f8 fast 128ch @256x256", 32, 256, 256, 128, 3)
prep_case("prep f8 fast 256ch @128x128", 32, 128, 128, 256, 3)
