"""Generate tests/golden/lpips/ (the LPIPS fixtures), offline:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_lpips.py

Neither the lpips package nor pyiqa is available offline, so the fixtures are built from two halves:
- the backbone is torchvision's own alexnet().features / vgg16().features module, loaded with the seeded weights of
  femasr_b200.spec.random_lpips_state_dict (net.slice{s}.{i} -> features.{i}); this half is independent of the engine's
  oracle (tests/lpips_oracle.py);
- the head is written out below from the published LPIPS v0.1 definition (ScalingLayer, normalize_tensor, the lin layers'
  1x1 no-bias conv, spatial_average, the left-to-right sum), so it is pinned only to that definition.

Inputs are uint8 images (a smooth random field plus texture); x1 is either x0 plus small noise (SR-like) or an unrelated
image.  normalize=True feeds u8 / 255 (what pyiqa passes), normalize=False feeds u8 / 127.5 - 1.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from femasr_b200.spec import LPIPS_CONVS, random_lpips_state_dict  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lpips")

# name, net, weight seed, B, H, W, normalize, per image: "sr" (x0 + small noise) or "far" (unrelated)
CASES = [
    ("alex_b2_64x64", "alex", 1, 2, 64, 64, False, ("sr", "far")),
    ("alex_b1_67x93", "alex", 2, 1, 67, 93, True, ("far",)),
    ("alex_b1_256x256", "alex", 3, 1, 256, 256, True, ("sr",)),
    ("vgg_b2_32x48", "vgg", 4, 2, 32, 48, True, ("far", "sr")),
    ("vgg_b1_256x256", "vgg", 5, 1, 256, 256, False, ("sr",)),
]


def image_u8(g: torch.Generator, H: int, W: int) -> torch.Tensor:
    """[3,H,W] uint8: a bilinear-upsampled 6x6 random field plus fine texture."""
    low = torch.rand(1, 3, 6, 6, generator=g)
    smooth = F.interpolate(low, size=(H, W), mode="bilinear", align_corners=False)[0]
    x = smooth * 200 + torch.rand(3, H, W, generator=g) * 55
    return x.round().clamp(0, 255).to(torch.uint8)


def pair_u8(g: torch.Generator, B: int, H: int, W: int, kinds) -> tuple:
    x0 = torch.stack([image_u8(g, H, W) for _ in range(B)])
    x1 = torch.empty_like(x0)
    for b, kind in enumerate(kinds):
        if kind == "sr":
            noise = torch.randint(-24, 25, (3, H, W), generator=g, dtype=torch.int16)
            x1[b] = (x0[b].to(torch.int16) + noise).clamp(0, 255).to(torch.uint8)
        else:
            x1[b] = image_u8(g, H, W)
    return x0, x1


def to_input(u8: torch.Tensor, normalize: bool) -> torch.Tensor:
    return u8.float() / 255.0 if normalize else u8.float() / 127.5 - 1.0


def torchvision_features(net: str, sd) -> torch.nn.Module:
    import torchvision
    feats = (torchvision.models.alexnet() if net == "alex" else torchvision.models.vgg16()).features.eval()
    feats.load_state_dict({f"{i}.{p}": sd[f"net.slice{s}.{i}.{p}"] for s, i, *_ in LPIPS_CONVS[net]
                           for p in ("weight", "bias")}, strict=True)
    return feats


def taps_of(net: str, feats: torch.nn.Module, x: torch.Tensor):
    """The ReLU outputs after the last conv of each LPIPS slice (alex: features[1, 4, 7, 9, 11]; vgg: [3, 8, 15, 22, 29])."""
    ends = [i + 1 for s, i, *_ in LPIPS_CONVS[net] if all(s2 != s or i2 <= i for s2, i2, *_ in LPIPS_CONVS[net])]
    out = []
    for j, m in enumerate(feats[: ends[-1] + 1]):
        x = m(x)
        if j in ends:
            out.append(x)
    return out


def lpips_from_definition(net, sd, feats, in0, in1, normalize):
    if normalize:
        in0, in1 = 2 * in0 - 1, 2 * in1 - 1
    shift, scale = sd["scaling_layer.shift"], sd["scaling_layer.scale"]
    f0 = taps_of(net, feats, (in0 - shift) / scale)
    f1 = taps_of(net, feats, (in1 - shift) / scale)
    res = []
    for k, (a, b) in enumerate(zip(f0, f1)):
        na = a / (torch.sqrt(torch.sum(a ** 2, dim=1, keepdim=True)) + 1e-10)
        nb = b / (torch.sqrt(torch.sum(b ** 2, dim=1, keepdim=True)) + 1e-10)
        res.append(F.conv2d((na - nb) ** 2, sd[f"lin{k}.model.1.weight"]).mean([2, 3], keepdim=True))
    val = res[0]
    for r in res[1:]:
        val = val + r
    return val, res


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    os.makedirs(OUT, exist_ok=True)
    for name, net, seed, B, H, W, normalize, kinds in CASES:
        sd = random_lpips_state_dict(net, seed)
        feats = torchvision_features(net, sd)
        u0, u1 = pair_u8(torch.Generator().manual_seed(500 + seed), B, H, W, kinds)
        with torch.no_grad():
            d, res = lpips_from_definition(net, sd, feats, to_input(u0, normalize), to_input(u1, normalize), normalize)
        rec = dict(net=net, seed=seed, normalize=int(normalize), x0_u8=u0.numpy(), x1_u8=u1.numpy(),
                   d=d.view(B).numpy(), r=torch.stack([r.view(B) for r in res]).numpy())
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **rec)
        print(f"{name}: d {d.view(B).tolist()} -> {os.path.getsize(path) / 1e3:.0f} kB")


if __name__ == "__main__":
    main()
