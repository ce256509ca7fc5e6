"""LPIPS v0.1 (Zhang et al., "The Unreasonable Effectiveness of Deep Features as a Perceptual Metric"; the `lpips`
package) computed on the engine: the validation metric and the perceptual-loss network of the training configs.

`LPIPS(net='alex' | 'vgg')` holds the `lpips` package's state_dict tensors under the same names
(scaling_layer.{shift,scale}, net.slice{1..5}.{i}.{weight,bias} with i the torchvision `features` index,
lin{0..4}.model.1.weight), so a combined LPIPS state_dict loads with `load_state_dict(strict=True)`.  The module only
HOLDS the tensors; forward runs in libfemasr_b200.so (hand-written sm_90a CUDA) through `femasr_b200.net.NativeLPIPS`.
There is no CPU or eager-PyTorch fallback.

pyiqa: per its documentation (not verified offline), `pyiqa.create_metric('lpips')` is this metric with net='alex'
and 'lpips-vgg' (the training configs' LPIPSLoss) the one with net='vgg'; pyiqa passes inputs in [0, 1], i.e.
normalize=True.

In scope: v0.1 with lpips=True and spatial=False, forward only (no gradients).  Nothing is ever downloaded: without
weight files the backbone gets torchvision's default init and the lins non-negative random values, with a UserWarning.
"""
from __future__ import annotations

import warnings
from typing import Dict, Optional

import torch

from .lib import FemasrError
from .module import EngineModule, attach
from .net import NativeLPIPS
from .spec import LPIPS_CONVS, lpips_spec, random_lpips_state_dict


def backbone_from_torchvision(net: str, sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """A torchvision alexnet / vgg16 state_dict (features.{i}.*; classifier.* is ignored) -> net.slice{s}.{i}.*.
    Raises naming every missing or unknown key."""
    want = {f"features.{i}.{p}": f"net.slice{s}.{i}.{p}" for s, i, *_ in LPIPS_CONVS[net] for p in ("weight", "bias")}
    unknown = sorted(k for k in sd if k not in want and not k.startswith("classifier."))
    missing = sorted(k for k in want if k not in sd)
    if unknown or missing:
        raise KeyError(f"torchvision {net} backbone file: missing keys {missing}, unknown keys {unknown}")
    return {want[k]: sd[k] for k in want}


def lins_from_lpips(net: str, sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """An lpips package lin-weights file (lin{k}.model.1.weight, e.g. its weights/v0.1/{net}.pth).  Raises naming every
    missing or unknown key."""
    want = [n for n, _s, kind, _f in lpips_spec(net) if kind == "lin"]
    unknown = sorted(k for k in sd if k not in want)
    missing = sorted(k for k in want if k not in sd)
    if unknown or missing:
        raise KeyError(f"lpips {net} lin-weights file: missing keys {missing}, unknown keys {unknown}")
    return {k: sd[k] for k in want}


class LPIPS(EngineModule):
    """The `lpips` package's LPIPS(net=net) (v0.1, lpips=True, spatial=False) in eval mode on the engine.

    backbone_path: a torchvision alexnet / vgg16 checkpoint (features.{i}.*); lin_path: an lpips lin-weights file
    (lin{k}.model.1.weight).  gemm_path -1 = the engine default (femasr_b200.default_gemm_path)."""

    def __init__(self, net: str = "alex", gemm_path: int = -1, version: str = "0.1", lpips: bool = True,
                 spatial: bool = False, backbone_path: Optional[str] = None, lin_path: Optional[str] = None,
                 **ignore_kwargs):
        super().__init__(gemm_path)
        if net not in ("alex", "vgg"):
            raise NotImplementedError(f"femasr_b200 computes LPIPS with net='alex' or 'vgg'; got net={net!r}")
        if version != "0.1" or not lpips or spatial:
            raise NotImplementedError("femasr_b200 computes LPIPS v0.1 with lpips=True and spatial=False only; got "
                                      f"version={version!r}, lpips={lpips}, spatial={spatial}")
        self.pnet_type = net
        tensors = random_lpips_state_dict(net)
        if backbone_path is None or lin_path is None:
            warnings.warn(f"LPIPS({net!r}): no {'backbone' if backbone_path is None else 'lin'} weight file given; "
                          "using untrained weights (nothing is downloaded) - the distances are not the published metric",
                          UserWarning, stacklevel=2)
        if backbone_path is not None:
            tensors.update(backbone_from_torchvision(net, torch.load(backbone_path, map_location="cpu")))
        if lin_path is not None:
            tensors.update(lins_from_lpips(net, torch.load(lin_path, map_location="cpu")))
        for name, _shape, kind, _f in lpips_spec(net):
            attach(self, name, tensors[name].float().contiguous(), buffer=kind in ("shift", "scale"))
        self.eval()

    def _make_engine(self, gemm_path: int) -> NativeLPIPS:
        return NativeLPIPS(self.pnet_type, gemm_path)

    @torch.no_grad()
    def forward(self, in0, in1, retPerLayer=False, normalize=False):
        """LPIPS.forward: in0, in1 [B,3,H,W] (in [-1, 1], or [0, 1] with normalize=True) -> d [B,1,1,1]; with
        retPerLayer (d, [r_0, ..., r_4]), each r_k [B,1,1,1].  vgg needs H, W multiples of 16, alex H, W >= 31."""
        if in0.shape != in1.shape:
            raise FemasrError(f"LPIPS: inputs of different shapes {tuple(in0.shape)} and {tuple(in1.shape)}")
        d, r = self._native(in0.device).forward(in0, in1.to(in0.device), normalize=bool(normalize))
        B = d.shape[0]
        val = d.view(B, 1, 1, 1)
        if retPerLayer:
            return val, [r[k].view(B, 1, 1, 1) for k in range(5)]
        return val
