"""The training configs' validation metrics on the engine, under pyiqa's names: PSNR and SSIM (hand-written sm_90a
kernels, femasr_b200/csrc/metrics.cu) and LPIPS (femasr_b200.lpips).

`create_metric(name, **opts)` stands in for `pyiqa.create_metric` as FeMaSRModel builds its metrics from a config's
`val.metrics` block (basicsr/models/femasr_model.py:28-34 of the reference): 'psnr', 'ssim', 'lpips' (AlexNet) and
'lpips-vgg' (VGG16).  Every metric is an nn.Module with forward(X, Y) -> [B] fp32, one score per image, on inputs in
[0, 1].  pyiqa's exact return shape is not known offline; a [B] tensor makes `.item()` work for B = 1, which is how
the model reads it.

The PSNR / SSIM definitions are pyiqa's as recalled, not verified offline (include/femasr_b200.h and DESIGN.md section 6
state them in full).  CUDA fp32 tensors only: there is no CPU fallback.
"""
from __future__ import annotations

import torch
from torch import nn

from . import lib as L
from .lpips import LPIPS

_COLOR_SPACES = {"yiq": L.METRIC_Y_YIQ, "ycbcr": L.METRIC_Y_YCBCR}
_CHECKED_DEVICES = set()      # CUDA device indices found to be sm_90


def _check_inputs(name: str, X: torch.Tensor, Y: torch.Tensor):
    if X.dim() != 4 or X.shape[1] != 3 or X.shape != Y.shape:
        raise L.FemasrError(f"{name}: expected two inputs [B,3,H,W] of one shape, got {tuple(X.shape)} and {tuple(Y.shape)}")
    if X.device.type != "cuda" or Y.device != X.device:
        raise L.FemasrError(f"{name}: femasr_b200 runs on a CUDA sm_90 (H100) device only (no CPU fallback); got inputs "
                            f"on '{X.device}' and '{Y.device}'")
    if X.dtype != torch.float32 or Y.dtype != torch.float32:
        raise L.FemasrError(f"{name}: expected fp32 inputs, got {X.dtype} and {Y.dtype}")


class _PixelMetric(nn.Module):
    _kind = None          # L.METRIC_PSNR / L.METRIC_SSIM
    _fn = None            # the C entry point

    def __init__(self, test_y_channel: bool, crop_border: int, color_space: str):
        super().__init__()
        if test_y_channel and color_space not in _COLOR_SPACES:
            raise ValueError(f"{self._name}: color_space must be 'yiq' or 'ycbcr'; got {color_space!r}")
        self.test_y_channel = bool(test_y_channel)
        self.crop_border = int(crop_border)
        self.color_space = color_space
        self.mode = _COLOR_SPACES[color_space] if test_y_channel else L.METRIC_RGB

    @torch.no_grad()
    def forward(self, X: torch.Tensor, Y: torch.Tensor) -> torch.Tensor:
        """X, Y [B,3,H,W] fp32 CUDA in [0, 1] -> [B] fp32, one score per image."""
        _check_inputs(self._name, X, Y)
        lib = L.load()
        X, Y = X.detach().contiguous(), Y.detach().contiguous()
        B, _, H, W = X.shape
        with torch.cuda.device(X.device):
            dev = torch.cuda.current_device()
            if dev not in _CHECKED_DEVICES:                    # cudaGetDeviceProperties costs milliseconds: once
                L.require_device()
                _CHECKED_DEVICES.add(dev)
            need = lib.femasr_metric_scratch_bytes(self._kind, B, H, W, self.crop_border)
            scratch = torch.empty(max(need, 8), dtype=torch.uint8, device=X.device)
            out = torch.empty(B, dtype=torch.float32, device=X.device)
            L.check(getattr(lib, self._fn)(X.data_ptr(), Y.data_ptr(), B, H, W, self.crop_border, self.mode,
                                           out.data_ptr(), scratch.data_ptr(), torch.cuda.current_stream().cuda_stream))
        return out

    def extra_repr(self):
        return f"test_y_channel={self.test_y_channel}, crop_border={self.crop_border}, color_space={self.color_space!r}"


class PSNR(_PixelMetric):
    """pyiqa's `psnr`: 10 log10(1 / (mse + 1e-8)) at data range 1, on the Y channel or the RGB channels."""
    _name, _kind, _fn = "psnr", L.METRIC_PSNR, "femasr_psnr"

    def __init__(self, test_y_channel: bool = False, crop_border: int = 0, color_space: str = "yiq"):
        super().__init__(test_y_channel, crop_border, color_space)


class SSIM(_PixelMetric):
    """pyiqa's `ssim`: Wang et al.'s SSIM at data range 255 (11x11 Gaussian, sigma 1.5, 'valid'), on the rounded Y
    channel or the RGB channels.  downsample=True is not implemented."""
    _name, _kind, _fn = "ssim", L.METRIC_SSIM, "femasr_ssim"

    def __init__(self, test_y_channel: bool = True, crop_border: int = 0, color_space: str = "yiq",
                 downsample: bool = False):
        if downsample:
            raise NotImplementedError("femasr_b200 computes SSIM with downsample=False only")
        super().__init__(test_y_channel, crop_border, color_space)


class LPIPSMetric(nn.Module):
    """pyiqa's `lpips` / `lpips-vgg` as a metric: inputs in [0, 1] (normalize=True) -> [B].  `net` is the LPIPS module
    (femasr_b200.lpips.LPIPS), so a combined state_dict loads with `metric.net.load_state_dict`."""

    def __init__(self, net: str, **lpips_opts):
        super().__init__()
        self.net = LPIPS(net, **lpips_opts)

    def forward(self, X: torch.Tensor, Y: torch.Tensor) -> torch.Tensor:
        return self.net(X, Y, normalize=True).view(-1)


_METRICS = {
    "psnr": (PSNR, {"test_y_channel", "crop_border", "color_space"}),
    "ssim": (SSIM, {"test_y_channel", "crop_border", "color_space", "downsample"}),
    "lpips": (lambda **o: LPIPSMetric("alex", **o), {"backbone_path", "lin_path", "gemm_path"}),
    "lpips-vgg": (lambda **o: LPIPSMetric("vgg", **o), {"backbone_path", "lin_path", "gemm_path"}),
}


def create_metric(name: str, as_loss: bool = False, device=None, **opts) -> nn.Module:
    """pyiqa.create_metric for the metrics of the training configs.  `better` is accepted and ignored (FeMaSRModel pops
    it); LPIPS weight files pass through as backbone_path / lin_path, since nothing is downloaded.  An unknown metric
    or option raises, naming it."""
    opts.pop("better", None)
    if name not in _METRICS:
        raise ValueError(f"create_metric: unknown metric {name!r}; femasr_b200 has {sorted(_METRICS)}")
    if as_loss:
        raise NotImplementedError(f"create_metric({name!r}, as_loss=True): femasr_b200 computes metrics without gradients")
    make, allowed = _METRICS[name]
    unknown = sorted(set(opts) - allowed)
    if unknown:
        raise TypeError(f"create_metric({name!r}): unknown option(s) {unknown}; allowed {sorted(allowed)}")
    metric = make(**opts).eval()
    return metric.to(device) if device is not None else metric
