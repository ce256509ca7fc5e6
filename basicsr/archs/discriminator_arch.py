"""`UNetDiscriminatorSN` behind the reference's ARCH_REGISTRY surface, executed by the H100-native engine.

Drop-in for basicsr/archs/discriminator_arch.py of the reference (the training configs' ``network_d``): same class name
and registry key, same constructor, the same 28 state_dict tensors (conv0 / conv9 weight and bias; weight_orig,
weight_u and weight_v of the spectral_norm convs conv1 ... conv8), so a reference checkpoint such as
FeMaSR_HRP_model_d.pth loads with strict=True.  The module only HOLDS the tensors; forward runs in libfemasr_b200.so
(hand-written sm_90a CUDA) through `femasr_b200.net.NativeDisc`.  There is no CPU or eager-PyTorch fallback.

In scope: eval mode (sigma = u . (W v) from the stored u, v, no power iteration), num_in_ch 3, num_feat 64, either
skip_connection.  Training mode would power-iterate and update u, v in place; it raises instead.
"""
from __future__ import annotations

import torch
from torch import nn

from basicsr.utils.registry import ARCH_REGISTRY
from femasr_b200.lib import FemasrError
from femasr_b200.module import EngineModule, attach
from femasr_b200.net import NativeDisc
from femasr_b200.spec import disc_spec


@ARCH_REGISTRY.register()
class UNetDiscriminatorSN(EngineModule):
    """U-Net discriminator with spectral normalisation (Real-ESRGAN), eval-mode forward on the engine."""

    def __init__(self, num_in_ch, num_feat=64, skip_connection=True, **ignore_kwargs):
        super().__init__(ignore_kwargs.get("gemm_path", -1))
        if num_in_ch != 3 or num_feat != 64:
            raise NotImplementedError("femasr_b200 runs UNetDiscriminatorSN with num_in_ch=3 and num_feat=64 only (the "
                                      f"shipped configuration); got num_in_ch={num_in_ch}, num_feat={num_feat}")
        self.num_in_ch, self.num_feat = num_in_ch, num_feat
        self.skip_connection = bool(skip_connection)
        for name, shape, kind, fan_in in disc_spec(num_in_ch, num_feat):
            if kind in ("sn_u", "sn_v"):
                # torch.nn.utils.spectral_norm: u, v = normalize(randn) buffers
                attach(self, name, nn.functional.normalize(torch.randn(shape), dim=0, eps=1e-12), buffer=True)
            else:
                bound = 1.0 / fan_in ** 0.5          # nn.Conv2d's default init: U(+-1/sqrt(fan_in)) for weight and bias
                attach(self, name, torch.empty(shape).uniform_(-bound, bound), buffer=False)

    def _make_engine(self, gemm_path: int) -> NativeDisc:
        return NativeDisc(self.skip_connection, gemm_path, self.num_in_ch, self.num_feat)

    @torch.no_grad()
    def forward(self, x):
        """discriminator_arch.py forward: x [B,3,H,W] -> [B,1,H,W] fp32 (H, W multiples of 8)."""
        if self.training:
            raise FemasrError("UNetDiscriminatorSN.forward runs in eval mode only: in training mode the reference's "
                              "spectral_norm power-iterates and updates weight_u / weight_v in place, which the engine "
                              "does not do; call .eval() first")
        return self._native(x.device).forward(x)
