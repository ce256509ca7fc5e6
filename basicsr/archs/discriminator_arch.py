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
from femasr_b200.net import NativeDisc
from femasr_b200.spec import disc_spec


def _attach(root: nn.Module, dotted: str, tensor: torch.Tensor, buffer: bool):
    module, leaf = dotted.split(".")
    node = root._modules.get(module)
    if node is None:
        node = nn.Module()
        root.add_module(module, node)
    if buffer:
        node.register_buffer(leaf, tensor)
    else:
        node.register_parameter(leaf, nn.Parameter(tensor, requires_grad=False))


@ARCH_REGISTRY.register()
class UNetDiscriminatorSN(nn.Module):
    """U-Net discriminator with spectral normalisation (Real-ESRGAN), eval-mode forward on the engine."""

    def __init__(self, num_in_ch, num_feat=64, skip_connection=True, **ignore_kwargs):
        super().__init__()
        if num_in_ch != 3 or num_feat != 64:
            raise NotImplementedError("femasr_b200 runs UNetDiscriminatorSN with num_in_ch=3 and num_feat=64 only (the "
                                      f"shipped configuration); got num_in_ch={num_in_ch}, num_feat={num_feat}")
        self.num_in_ch, self.num_feat = num_in_ch, num_feat
        self.skip_connection = bool(skip_connection)
        self.gemm_path = int(ignore_kwargs.get("gemm_path", -1))    # -1: engine default
        for name, shape, kind, fan_in in disc_spec(num_in_ch, num_feat):
            if kind in ("sn_u", "sn_v"):
                # torch.nn.utils.spectral_norm: u, v = normalize(randn) buffers
                _attach(self, name, nn.functional.normalize(torch.randn(shape), dim=0, eps=1e-12), buffer=True)
            else:
                bound = 1.0 / fan_in ** 0.5          # nn.Conv2d's default init: U(+-1/sqrt(fan_in)) for weight and bias
                _attach(self, name, torch.empty(shape).uniform_(-bound, bound), buffer=False)
        self._engine = None
        self._engine_sig = None

    def load_state_dict(self, *a, **kw):
        out = super().load_state_dict(*a, **kw)
        self._engine_sig = None
        return out

    def __getstate__(self):
        # the engine is a process-local native handle: copies / pickles rebuild it lazily from the tensors
        state = self.__dict__.copy()
        state["_engine"] = None
        state["_engine_sig"] = None
        return state

    def _native(self, device: torch.device) -> NativeDisc:
        """The engine with the module's CURRENT tensors (re-uploaded when a (data_ptr, _version) changes)."""
        from femasr_b200 import default_gemm_path
        tensors = self.state_dict(keep_vars=True)
        sig = tuple((v.data_ptr(), v._version) for v in tensors.values())
        if self._engine is None:
            gp = self.gemm_path if self.gemm_path >= 0 else default_gemm_path()
            self._engine = NativeDisc(self.skip_connection, gp, self.num_in_ch, self.num_feat)
        if sig != self._engine_sig:
            self._engine.load_state_dict(tensors, device)
            self._engine_sig = sig
        return self._engine

    @torch.no_grad()
    def forward(self, x):
        """discriminator_arch.py forward: x [B,3,H,W] -> [B,1,H,W] fp32 (H, W multiples of 8)."""
        if self.training:
            raise FemasrError("UNetDiscriminatorSN.forward runs in eval mode only: in training mode the reference's "
                              "spectral_norm power-iterates and updates weight_u / weight_v in place, which the engine "
                              "does not do; call .eval() first")
        return self._native(x.device).forward(x)
