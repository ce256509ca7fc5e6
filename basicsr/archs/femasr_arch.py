"""`FeMaSRNet` behind the reference's ARCH_REGISTRY surface, executed by the H100-native engine.

Drop-in for /root/reference/basicsr/archs/femasr_arch.py:214-479: same class name and registry key,
same keyword-only constructor, same state_dict keys and shapes (SURVEY.md 8b), same method signatures
and return tuples.  The module only HOLDS the parameters (so `.to()`, `.eval()`, `load_state_dict`,
`state_dict` behave as usual); all arithmetic of forward / encode_and_decode / test / test_tile /
decode_indices runs in libfemasr_b200.so (hand-written sm_90a CUDA) through `femasr_b200.net`.
There is no CPU or eager-PyTorch fallback: calling the network without a CUDA sm_90 (H100) device raises.

In scope: norm_type 'gn', act_type 'silu'; one codebook at scale 32 or the multi-scale variant with further codebooks
at 64 / 128 (femasr_arch.py:280-299); LQ_stage=True with scale_factor 2 or 4 (the SR network) and LQ_stage=False (the
HQ autoencoder that produces gt_indices / codebook visualisations); the gt_indices loss value (femasr_arch.py:84-90);
use_semantic_loss=True (the HQ-pretrain stage's VGG19 relu4_4 semantic loss, femasr_arch.py:301-309, 318-320, 344-347);
inference only (no autograd through the engine).  Anything else raises NotImplementedError at construction instead of
silently computing something different.
"""
from __future__ import annotations

import math
import os
import warnings

import numpy as np
import torch
from torch import nn

from basicsr.utils.registry import ARCH_REGISTRY
from femasr_b200.lib import FemasrError
from femasr_b200.module import EngineModule, attach
from femasr_b200.module import Node as _Node  # noqa: F401  (whole-module pickles name the containers by this path)
from femasr_b200.net import NativeNet
from femasr_b200.spec import (VGG_CONVS, VGG_TORCHVISION_INDEX, normalize_codebooks, param_spec, relative_position_index,
                              shift_attn_mask, vgg_init)

VGG_PRETRAIN_PATH = 'experiments/pretrained_models/vgg19-dcbb9e9d.pth'     # vgg_arch.py:9, relative to the working dir


def _vgg_pretrained():
    """The extractor's conv tensors from torchvision's vgg19 state_dict file (features.{0,2,5,...,25} -> conv1_1 ...
    conv4_4) when it exists, like the reference (vgg_arch.py:104-107); else None.  Never downloads."""
    if not os.path.exists(VGG_PRETRAIN_PATH):
        return None
    sd = torch.load(VGG_PRETRAIN_PATH, map_location="cpu")
    out = {}
    for (name, _ci, _co), i in zip(VGG_CONVS, VGG_TORCHVISION_INDEX):
        for t in ("weight", "bias"):
            out[f"vgg_feat_extractor.vgg_net.{name}.{t}"] = sd[f"features.{i}.{t}"].detach().float().clone()
    return out


def _init_tensor(shape, kind: str, fan_in: int, n_e: int) -> torch.Tensor:
    """Default initialisation with the reference's distributions (nn.Conv2d/nn.Linear kaiming-uniform
    a=sqrt(5) == U(+-1/sqrt(fan_in)) for weight and bias; GN/LN ones/zeros; rel-pos table
    trunc_normal(std=.02), network_swinir.py:111; codebook U(+-1/n_e), femasr_arch.py:33)."""
    if kind in ("w", "b"):
        bound = 1.0 / math.sqrt(fan_in)
        return torch.empty(shape).uniform_(-bound, bound)
    if kind == "norm_w":
        return torch.ones(shape)
    if kind == "norm_b":
        return torch.zeros(shape)
    if kind == "rpb":
        return nn.init.trunc_normal_(torch.zeros(shape), std=0.02)
    if kind == "codebook":
        return torch.empty(shape).uniform_(-1.0 / n_e, 1.0 / n_e)
    raise ValueError(kind)


@ARCH_REGISTRY.register()
class FeMaSRNet(EngineModule):
    def __init__(self, *, in_channel=3, codebook_params=None, gt_resolution=256, LQ_stage=False,
                 norm_type='gn', act_type='silu', use_quantize=True, scale_factor=4,
                 use_semantic_loss=False, use_residual=True, **ignore_kwargs):
        super().__init__(ignore_kwargs.get("gemm_path", -1))
        cb = np.array(codebook_params)
        if cb.ndim != 2 or cb.shape[1] != 3:
            raise ValueError("codebook_params must be [[scale, n_e, e_dim], ...]")
        unsupported = []
        try:
            self.codebooks = normalize_codebooks(cb.tolist())
            if len(self.codebooks) > 3 or any(n % 64 or e % 64 for _s, n, e in self.codebooks):
                unsupported.append("codebook sizes / dims that are not multiples of 64")
        except NotImplementedError as ex:
            unsupported.append(str(ex))
        if norm_type != 'gn' or act_type != 'silu':
            unsupported.append(f"norm_type={norm_type!r}/act_type={act_type!r}")
        if (LQ_stage and scale_factor not in (2, 4)) or gt_resolution != 256 or in_channel != 3:
            unsupported.append("LQ-stage scale_factor not in {2,4} / gt_resolution != 256 / in_channel != 3")
        if unsupported:
            raise NotImplementedError("femasr_b200 implements the inference hot path only; unsupported: "
                                      + "; ".join(unsupported))
        self.codebook_scale = cb[:, 0]
        self.n_e, self.e_dim = int(cb[0, 1]), int(cb[0, 2])
        self.use_quantize = use_quantize
        self.in_channel = in_channel
        self.gt_res = gt_resolution
        self.LQ_stage = LQ_stage
        self.scale_factor = scale_factor if LQ_stage else 1      # femasr_arch.py:241
        self.use_residual = use_residual
        self.use_semantic_loss = bool(use_semantic_loss)     # may be toggled like the reference's test() does (:451-452)
        self._semantic_params = bool(use_semantic_loss)      # whether conv_semantic / vgg_feat_extractor exist
        self.max_depth = int(np.log2(gt_resolution // self.codebook_scale[0]))

        vgg = None
        if self._semantic_params:
            vgg = _vgg_pretrained()
            if vgg is None:
                warnings.warn(f"use_semantic_loss: {VGG_PRETRAIN_PATH} not found; the VGG19 feature extractor is "
                              "initialised randomly (torchvision's VGG init). ImageNet VGG19 weights are expected from a "
                              "checkpoint; nothing is downloaded.", UserWarning, stacklevel=2)
        for name, shape, kind, fan_in in param_spec(self.scale_factor, self.e_dim, self.n_e, in_channel,
                                                    codebooks=self.codebooks, semantic=self._semantic_params):
            if kind == "rpi":
                attach(self, name, relative_position_index(), buffer=True)
            elif kind == "mask":
                attach(self, name, shift_attn_mask(32, 32), buffer=True)
            elif kind in ("vgg_mean", "vgg_std"):
                attach(self, name, vgg_init(shape, kind, fan_in), buffer=True)
            elif kind in ("vgg_w", "vgg_b"):
                t = vgg[name] if vgg is not None else vgg_init(shape, kind, fan_in)
                if tuple(t.shape) != tuple(shape):
                    raise ValueError(f"{VGG_PRETRAIN_PATH}: {name} has shape {tuple(t.shape)}, expected {tuple(shape)}")
                attach(self, name, t, buffer=False)
            else:
                attach(self, name, _init_tensor(shape, kind, fan_in, fan_in), buffer=False)   # codebook: fan_in = its n_e

    def _make_engine(self, gemm_path: int) -> NativeNet:
        return NativeNet(self.scale_factor, self.n_e, self.e_dim, self.use_quantize, self.use_residual,
                         gemm_path=gemm_path, codebooks=self.codebooks, use_semantic_loss=self._semantic_params)

    # ------------------------------------------------------------------ reference surface
    def encode_and_decode(self, input, gt_indices=None, current_iter=None):
        """femasr_arch.py:311-374 -> (out_img, codebook_loss, semantic_loss, [indices per codebook]).
        ``gt_indices`` (list, one map per codebook) switches codebook_loss to the supervised form (:84-90); the value
        is computed, no autograd graph is attached.  semantic_loss is the VGG19 relu4_4 loss (:344-347, 372) while
        ``use_semantic_loss`` is set, else codebook_loss * 0."""
        want_sem = bool(self.use_semantic_loss)
        if want_sem and not self._semantic_params:
            raise FemasrError("use_semantic_loss was switched on for a network built without it "
                              "(it has no conv_semantic / vgg_feat_extractor)")
        eng = self._native(input.device)
        if eng.use_graph and input.is_cuda and gt_indices is None and len(self.codebooks) == 1:
            # fixed launch list replayed as a CUDA graph; results are copied out of the graph's static buffers so the
            # returned tensors stay valid across calls like the reference's
            res = eng.forward_graph(input, want_sem=want_sem)
            if eng.last_from_graph:
                res = tuple(t.clone() for t in res)
        else:
            res = eng.forward(input, gt_indices=gt_indices, want_sem=want_sem)
        out, loss, idx = res[:3]
        sem = res[3] if want_sem else loss * 0
        return out, loss, sem, (idx if isinstance(idx, list) else [idx])

    def decode_indices(self, indices):
        """femasr_arch.py:376-385."""
        assert len(indices.shape) == 4, f'shape of indices must be (b, 1, h, w), but got {indices.shape}'
        return self._native(indices.device).decode_indices(indices)

    @torch.no_grad()
    def test_tile(self, input, tile_size=240, tile_pad=16):
        """femasr_arch.py:387-447."""
        return self._native(input.device).test_tile(input, tile_size, tile_pad)

    @torch.no_grad()
    def test(self, input):
        """femasr_arch.py:449-468."""
        return self._native(input.device).test(input)

    @torch.no_grad()
    def sr_uint8(self, images):
        """Extension (not in the reference): uint8 BGR HWC batch in, uint8 BGR HWC batch out, boundary fused on
        the device - img2tensor, /255, test() padding and crop, tensor2img (inference_femasr.py:54-64)."""
        return self._native(images.device).sr_uint8(images)

    @torch.no_grad()
    def encode_codes(self, input):
        """Extension: the codebook indices of `input` in the compact wire format (femasr_b200/wire.py: ceil(log2 n_e) bits
        per code, packed on the device) -> (uint8 stream, index-map shape [B,1,h,w]).  Single-codebook nets."""
        from femasr_b200.wire import pack_codes
        idx = self.encode_and_decode(input)[3]
        if len(idx) != 1:
            raise NotImplementedError("encode_codes: single-codebook networks only")
        return pack_codes(idx[0], self.n_e), tuple(idx[0].shape)

    @torch.no_grad()
    def decode_codes(self, packed, shape):
        """Extension: inverse of encode_codes - unpack on the device and run decode_indices (femasr_arch.py:376-385)."""
        from femasr_b200.wire import unpack_codes
        return self.decode_indices(unpack_codes(packed, tuple(shape), self.n_e))

    def forward(self, input, gt_indices=None):
        """femasr_arch.py:470-479."""
        return self.encode_and_decode(input, gt_indices)
