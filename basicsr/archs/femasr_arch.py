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
inference only (no autograd through the engine).  Anything else raises NotImplementedError at construction instead of
silently computing something different.
"""
from __future__ import annotations

import math

import numpy as np
import torch
from torch import nn

from basicsr.utils.registry import ARCH_REGISTRY
from femasr_b200.net import NativeNet
from femasr_b200.spec import normalize_codebooks, param_spec, relative_position_index, shift_attn_mask


class _Node(nn.Module):
    """A bare container; the tree of these reproduces the reference's dotted parameter names."""


def _attach(root: nn.Module, dotted: str, tensor: torch.Tensor, buffer: bool):
    *path, leaf = dotted.split(".")
    node = root
    for part in path:
        nxt = node._modules.get(part)
        if nxt is None:
            nxt = _Node()
            node.add_module(part, nxt)
        node = nxt
    if buffer:
        node.register_buffer(leaf, tensor)
    else:
        node.register_parameter(leaf, nn.Parameter(tensor, requires_grad=False))


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
class FeMaSRNet(nn.Module):
    def __init__(self, *, in_channel=3, codebook_params=None, gt_resolution=256, LQ_stage=False,
                 norm_type='gn', act_type='silu', use_quantize=True, scale_factor=4,
                 use_semantic_loss=False, use_residual=True, **ignore_kwargs):
        super().__init__()
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
        if use_semantic_loss:
            unsupported.append("use_semantic_loss=True (training-only VGG branch)")
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
        self.use_semantic_loss = False
        self.max_depth = int(np.log2(gt_resolution // self.codebook_scale[0]))
        self.gemm_path = int(ignore_kwargs.get("gemm_path", -1))    # -1: engine default

        for name, shape, kind, fan_in in param_spec(self.scale_factor, self.e_dim, self.n_e, in_channel,
                                                    codebooks=self.codebooks):
            if kind == "rpi":
                _attach(self, name, relative_position_index(), buffer=True)
            elif kind == "mask":
                _attach(self, name, shift_attn_mask(32, 32), buffer=True)
            else:
                _attach(self, name, _init_tensor(shape, kind, fan_in, fan_in), buffer=False)   # codebook: fan_in = its n_e
        self._engine = None
        self._engine_sig = None
        self._plist = None

    # ------------------------------------------------------------------ engine plumbing
    def _float_params(self):
        return {k: v for k, v in self.state_dict(keep_vars=True).items() if v.dtype == torch.float32
                and not k.endswith("attn_mask")}

    def _param_list(self):
        """(name, tensor) pairs of the engine's parameters, cached: walking state_dict() costs ~1 ms per call (437
        tensors), which the reference's batch-1 loop would pay per image.  Invalidated whenever the tensor OBJECTS may
        have been replaced: `_apply` (.to/.cuda/.float/...), `load_state_dict`."""
        if self._plist is None:
            self._plist = list(self._float_params().items())
        return self._plist

    def _apply(self, fn, *a, **kw):
        out = super()._apply(fn, *a, **kw)
        self._plist = None
        return out

    def load_state_dict(self, *a, **kw):
        out = super().load_state_dict(*a, **kw)
        self._plist = None
        self._engine_sig = None
        return out

    def refresh_weights(self):
        """Force a re-upload of the parameters on the next call.  Needed only after in-place surgery that bypasses
        autograd's version counter (`p.data.copy_(...)`, e.g. BasicSR's model_ema): `(data_ptr, _version)` is how
        changes are detected, and `.data` writes do not bump `_version`."""
        self._plist = None
        self._engine_sig = None

    def _native(self, device: torch.device) -> NativeNet:
        """The engine with the module's CURRENT parameter values (re-uploaded when they change)."""
        from femasr_b200 import default_gemm_path
        plist = self._param_list()
        sig = tuple((v.data_ptr(), v._version) for _k, v in plist)      # ~0.07 ms (was ~1.1 ms through state_dict())
        if self._engine is None:
            gp = self.gemm_path if self.gemm_path >= 0 else default_gemm_path()
            self._engine = NativeNet(self.scale_factor, self.n_e, self.e_dim, self.use_quantize,
                                     self.use_residual, gemm_path=gp, codebooks=self.codebooks)
        if sig != self._engine_sig:
            self._engine.load_state_dict(dict(plist), device)
            self._engine_sig = sig
        return self._engine

    def __getstate__(self):
        # the engine is a process-local native handle: copies / pickles rebuild it lazily from the parameters
        state = self.__dict__.copy()
        state["_engine"] = None
        state["_engine_sig"] = None
        state["_plist"] = None
        return state

    # ------------------------------------------------------------------ reference surface
    def encode_and_decode(self, input, gt_indices=None, current_iter=None):
        """femasr_arch.py:311-374 -> (out_img, codebook_loss, semantic_loss, [indices per codebook]).
        ``gt_indices`` (list, one map per codebook) switches codebook_loss to the supervised form (:84-90); the value
        is computed, no autograd graph is attached."""
        eng = self._native(input.device)
        if eng.use_graph and input.is_cuda and gt_indices is None and len(self.codebooks) == 1:
            # fixed launch list replayed as a CUDA graph; results are copied out of the graph's static buffers so the
            # returned tensors stay valid across calls like the reference's
            out, loss, idx = eng.forward_graph(input)
            if eng.last_from_graph:
                out, loss, idx = out.clone(), loss.clone(), idx.clone()
        else:
            out, loss, idx = eng.forward(input, gt_indices=gt_indices)
        return out, loss, loss * 0, (idx if isinstance(idx, list) else [idx])

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
