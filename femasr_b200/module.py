"""The `nn.Module` side shared by every engine-backed network (FeMaSRNet, UNetDiscriminatorSN, LPIPS).

Such a module only HOLDS the reference's tensors under the reference's dotted names; its native handle
(`femasr_b200.net`) keeps repacked device copies of them.  `EngineModule` creates that handle on first use and uploads
the tensors again whenever one of them changes.
"""
from __future__ import annotations

import torch
from torch import nn

from . import default_gemm_path


class Node(nn.Module):
    """A bare container; a tree of these reproduces the reference's dotted tensor names."""


def attach(root: nn.Module, dotted: str, tensor: torch.Tensor, buffer: bool):
    """Register ``tensor`` under ``root`` as the buffer or (requires_grad=False) parameter named ``dotted``."""
    *path, leaf = dotted.split(".")
    node = root
    for part in path:
        child = node._modules.get(part)
        if child is None:
            child = Node()
            node.add_module(part, child)
        node = child
    if buffer:
        node.register_buffer(leaf, tensor)
    else:
        node.register_parameter(leaf, nn.Parameter(tensor, requires_grad=False))


class EngineModule(nn.Module):
    """Base of the engine-backed networks.  Subclasses build their tensor tree with `attach` and implement
    `_make_engine`; `_native(device)` returns the handle holding the module's current tensor values.

    A change is seen through each engine tensor's ``(data_ptr, _version)``: in-place updates, `load_state_dict`,
    `.to()` and assigning a new Parameter are all caught.  Writes through ``.data`` (BasicSR's model_ema) do not bump
    ``_version``, and replacing a whole submodule swaps the container the tensor is looked up in: call
    `refresh_weights()` after either."""

    # Class-level defaults: copies, pickles and whole-module pickles made before `_slots` existed start without a handle.
    _engine = None
    _engine_sig = None
    _slots = None           # per engine name, in engine order: (the container's parameter or buffer dict, leaf name)

    def __init__(self, gemm_path: int = -1):
        super().__init__()
        self.gemm_path = int(gemm_path)    # -1: femasr_b200.default_gemm_path()

    def _make_engine(self, gemm_path: int):
        """The subclass's `femasr_b200.net` handle (not yet created on a device)."""
        raise NotImplementedError

    def _slot(self, name: str):
        path, _, leaf = name.rpartition(".")
        node = self.get_submodule(path)
        return (node._parameters if leaf in node._parameters else node._buffers), leaf

    def _native(self, device: torch.device):
        """The engine with the module's CURRENT tensor values (re-uploaded when one changes)."""
        if self._engine is None:
            self._engine = self._make_engine(self.gemm_path if self.gemm_path >= 0 else default_gemm_path())
        if self._slots is None:
            self._slots = [self._slot(n) for n in self._engine.names]
        tensors = [store[leaf] for store, leaf in self._slots]
        sig = tuple((t.data_ptr(), t._version) for t in tensors)
        if sig != self._engine_sig:
            self._engine.load_state_dict(dict(zip(self._engine.names, tensors)), device)
            self._engine_sig = sig
        return self._engine

    def refresh_weights(self):
        """Upload every tensor again on the next call (after ``.data`` writes or a replaced submodule)."""
        self._engine_sig = None
        self._slots = None

    def load_state_dict(self, *a, **kw):
        out = super().load_state_dict(*a, **kw)
        self._engine_sig = None
        return out

    def __getstate__(self):
        # the engine is a process-local native handle: copies / pickles rebuild it lazily from the tensors
        state = self.__dict__.copy()
        for k in ("_engine", "_engine_sig", "_slots"):
            state.pop(k, None)
        return state
