"""Host side of the H100-native FeMaSR path: owns the C engine handle, the device workspace and the
test()/test_tile() scheduling.  PyTorch is used for device memory and the current stream only; all
arithmetic happens in libfemasr_b200.so through the C ABI (include/femasr_b200.h).

Mirrors the reference operator surface for this path (femasr_arch.py:311-479):
encode_and_decode/forward -> NativeNet.forward, test -> NativeNet.test, test_tile -> NativeNet.test_tile,
decode_indices -> NativeNet.decode_indices; UNetDiscriminatorSN.forward (discriminator_arch.py) -> NativeDisc.forward;
the lpips package's LPIPS.forward -> NativeLPIPS.forward.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from collections import OrderedDict
from typing import Dict, List, Optional, Tuple

import torch

from . import lib as L
from .spec import disc_spec, lpips_spec, normalize_codebooks, param_spec


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def tile_plan(height: int, width: int, tile_size: int, tile_pad: int) -> List[dict]:
    """Tile windows of test_tile (femasr_arch.py:401-441): input window with halo clamped to the image,
    output window, and the crop (offset inside the tile output, size), all in LR pixels."""
    plan = []
    for ty in range(math.ceil(height / tile_size)):
        for tx in range(math.ceil(width / tile_size)):
            x0, y0 = tx * tile_size, ty * tile_size
            x1, y1 = min(x0 + tile_size, width), min(y0 + tile_size, height)
            px0, px1 = max(x0 - tile_pad, 0), min(x1 + tile_pad, width)
            py0, py1 = max(y0 - tile_pad, 0), min(y1 + tile_pad, height)
            plan.append({"in": (py0, py1, px0, px1), "out": (y0, y1, x0, x1), "crop": (y0 - py0, x0 - px0)})
    return plan


def padded_size(n: int, scale: int) -> int:
    """test() always pads to the NEXT multiple of wsz = 8//scale*8, even when n is one (femasr_arch.py:455-458)."""
    wsz = 8 // scale * 8
    return (n // wsz + 1) * wsz


class _Engine:
    """What every engine handle shares: creation on first use on a CUDA device, the parameter upload by reference name,
    the device workspace and the per-kernel profile.  Subclasses set ``lib``, ``_h``, ``_ws``, ``device``, ``names``
    and implement ``_create``."""

    def _create(self):
        raise NotImplementedError

    # ------------------------------------------------------------------ lifecycle
    def _ensure(self, device: torch.device):
        if device.type != "cuda":
            raise L.FemasrError("femasr_b200 runs on a CUDA sm_90 (H100) device only (no CPU fallback); "
                                f"got tensors on '{device}'")
        if self._h.value is None:
            with torch.cuda.device(device):
                L.require_device()
                self._create()
            self.device = device
        elif device != self.device:
            raise L.FemasrError(f"engine lives on {self.device}, input is on {device}")

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value is not None:
            self.lib.femasr_net_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def load_state_dict(self, sd: Dict[str, torch.Tensor], device: torch.device):
        """Upload every float parameter by its reference name (engine keeps repacked device copies)."""
        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self._ensure(device)
        with torch.cuda.device(device):
            for name in self.names:
                if name not in sd:
                    raise L.FemasrError(f"state_dict is missing '{name}'")
                t = sd[name].detach()
                if t.dtype != torch.float32:
                    t = t.float()
                t = t.contiguous()
                on_dev = t.device.type == "cuda"
                if on_dev and t.device != device:
                    t = t.to(device)
                L.check(self.lib.femasr_net_set_param(self._h, name.encode(), t.data_ptr(), t.numel(),
                                                      int(on_dev), _stream()))
            L.check(self.lib.femasr_net_params_complete(self._h))
            torch.cuda.current_stream().synchronize()

    def _workspace(self, nbytes: int) -> torch.Tensor:
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = None
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        return self._ws

    def set_profile(self, enable: bool):
        L.check(self.lib.femasr_net_set_profile(self._h, int(enable)))

    def profile(self) -> dict:
        """{kernel: {launches, ms, flops}} of the launches since set_profile(True) (CUDA-event timed)."""
        import json
        return json.loads(self.lib.femasr_net_profile_json(self._h).decode())

    def last_launch_count(self) -> int:
        return int(self.lib.femasr_net_last_launch_count(self._h))


class NativeNet(_Engine):
    def __init__(self, scale_factor: int, n_e: int, e_dim: int, use_quantize: bool = True,
                 use_residual: bool = True, gemm_path: int = 0, codebooks=None, use_semantic_loss: bool = False):
        """``codebooks``: the reference's ``codebook_params`` rows [[scale, n_e, e_dim], ...] for the multi-scale
        variant (femasr_arch.py:231-235); default one codebook (32, n_e, e_dim).  ``use_semantic_loss``: the engine also
        holds the VGG19 / conv_semantic tensors (femasr_arch.py:301-309) and forward(want_sem=True) computes the HQ
        stage's semantic loss."""
        self.lib = L.load()
        self.scale = int(scale_factor)
        self.codebooks = normalize_codebooks(codebooks, n_e, e_dim)
        self.n_e, self.e_dim = self.codebooks[0][1], self.codebooks[0][2]
        K = len(self.codebooks)
        pad = lambda v: (C.c_int * 3)(*(list(v) + [0] * (3 - K)))
        self.cfg = L.NetConfig(self.scale, self.n_e, self.e_dim, 3, int(bool(use_quantize)),
                               int(bool(use_residual)), int(gemm_path), K, pad([c[0] for c in self.codebooks]),
                               pad([c[1] for c in self.codebooks]), pad([c[2] for c in self.codebooks]))
        self._h = C.c_void_p()
        self._ws: Optional[torch.Tensor] = None
        self._taps: Dict[str, torch.Tensor] = {}
        self.device: Optional[torch.device] = None
        self.use_semantic_loss = bool(use_semantic_loss)
        self.names = [n for (n, _s, kind, _f) in param_spec(self.scale, self.e_dim, self.n_e, codebooks=self.codebooks,
                                                             semantic=self.use_semantic_loss)
                      if kind not in ("rpi", "mask")]
        # the forward is a fixed launch list per input shape: replay it as a CUDA graph (no per-launch host work)
        self.use_graph = os.environ.get("FEMASR_CUDA_GRAPH", "1") != "0"
        # Captured graphs pin their workspace and static buffers (13 GB at 32x128x128), so the cache is a small LRU and
        # a shape is captured only when it comes back: a folder of 38 differently sized images (the reference's testset)
        # runs eagerly on the ONE shared workspace instead of accumulating 38 graphs.
        self.graph_cache_size = max(0, int(os.environ.get("FEMASR_GRAPH_CACHE", "4")))
        self._graphs: "OrderedDict[Tuple[int, ...], dict]" = OrderedDict()
        self._seen_shapes: "OrderedDict[Tuple[int, ...], int]" = OrderedDict()
        self.last_from_graph = False     # whether the last forward_graph() result lives in a graph's static buffers

    def _create(self):
        L.check(self.lib.femasr_net_create(C.byref(self.cfg), C.byref(self._h)))
        if self.use_semantic_loss:
            L.check(self.lib.femasr_net_enable_semantic(self._h))

    def load_state_dict(self, sd: Dict[str, torch.Tensor], device: torch.device):
        self._graphs.clear()           # captured graphs hold the old weight pointers' contents only by address: re-capture
        super().load_state_dict(sd, device)

    # ------------------------------------------------------------------ graph entry points
    def index_shapes(self, B: int, H: int, W: int) -> List[Tuple[int, int, int, int]]:
        """Shapes of the per-codebook index maps for a [B,3,H,W] input."""
        div = {4: 2, 2: 4, 1: 8}[self.scale]
        h, w = H // div, W // div
        return [(B, 1, h * cs // 32, w * cs // 32) for cs, _n, _e in self.codebooks]

    def forward(self, x: torch.Tensor, want_indices: bool = True, want_loss: bool = True,
                taps: Optional[List[str]] = None, gt_indices=None, want_sem: bool = False):
        """encode_and_decode.  x [B,3,H,W] fp32 cuda -> (y [B,3,sH,sW], loss scalar tensor | None,
        indices [B,1,h,w] int64 | None[, sem][, {stage: NHWC tensor}]); multi-scale nets return a list of index maps, one
        per codebook.  ``gt_indices`` (tensor or list, one map per codebook) selects the supervised loss of
        femasr_arch.py:84-90 (LQ stage).  ``want_sem``: also the semantic loss (scalar tensor, femasr_arch.py:344-347,
        372), returned after the indices; needs use_semantic_loss and the HQ stage with one codebook of e_dim 512."""
        if x.dim() != 4 or x.shape[1] != 3:
            raise L.FemasrError(f"expected input [B,3,H,W], got {tuple(x.shape)}")
        self._ensure(x.device)
        x = x.detach()
        if x.dtype != torch.float32:
            x = x.float()
        x = x.contiguous()
        B, _, H, W = x.shape
        s = self.scale
        with torch.cuda.device(self.device):
            y = torch.empty((B, 3, H * s, W * s), dtype=torch.float32, device=self.device)
            div = {4: 2, 2: 4, 1: 8}[s]
            h, w = H // div, W // div
            ishapes = self.index_shapes(B, H, W)
            isizes = [math.prod(sh) for sh in ishapes]
            flat = torch.empty(sum(isizes), dtype=torch.int64, device=self.device) if want_indices else None
            idx = None
            if want_indices:
                parts = [p.view(sh) for p, sh in zip(torch.split(flat, isizes), ishapes)]
                idx = parts[0] if len(parts) == 1 else parts
            gt = None
            if gt_indices is not None:
                gl = [gt_indices] if torch.is_tensor(gt_indices) else list(gt_indices)
                if len(gl) != len(ishapes) or any(g.numel() != n for g, n in zip(gl, isizes)):
                    raise L.FemasrError(f"gt_indices must hold one map per codebook with {isizes} entries")
                for g_, (_cs, ne_, _e) in zip(gl, self.codebooks):
                    self._check_index_range(g_, ne_, "forward(gt_indices)")
                gt = torch.cat([g.detach().to(self.device, torch.int64).reshape(-1) for g in gl]).contiguous()
            loss = torch.empty((), dtype=torch.float32, device=self.device) if want_loss else None
            if want_sem and not self.use_semantic_loss:
                raise L.FemasrError("the semantic loss needs an engine built with use_semantic_loss=True")
            sem = torch.empty((), dtype=torch.float32, device=self.device) if want_sem else None
            tap_out = {}
            if taps:
                shapes = self.tap_shapes(B, H, W)
                for name in taps:
                    t = torch.empty(shapes[name], dtype=torch.float32, device=self.device)
                    tap_out[name] = t
                    L.check(self.lib.femasr_net_set_tap(self._h, name.encode(), t.data_ptr(), t.numel()))
            # sized AFTER the taps are registered: the engine's plan (and so its workspace) depends on them
            need = C.c_size_t()
            try:
                L.check(self.lib.femasr_net_workspace_bytes_sem(self._h, B, H, W, int(want_sem), C.byref(need)))
                ws = self._workspace(need.value)
                L.check(self.lib.femasr_net_forward_sem(self._h, x.data_ptr(), y.data_ptr(), _ptr(flat), _ptr(loss),
                                                        _ptr(gt), _ptr(sem), B, H, W, ws.data_ptr(), ws.numel(),
                                                        _stream()))
            finally:
                for name in tap_out:
                    self.lib.femasr_net_set_tap(self._h, name.encode(), None, 0)
        res = (y, loss, idx) + ((sem,) if want_sem else ())
        if taps:
            return res + (tap_out,)
        return res

    def forward_graph(self, x: torch.Tensor, want_sem: bool = False):
        """encode_and_decode through a captured CUDA graph.  Returns (y, loss, idx), with ``want_sem`` (y, loss, idx, sem);
        when they come out of a graph they live in its static output buffers: valid until the next call with the same
        shape (clone to keep).
        Policy: the first sighting of a shape runs eagerly (shared workspace); the second captures; at most
        ``graph_cache_size`` graphs are kept (least recently used evicted, its workspace and buffers freed)."""
        self._ensure(x.device)
        x = x.detach().float().contiguous()
        key = tuple(x.shape) + (("sem",) if want_sem else ())
        ent = self._graphs.get(key)
        if ent is None:
            seen = self._seen_shapes.pop(key, 0) + 1
            self._seen_shapes[key] = seen
            while len(self._seen_shapes) > 64:
                self._seen_shapes.popitem(last=False)
            if seen < 2 or self.graph_cache_size == 0:
                self.last_from_graph = False
                return self.forward(x, want_sem=want_sem)
            while len(self._graphs) >= self.graph_cache_size:
                self._graphs.popitem(last=False)          # drops the graph, its workspace and static buffers
            with torch.cuda.device(self.device):
                xs = torch.empty_like(x)
                xs.copy_(x)
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    self.forward(xs, want_sem=want_sem)   # warm-up: one-time attribute/workspace set-up happens here
                    side.synchronize()
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g, stream=side):
                        outs = self.forward(xs, want_sem=want_sem)
                torch.cuda.current_stream().wait_stream(side)
                ent = {"graph": g, "x": xs, "outs": outs, "ws": self._ws}
                self._ws = None                           # the captured launches own this workspace from now on
                self._graphs[key] = ent
        else:
            self._graphs.move_to_end(key)
        self.last_from_graph = True
        ent["x"].copy_(x, non_blocking=True)
        ent["graph"].replay()
        return ent["outs"]

    def release_graphs(self):
        """Drop every captured graph (and the workspaces they pin)."""
        self._graphs.clear()
        self._seen_shapes.clear()

    def tap_shapes(self, B: int, H: int, W: int) -> Dict[str, Tuple[int, ...]]:
        s = self.scale
        div = {4: 2, 2: 4, 1: 8}[s]
        h, w = H // div, W // div
        c0 = {4: 256, 2: 128, 1: 64}[s]
        return {"in_conv": (B, H - 1, W - 1, c0), "down": (B, h, w, 256), "swin": (B, h, w, 256),
                "up1": (B, 2 * h, 2 * w, 256), "up2": (B, 4 * h, 4 * w, 128), "z": (B, h, w, self.e_dim),
                "zq": (B, h, w, self.e_dim), "after_quant": (B, h, w, 256), "dec0": (B, 2 * h, 2 * w, 256),
                "dec1": (B, 4 * h, 4 * w, 128), "dec2": (B, 8 * h, 8 * w, 64),
                "vgg": (B, H // 8, W // 8, 512), "semantic": (B, h, w, 512),
                **{f"z{k}": (B, h * cs // 32, w * cs // 32, e) for k, (cs, _n, e) in enumerate(self.codebooks) if k}}

    def decode_indices(self, indices: torch.Tensor) -> torch.Tensor:
        assert indices.dim() == 4, f"shape of indices must be (b, 1, h, w), but got {indices.shape}"
        self._ensure(indices.device)
        idx = indices.detach().to(torch.int64).contiguous()
        B, _, h, w = idx.shape
        self._check_index_range(idx, self.n_e, "decode_indices")
        with torch.cuda.device(self.device):
            need = C.c_size_t()
            L.check(self.lib.femasr_net_decode_workspace_bytes(self._h, B, h, w, C.byref(need)))
            ws = self._workspace(need.value)
            y = torch.empty((B, 3, 8 * h, 8 * w), dtype=torch.float32, device=self.device)
            L.check(self.lib.femasr_net_decode_indices(self._h, idx.data_ptr(), y.data_ptr(), B, h, w,
                                                       ws.data_ptr(), ws.numel(), _stream()))
        return y

    @staticmethod
    def _check_index_range(idx: torch.Tensor, n_e: int, what: str):
        """The reference raises on an index outside the codebook (scatter_ in get_codebook_entry / the gt one-hot,
        femasr_arch.py:70-78,102-112); the kernels clamp for memory safety, so the range is checked here."""
        if idx.numel():
            lo, hi = int(idx.min()), int(idx.max())
            if lo < 0 or hi >= n_e:
                raise L.FemasrError(f"{what}: codebook index out of range [0, {n_e}): min {lo}, max {hi}")

    def flops(self, B: int, H: int, W: int) -> float:
        return float(self.lib.femasr_net_flops(self._h, B, H, W))

    # ------------------------------------------------------------------ test() / test_tile()
    def test(self, x: torch.Tensor) -> torch.Tensor:
        """femasr_arch.py:449-468: flip-pad, encode_and_decode, crop."""
        self._ensure(x.device)
        x = x.detach().float().contiguous()
        B, Cc, h, w = x.shape
        s = self.scale
        hp, wp = padded_size(h, s), padded_size(w, s)
        with torch.cuda.device(self.device):
            xp = torch.empty((B, Cc, hp, wp), dtype=torch.float32, device=self.device)
            L.check(self.lib.femasr_flip_pad(x.data_ptr(), xp.data_ptr(), B, Cc, h, w, hp, wp, _stream()))
            yp, _, _ = self.forward(xp, want_indices=False, want_loss=False)
            y = torch.empty((B, 3, h * s, w * s), dtype=torch.float32, device=self.device)
            L.check(self.lib.femasr_copy_window(yp.data_ptr(), y.data_ptr(), B, 3, hp * s, wp * s, h * s, w * s,
                                                0, 0, 0, 0, h * s, w * s, _stream()))
        return y

    def sr_uint8(self, images: torch.Tensor) -> torch.Tensor:
        """Whole-image SR with the uint8 boundary on the device: images uint8 [B,h,w,3] BGR (what cv2.imread
        returns, stacked) on the GPU -> uint8 [B,s*h,s*w,3] BGR.  Equals tensor2img(test(img2tensor(img)/255.))
        of the reference's inference loop (inference_femasr.py:54-64) for same-shape images, with one quarter of
        the device->host bytes and no host-side float image math."""
        if images.dtype != torch.uint8 or images.dim() != 4 or images.shape[3] != 3:
            raise L.FemasrError(f"expected uint8 [B,h,w,3], got {images.dtype} {tuple(images.shape)}")
        self._ensure(images.device)
        images = images.contiguous()
        B, h, w, _ = images.shape
        s = self.scale
        hp, wp = padded_size(h, s), padded_size(w, s)
        with torch.cuda.device(self.device):
            xp = torch.empty((B, 3, hp, wp), dtype=torch.float32, device=self.device)
            L.check(self.lib.femasr_u8_to_input(images.data_ptr(), xp.data_ptr(), B, h, w, hp, wp, _stream()))
            yp = (self.forward_graph(xp) if self.use_graph else self.forward(xp, want_indices=False, want_loss=False))[0]
            out = torch.empty((B, h * s, w * s, 3), dtype=torch.uint8, device=self.device)
            L.check(self.lib.femasr_output_to_u8(yp.data_ptr(), out.data_ptr(), B, hp * s, wp * s, h * s, w * s, _stream()))
        return out

    def test_tile(self, x: torch.Tensor, tile_size: int = 240, tile_pad: int = 16,
                  max_batch: int = 64) -> torch.Tensor:
        """femasr_arch.py:387-447.  Tiles are independent (every op on the path is per-sample), so
        same-shape tiles are stacked into one batch per forward instead of the reference's
        one-tile-at-a-time loop; results are identical per tile."""
        self._ensure(x.device)
        x = x.detach().float().contiguous()
        B, Cc, H, W = x.shape
        s = self.scale
        plan = tile_plan(H, W, tile_size, tile_pad)
        groups: Dict[Tuple[int, int], List[dict]] = {}
        for t in plan:
            py0, py1, px0, px1 = t["in"]
            groups.setdefault((py1 - py0, px1 - px0), []).append(t)
        with torch.cuda.device(self.device):
            out = torch.zeros((B, Cc, H * s, W * s), dtype=torch.float32, device=self.device)
            st = _stream()
            for (th, tw), tiles in groups.items():
                per = max(1, max_batch // B)
                for i in range(0, len(tiles), per):
                    chunk = tiles[i:i + per]
                    tb = torch.empty((len(chunk) * B, Cc, th, tw), dtype=torch.float32, device=self.device)
                    for k, t in enumerate(chunk):
                        py0, _py1, px0, _px1 = t["in"]
                        dst = tb.data_ptr() + k * B * Cc * th * tw * 4
                        L.check(self.lib.femasr_copy_window(x.data_ptr(), dst, B, Cc, H, W, th, tw,
                                                            py0, px0, 0, 0, th, tw, st))
                    yt = self.test(tb)
                    for k, t in enumerate(chunk):
                        y0, y1, x0, x1 = t["out"]
                        cy, cx = t["crop"]
                        src = yt.data_ptr() + k * B * Cc * th * s * tw * s * 4
                        L.check(self.lib.femasr_copy_window(src, out.data_ptr(), B, Cc, th * s, tw * s, H * s, W * s,
                                                            cy * s, cx * s, y0 * s, x0 * s, (y1 - y0) * s,
                                                            (x1 - x0) * s, st))
        return out


class NativeDisc(_Engine):
    """UNetDiscriminatorSN (discriminator_arch.py) on the engine: forward(x [B,3,H,W]) -> [B,1,H,W], eval mode."""

    def __init__(self, skip_connection: bool = True, gemm_path: int = 0, num_in_ch: int = 3, num_feat: int = 64):
        self.lib = L.load()
        self.dcfg = L.DiscConfig(int(num_in_ch), int(num_feat), int(bool(skip_connection)), int(gemm_path))
        self._h = C.c_void_p()
        self._ws: Optional[torch.Tensor] = None
        self.device: Optional[torch.device] = None
        self.names = [n for (n, _s, _k, _f) in disc_spec(num_in_ch, num_feat)]

    def _create(self):
        L.check(self.lib.femasr_disc_create(C.byref(self.dcfg), C.byref(self._h)))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if x.dim() != 4 or x.shape[1] != self.dcfg.num_in_ch:
            raise L.FemasrError(f"expected input [B,{self.dcfg.num_in_ch},H,W], got {tuple(x.shape)}")
        self._ensure(x.device)
        x = x.detach().float().contiguous()
        B, _, H, W = x.shape
        with torch.cuda.device(self.device):
            y = torch.empty((B, 1, H, W), dtype=torch.float32, device=self.device)
            need = C.c_size_t()
            L.check(self.lib.femasr_disc_workspace_bytes(self._h, B, H, W, C.byref(need)))
            ws = self._workspace(need.value)
            L.check(self.lib.femasr_disc_forward(self._h, x.data_ptr(), y.data_ptr(), B, H, W, ws.data_ptr(), ws.numel(),
                                                 _stream()))
        return y

    def flops(self, B: int, H: int, W: int) -> float:
        return float(self.lib.femasr_disc_flops(self._h, B, H, W))


class NativeLPIPS(_Engine):
    """LPIPS v0.1 (the lpips package, net 'alex' | 'vgg') on the engine: forward(x0, x1) -> (d [B], r [5, B])."""

    def __init__(self, net: str = "alex", gemm_path: int = 0):
        self.lib = L.load()
        self.net = net
        self.lcfg = L.LpipsConfig({"alex": 0, "vgg": 1}[net], int(gemm_path))
        self._h = C.c_void_p()
        self._ws: Optional[torch.Tensor] = None
        self.device: Optional[torch.device] = None
        self.names = [n for (n, _s, _k, _f) in lpips_spec(net)]

    def _create(self):
        L.check(self.lib.femasr_lpips_create(C.byref(self.lcfg), C.byref(self._h)))

    def forward(self, x0: torch.Tensor, x1: torch.Tensor, normalize: bool = False):
        """x0, x1 [B,3,H,W] -> (d [B], per-layer r [5,B]) fp32 on the device."""
        if x0.dim() != 4 or x0.shape[1] != 3 or x0.shape != x1.shape:
            raise L.FemasrError(f"expected two inputs [B,3,H,W] of one shape, got {tuple(x0.shape)} and {tuple(x1.shape)}")
        self._ensure(x0.device)
        if x1.device != x0.device:
            raise L.FemasrError(f"inputs on different devices: {x0.device} and {x1.device}")
        x0 = x0.detach().float().contiguous()
        x1 = x1.detach().float().contiguous()
        B, _, H, W = x0.shape
        with torch.cuda.device(self.device):
            d = torch.empty(B, dtype=torch.float32, device=self.device)
            r = torch.empty(5, B, dtype=torch.float32, device=self.device)
            need = C.c_size_t()
            L.check(self.lib.femasr_lpips_workspace_bytes(self._h, B, H, W, C.byref(need)))
            ws = self._workspace(need.value)
            L.check(self.lib.femasr_lpips_forward(self._h, x0.data_ptr(), x1.data_ptr(), d.data_ptr(), r.data_ptr(), B, H,
                                                  W, int(bool(normalize)), ws.data_ptr(), ws.numel(), _stream()))
        return d, r

    def flops(self, B: int, H: int, W: int) -> float:
        return float(self.lib.femasr_lpips_flops(self._h, B, H, W))
