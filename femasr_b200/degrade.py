"""BSRGAN's degradation_bsrgan on the engine: synthesis of low-quality training inputs from HQ crops, as the
reference's generate_dataset.py and BSRGANTrainDataset run it (basicsr/data/bsrgan_util.py:581-669 of the reference).

`degradation_bsrgan(img, sf, lq_patchsize, isp_model, use_crop)` draws from the global `random` and `np.random`
streams exactly as the reference does (the same calls, in the same order, with the same arguments; the noise fields
too, on the host) and runs every image operation as an sm_90a kernel (femasr_b200/csrc/degrade.cu): the blurs as fp64
mirror convolutions, the cv2 and MATLAB resizes as separable passes over tap tables built here the way cv2 and
imresize_np build theirs, the noise add, and the JPEG round trip bit for bit as libjpeg-turbo computes it.  A numpy
image gives numpy (lq, hq); a CUDA tensor gives CUDA tensors.  `bsrgan_plan` makes the same draws without a GPU and
returns the operation records only.

Not bit-identical end to end: single2uint rounds before each JPEG round trip, so a last-ulp difference from a resize
can move a byte and, through the quantised DCT, an 8x8 block.  DESIGN.md section "BSRGAN degradation" gives the bars.
"""
from __future__ import annotations

import math
import random

import numpy as np

_STD_LUMA = [16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
             14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
             49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99]
_STD_CHROMA = [17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
               47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32


def jpeg_quant_tables(quality):
    """The luma and chroma quantisation tables (natural order) a baseline encoder uses at `quality` in [1, 100]: the
    JPEG standard's Annex K tables scaled by 5000/q below 50 and 200 - 2q above, rounded, limited to [1, 255]."""
    q = int(quality)
    if not 1 <= q <= 100:
        raise ValueError(f"JPEG quality must be in [1, 100], got {quality}")
    s = 5000 // q if q < 50 else 200 - 2 * q
    return tuple([min(max((v * s + 50) // 100, 1), 255) for v in t] for t in (_STD_LUMA, _STD_CHROMA))


def mirror_index(i, n):
    """ndimage's 'mirror' boundary (reflect about the edge samples, period 2n - 2) for any integer offsets."""
    i = np.asarray(i)
    if n == 1:
        return np.zeros_like(i)
    p = 2 * n - 2
    i = np.mod(i, p)
    return np.where(i >= n, p - i, i)


# ------------------------------------------------------------------------------------------------------- kernel taps
def fspecial_gaussian(hsize, sigma):
    """MATLAB's fspecial('gaussian', hsize, sigma): exp(-(x^2 + y^2) / (2 sigma^2)) on the centred grid, taps below
    eps * max set to zero, normalised to sum 1 (fp64)."""
    r = (hsize - 1.0) / 2.0
    x, y = np.meshgrid(np.arange(-r, r + 1), np.arange(-r, r + 1))
    h = np.exp(-(x * x + y * y) / (2 * sigma * sigma))
    h[h < np.finfo(float).eps * h.max()] = 0
    s = h.sum()
    return h / s if s != 0 else h


def _normal_pdf_2d(pts, cov):
    """The bivariate normal density (mean 0) at pts [..., 2], through the eigendecomposition of cov like SciPy's."""
    s, u = np.linalg.eigh(cov)
    w = u * (1.0 / np.sqrt(s))
    maha = np.sum(np.square(pts @ w), axis=-1)
    return np.exp(-0.5 * (2 * np.log(2 * np.pi) + np.sum(np.log(s)) + maha))


def anisotropic_gaussian(ksize, theta, l1, l2):
    """The ksize x ksize Gaussian with covariance V diag(l1, l2) V^-1, V built from the direction theta (gm_blur_kernel's
    grid: offsets y - size/2 - 0.5 + 1), normalised to sum 1."""
    v = np.array([[np.cos(theta), -np.sin(theta)], [np.sin(theta), np.cos(theta)]]) @ np.array([1.0, 0.0])
    V = np.array([[v[0], v[1]], [v[1], -v[0]]])
    cov = V @ np.diag([l1, l2]) @ np.linalg.inv(V)
    c = ksize / 2.0 + 0.5
    yy, xx = np.meshgrid(np.arange(ksize) - c + 1, np.arange(ksize) - c + 1, indexing="ij")
    k = _normal_pdf_2d(np.stack([xx, yy], -1), cov)
    return k / np.sum(k)


def shift_kernel(k, sf):
    """shift_pixel(k, sf): k resampled at (i + (sf-1)/2, j + (sf-1)/2), clamped to the last row / column, by linear
    interpolation on its grid (what interp2d(kind='linear') evaluates on a regular grid)."""
    n, m = k.shape
    shift = (sf - 1) * 0.5

    def axis(size):
        p = np.clip(np.arange(size, dtype=float) + shift, 0, size - 1)
        i0 = np.minimum(np.floor(p).astype(int), size - 2) if size > 1 else np.zeros(size, int)
        return i0, p - i0

    r0, fr = axis(n)
    c0, fc = axis(m)
    top = k[r0][:, c0] * (1 - fc) + k[r0][:, c0 + 1] * fc
    bot = k[r0 + 1][:, c0] * (1 - fc) + k[r0 + 1][:, c0 + 1] * fc
    return top * (1 - fr)[:, None] + bot * fr[:, None]


def orth(a):
    """scipy.linalg.orth: the left singular vectors of a whose singular values exceed max(M, N) * s_max * eps."""
    u, s, _ = np.linalg.svd(a, full_matrices=False)
    tol = max(a.shape) * s.max() * np.finfo(float).eps
    return u[:, :int(np.sum(s > tol))]


# ----------------------------------------------------------------------------------------------------- resize tables
_F = np.float32


def _pad_taps(rows):
    """[(indices, weights)] per output -> (idx [O, K] int32, w [O, K] fp32), short rows padded with zero weights."""
    K = max(len(i) for i, _ in rows)
    idx = np.zeros((len(rows), K), np.int32)
    w = np.zeros((len(rows), K), np.float32)
    for o, (i, v) in enumerate(rows):
        idx[o, :len(i)], w[o, :len(v)] = i, v
        idx[o, len(i):] = i[-1]
    return idx, w


def _linear_axis(n, on, scale, inv, area_mode):
    rows = []
    for d in range(on):
        if area_mode:
            sx = math.floor(d * scale)
            fx = _F((d + 1) - (sx + 1) * inv)
            fx = _F(0) if fx <= 0 else _F(fx - _F(math.floor(fx)))
        else:
            fx = (d + 0.5) * scale - 0.5
            sx = math.floor(fx)
            fx -= sx
        if sx < 0:
            fx, sx = 0.0, 0
        if sx >= n - 1:
            fx, sx = 0.0, n - 1
        rows.append(([sx, min(sx + 1, n - 1)], [_F(1 - fx), _F(fx)]))
    return _pad_taps(rows)


def _cubic_axis(n, on, scale):
    A = -0.75
    rows = []
    for d in range(on):
        x = (d + 0.5) * scale - 0.5
        sx = math.floor(x)
        x = float(_F(x - sx))                 # the fraction in fp32, the coefficients from it in fp64, then fp32
        c0 = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A
        c1 = ((A + 2) * x - (A + 3)) * x * x + 1
        c2 = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1
        rows.append(([min(max(sx - 1 + k, 0), n - 1) for k in range(4)], [_F(c) for c in (c0, c1, c2, 1 - c0 - c1 - c2)]))
    return _pad_taps(rows)


def _area_axis(n, on, scale):
    rows = []
    for d in range(on):
        f1 = d * scale
        f2 = f1 + scale
        cell = min(scale, n - f1)
        s1, s2 = math.ceil(f1), math.floor(f2)
        s2 = min(s2, n - 1)
        s1 = min(s1, s2)
        i, w = [], []
        if s1 - f1 > 1e-3:
            i.append(s1 - 1)
            w.append(_F((s1 - f1) / cell))
        for s in range(s1, s2):
            i.append(s)
            w.append(_F(1.0 / cell))
        if f2 - s2 > 1e-3:
            i.append(s2)
            w.append(_F(min(min(f2 - s2, 1.0), cell) / cell))
        rows.append((i, w))
    return _pad_taps(rows)


def cv2_resize_taps(H, W, oh, ow, interp):
    """cv2.resize of a float image [H, W] to [oh, ow] as two separable passes: ((col_idx, col_w), (row_idx, row_w)),
    columns first as cv2 computes it.  interp 1 INTER_LINEAR, 2 INTER_CUBIC, 3 INTER_AREA; coordinates and weights
    as cv2 computes them (fp32 weights).  A 2x linear downscale is the 2x2 box average, as in cv2."""
    if interp not in (1, 2, 3):
        raise ValueError(f"cv2 interpolation must be 1, 2 or 3, got {interp}")
    if min(H, W, oh, ow) < 1:
        raise ValueError(f"resize from {H}x{W} to {oh}x{ow}: sides must be >= 1")
    inv_x, inv_y = ow / W, oh / H
    sx, sy = 1.0 / inv_x, 1.0 / inv_y
    ix, iy = int(round(sx)), int(round(sy))
    area_fast = abs(sx - ix) < np.finfo(float).eps and abs(sy - iy) < np.finfo(float).eps
    if interp == 1 and area_fast and ix == 2 and iy == 2:
        interp = 3
    if interp == 3 and sx >= 1 and sy >= 1:
        return _area_axis(W, ow, sx), _area_axis(H, oh, sy)
    if interp == 2:
        return _cubic_axis(W, ow, sx), _cubic_axis(H, oh, sy)
    area = interp == 3
    return _linear_axis(W, ow, sx, inv_x, area), _linear_axis(H, oh, sy, inv_y, area)


def _matlab_cubic(x):
    ax = np.abs(x)
    ax2, ax3 = ax * ax, ax * ax * ax
    return ((_F(1.5) * ax3 - _F(2.5) * ax2 + _F(1)) * (ax <= 1) +
            (_F(-0.5) * ax3 + _F(2.5) * ax2 - _F(4) * ax + _F(2)) * ((ax > 1) & (ax <= 2))).astype(np.float32)


def matlab_resize_taps(n, scale):
    """imresize_np's weights and indices along one axis of length n (MATLAB's antialiased bicubic, computed in fp32
    like the reference's torch code), as (idx [ceil(n scale), K] into the unpadded axis, w): the symmetric padding
    becomes the reflection i -> -i - 1, i -> 2n - 1 - i."""
    on = math.ceil(n * scale)
    width = 4.0 / scale if scale < 1 else 4.0
    u = np.arange(1, on + 1, dtype=np.float32) / _F(scale) + _F(0.5 * (1 - 1 / scale))
    left = np.floor(u - _F(width / 2))
    P = math.ceil(width) + 2
    ind = left[:, None] + np.arange(P, dtype=np.float32)[None, :]
    dist = u[:, None] - ind
    w = _F(scale) * _matlab_cubic(dist * _F(scale)) if scale < 1 else _matlab_cubic(dist)
    w = (w / w.sum(1, keepdims=True)).astype(np.float32)
    if np.any(w[:, 0] == 0):
        ind, w = ind[:, 1:], w[:, 1:]
    if np.any(w[:, -1] == 0):
        ind, w = ind[:, :-1], w[:, :-1]
    i = ind.astype(np.int64) - 1
    i = np.where(i < 0, -i - 1, i)
    i = np.where(i >= n, 2 * n - 1 - i, i)
    return np.clip(i, 0, n - 1).astype(np.int32), np.ascontiguousarray(w)


# -------------------------------------------------------------------------------------------------------- backends
class _Dry:
    """Shapes only: the plan of a run without a GPU."""
    shape = staticmethod(lambda img: img)
    noise = jpeg = staticmethod(lambda img, *_: img)
    resize = staticmethod(lambda img, taps, out_hw, *_: out_hw)
    conv = staticmethod(lambda img, k, stride, clip: (-(-img[0] // stride), -(-img[1] // stride)))
    crop = staticmethod(lambda img, r, c, n: (n, n))


class _Gpu:
    """Every image operation as a degrade.cu kernel on `device`, on its current stream; each returns a new image.
    `timer` (optional) gets begin() / end(op, start) around each step."""

    def __init__(self, device, timer=None):
        import torch
        from . import lib as L
        self.torch, self.L, self.device, self.timer = torch, L, device, timer
        with torch.cuda.device(device):
            L.require_device()

    def _launch(self, fn, *args):
        self.L.check(getattr(self.L.load(), fn)(*args, self.torch.cuda.current_stream(self.device).cuda_stream))

    def _empty(self, h, w):
        return self.torch.empty((h, w, 3), dtype=self.torch.float32, device=self.device)

    def _dev(self, a):
        return self.torch.from_numpy(np.ascontiguousarray(a)).to(self.device)

    def shape(self, img):
        return tuple(img.shape[:2])

    def conv(self, img, k, stride, clip):
        H, W = img.shape[:2]
        y, k = self._empty(-(-H // stride), -(-W // stride)), np.ascontiguousarray(k, np.float64)
        self._launch("femasr_degrade_mirror_conv", img.data_ptr(), y.data_ptr(), H, W, k.ctypes.data, k.shape[0],
                     k.shape[1], stride, int(clip))
        return y

    def resize(self, img, taps, out_hw, order, clip):
        """Two passes, axis order[0] first (0 rows, 1 columns); taps[axis] = (idx, w); the clip on the second."""
        for n, axis in enumerate(order):
            H, W = img.shape[:2]
            idx, w = (self._dev(t) for t in taps[axis])
            y = self._empty(out_hw[0], W) if axis == 0 else self._empty(H, out_hw[1])
            self._launch("femasr_degrade_resize_pass", img.data_ptr(), y.data_ptr(), H, W, axis, out_hw[axis],
                         idx.data_ptr(), w.data_ptr(), idx.shape[1], int(clip and n == 1))
            img = y
        return img

    def noise(self, img, field):
        y, f = self._empty(*img.shape[:2]), self._dev(field.astype(np.float32))
        self._launch("femasr_degrade_noise_add", img.data_ptr(), f.data_ptr(), field.shape[2], *img.shape[:2],
                     y.data_ptr())
        return y

    def jpeg(self, img, quality):
        H, W = img.shape[:2]
        y = self._empty(H, W)
        ws = self.torch.empty(self.L.load().femasr_degrade_jpeg_workspace_bytes(H, W), dtype=self.torch.uint8,
                              device=self.device)
        q = np.ascontiguousarray(jpeg_quant_tables(quality), np.int32)
        self._launch("femasr_degrade_jpeg", img.data_ptr(), y.data_ptr(), H, W, q.ctypes.data, ws.data_ptr())
        return y

    def crop(self, img, r, c, n):
        return img[r:r + n, c:c + n].contiguous()


# ------------------------------------------------------------------------------------------------------- the model
_INTERP = (1, 2, 3)                  # cv2.INTER_LINEAR, INTER_CUBIC, INTER_AREA


def _run(img, sf, lq_patchsize, use_crop, be, trace, keep):
    """degradation_bsrgan's steps on backend `be`; img is the mod-cropped image (a shape for _Dry).  Returns
    (lq, (rnd_h, rnd_w) or None)."""

    def step(op, x, fn, field=None, **params):
        t0 = be.timer.begin() if getattr(be, "timer", None) else None
        y = fn()
        if t0 is not None:
            be.timer.end(op, t0)
        if trace is not None:
            r = dict(op=op, params=params, in_shape=tuple(be.shape(x)), out_shape=tuple(be.shape(y)))
            if keep:
                r["input"], r["output"] = x, y
                if field is not None:
                    r["field"] = field
            trace.append(r)
        return y

    def resize(x, size, interp, name="cv2.resize"):
        h, w = be.shape(x)
        taps = cv2_resize_taps(h, w, size[1], size[0], interp)
        return step(name, x, lambda: be.resize(x, (taps[1], taps[0]), (size[1], size[0]), (1, 0), True),
                    dsize=tuple(size), interpolation=interp)

    def add_blur(x, sf):
        wd2, wd = 4.0 + sf, 2.0 + 0.2 * sf
        if random.random() < 0.5:
            l1 = wd2 * random.random()
            l2 = wd2 * random.random()
            ks = 2 * random.randint(2, 11) + 3
            k = anisotropic_gaussian(ks, random.random() * np.pi, l1, l2)
        else:
            ks = 2 * random.randint(2, 11) + 3
            k = fspecial_gaussian(ks, wd * random.random())
        return step("convolve", x, lambda: be.conv(x, k, 1, False), weights=k, stride=1)

    def add_noise(x):
        level = random.randint(2, 25)
        rnum = np.random.rand()
        h, w = be.shape(x)
        if rnum > 0.6:
            f = np.random.normal(0, level / 255.0, (h, w, 3)).astype(np.float32)
            mode, extra = "color", dict(scale=level / 255.0)
        elif rnum < 0.4:
            f = np.random.normal(0, level / 255.0, (h, w, 1)).astype(np.float32)
            mode, extra = "gray", dict(scale=level / 255.0)
        else:
            L2 = (25 / 255.) ** 2
            Dg = np.diag(np.random.rand(3))
            U = orth(np.random.rand(3, 3))
            cov = np.abs(L2 * np.dot(np.dot(np.transpose(U), Dg), U))
            f = np.random.multivariate_normal([0, 0, 0], cov, (h, w)).astype(np.float32)
            mode, extra = "correlated", dict(cov=cov)
        return step("noise", x, lambda: be.noise(x, f), field=f, mode=mode, level=level, **extra)

    def add_jpeg(x):
        q = random.randint(30, 95)
        return step("imencode", x, lambda: be.jpeg(x, q), quality=q)

    if sf == 4 and random.random() < 0.25:                       # downsample1
        h, w = be.shape(img)
        if np.random.rand() < 0.5:
            img = resize(img, (int(1 / 2 * w), int(1 / 2 * h)), random.choice(_INTERP))
        else:
            taps = (matlab_resize_taps(h, 1 / 2), matlab_resize_taps(w, 1 / 2))
            out = (math.ceil(h / 2), math.ceil(w / 2))
            img = step("imresize_np", img, lambda: be.resize(img, taps, out, (0, 1), True), scale=0.5)
        sf = 2

    order = random.sample(range(7), 7)
    i2, i3 = order.index(2), order.index(3)
    if i2 > i3:
        order[i2], order[i3] = order[i3], order[i2]
    for i in order:
        if i in (0, 1):
            img = add_blur(img, sf)
        elif i == 2:
            h, w = be.shape(img)
            a, b = w, h
            if random.random() < 0.75:
                sf1 = random.uniform(1, 2 * sf)
                img = resize(img, (int(1 / sf1 * w), int(1 / sf1 * h)), random.choice(_INTERP))
            else:
                k = shift_kernel(fspecial_gaussian(25, random.uniform(0.1, 0.6 * sf)), sf)
                k = k / k.sum()
                x0 = img
                img = step("convolve", x0, lambda: be.conv(x0, k, sf, True), weights=k, stride=sf)
        elif i == 3:
            img = resize(img, (int(1 / sf * a), int(1 / sf * b)), random.choice(_INTERP))
        elif i == 4:
            img = add_noise(img)
        elif i == 5:
            if random.random() < 0.9:
                img = add_jpeg(img)
        elif i == 6:
            random.random()                                         # the ISP draw (isp_model is None)
    img = add_jpeg(img)
    if not use_crop:
        return img, None
    h, w = be.shape(img)
    rnd_h = random.randint(0, h - lq_patchsize)
    rnd_w = random.randint(0, w - lq_patchsize)
    img = step("crop", img, lambda: be.crop(img, rnd_h, rnd_w, lq_patchsize), rnd_h=rnd_h, rnd_w=rnd_w)
    return img, (rnd_h, rnd_w)


def _mod_crop_shape(h1, w1, sf, lq_patchsize):
    # rows limited by the width's multiple of sf and columns by the height's, as the reference writes it
    h, w = min(h1, w1 - w1 % sf), min(w1, h1 - h1 % sf)
    if h < lq_patchsize * sf or w < lq_patchsize * sf:
        raise ValueError(f"img size ({h1}X{w1}) is too small!")
    return h, w


def degradation_bsrgan(img, sf=4, lq_patchsize=72, isp_model=None, use_crop=True, *, trace=None,
                       trace_tensors=False, _timer=None):
    """The reference's degradation_bsrgan on the engine.  img: HWC fp32 RGB in [0, 1], a numpy array (returns numpy
    (lq, hq)) or a CUDA tensor on an sm_90 device (returns CUDA tensors).  Draws from `random` and `np.random` exactly
    as the reference does.  trace: a list that receives one record per operation (op, params, in_shape, out_shape,
    and with trace_tensors=True the operation's input and output)."""
    if isp_model is not None:
        raise NotImplementedError("degradation_bsrgan: no ISP model exists for the engine (the reference ships none)")
    import torch
    is_np = isinstance(img, np.ndarray)
    if is_np:
        if img.ndim != 3 or img.shape[2] != 3 or img.dtype != np.float32:
            raise ValueError(f"degradation_bsrgan: expected an HWC float32 RGB array, got {img.dtype} {img.shape}")
        dev = torch.device("cuda", torch.cuda.current_device())
    else:
        if img.dim() != 3 or img.shape[2] != 3 or img.dtype != torch.float32 or img.device.type != "cuda":
            raise ValueError("degradation_bsrgan: expected an HWC float32 RGB CUDA tensor (femasr_b200 has no CPU "
                             f"path), got {img.dtype} {tuple(img.shape)} on {img.device}")
        dev = img.device
    sf_ori = sf
    h1, w1 = img.shape[:2]
    h, w = _mod_crop_shape(h1, w1, sf, lq_patchsize)
    x = (torch.from_numpy(np.ascontiguousarray(img[:h, :w])).to(dev) if is_np else img[:h, :w].contiguous())
    hq = img[:h, :w].copy() if is_np else x.clone()
    with torch.cuda.device(dev):
        lq, rc = _run(x, sf, lq_patchsize, use_crop, _Gpu(dev, _timer), trace, trace_tensors)
    if rc is not None:
        r, c = rc[0] * sf_ori, rc[1] * sf_ori
        hq = hq[r:r + lq_patchsize * sf_ori, c:c + lq_patchsize * sf_ori]
    if is_np:
        return lq.cpu().numpy(), hq
    return lq, hq


def bsrgan_plan(h, w, sf=4, lq_patchsize=72, use_crop=True):
    """degradation_bsrgan's operation records for an h x w input, without a GPU: the same draws from `random` and
    `np.random` (noise fields included, then discarded), the same records as degradation_bsrgan(trace=...)."""
    records = []
    hh, ww = _mod_crop_shape(h, w, sf, lq_patchsize)
    _run((hh, ww), sf, lq_patchsize, use_crop, _Dry(), records, False)
    return records
