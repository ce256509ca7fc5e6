"""numpy oracles of the BSRGAN degradation steps (femasr_b200/csrc/degrade.cu computes the same on the GPU).

- `jpeg_roundtrip`: add_JPEG_noise's cv2.imencode('.jpg') / cv2.imdecode pair after single2uint, restated from the
  JPEG standard's baseline process as libjpeg-turbo's integer paths compute it (4:2:0, islow FDCT / IDCT, fancy
  upsampling).  Integer arithmetic throughout, so it equals cv2 byte for byte (tests/test_degrade.py).
- `mirror_convolve`: ndimage.convolve(img, k[..., None], mode='mirror') in fp64, optionally keeping [0::s, 0::s].
- `apply_taps`: a separable resize pass from the host tap tables of femasr_b200.degrade, in fp32 like the kernel.
"""
from __future__ import annotations

import numpy as np

from femasr_b200 import degrade as D

# ---------------------------------------------------------------------------------------------------------------- JPEG
_FIX = {k: int(v * 8192 + 0.5) for k, v in {
    "0_298631336": 0.298631336, "0_390180644": 0.390180644, "0_541196100": 0.541196100, "0_765366865": 0.765366865,
    "0_899976223": 0.899976223, "1_175875602": 1.175875602, "1_501321110": 1.501321110, "1_847759065": 1.847759065,
    "1_961570560": 1.961570560, "2_053119869": 2.053119869, "2_562915447": 2.562915447, "3_072711026": 3.072711026}.items()}


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, axis, pass2):
    """One islow FDCT pass (CONST_BITS 13, PASS1_BITS 2) along `axis` of an int64 array of 8-vectors."""
    v = [np.take(d, i, axis=axis) for i in range(8)]
    t0, t7 = v[0] + v[7], v[0] - v[7]
    t1, t6 = v[1] + v[6], v[1] - v[6]
    t2, t5 = v[2] + v[5], v[2] - v[5]
    t3, t4 = v[3] + v[4], v[3] - v[4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    out = [None] * 8
    sh = 13 + 2 if pass2 else 13 - 2
    if pass2:
        out[0], out[4] = _descale(t10 + t11, 2), _descale(t10 - t11, 2)
    else:
        out[0], out[4] = (t10 + t11) << 2, (t10 - t11) << 2
    z1 = (t12 + t13) * _FIX["0_541196100"]
    out[2] = _descale(z1 + t13 * _FIX["0_765366865"], sh)
    out[6] = _descale(z1 - t12 * _FIX["1_847759065"], sh)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * _FIX["1_175875602"]
    t4, t5, t6, t7 = (t4 * _FIX["0_298631336"], t5 * _FIX["2_053119869"], t6 * _FIX["3_072711026"],
                      t7 * _FIX["1_501321110"])
    z1, z2 = -z1 * _FIX["0_899976223"], -z2 * _FIX["2_562915447"]
    z3, z4 = -z3 * _FIX["1_961570560"] + z5, -z4 * _FIX["0_390180644"] + z5
    out[7] = _descale(t4 + z1 + z3, sh)
    out[5] = _descale(t5 + z2 + z4, sh)
    out[3] = _descale(t6 + z2 + z3, sh)
    out[1] = _descale(t7 + z1 + z4, sh)
    return np.stack(out, axis=axis)


def _idct_1d(d, axis, pass2):
    """One islow IDCT pass along `axis` (pass 1 descales by 11 bits, pass 2 by 18)."""
    v = [np.take(d, i, axis=axis) for i in range(8)]
    z1 = (v[2] + v[6]) * _FIX["0_541196100"]
    t2 = z1 - v[6] * _FIX["1_847759065"]
    t3 = z1 + v[2] * _FIX["0_765366865"]
    t0, t1 = (v[0] + v[4]) << 13, (v[0] - v[4]) << 13
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    t0, t1, t2, t3 = v[7], v[5], v[3], v[1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * _FIX["1_175875602"]
    t0, t1, t2, t3 = (t0 * _FIX["0_298631336"], t1 * _FIX["2_053119869"], t2 * _FIX["3_072711026"],
                      t3 * _FIX["1_501321110"])
    z1, z2 = -z1 * _FIX["0_899976223"], -z2 * _FIX["2_562915447"]
    z3, z4 = -z3 * _FIX["1_961570560"] + z5, -z4 * _FIX["0_390180644"] + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    sh = 13 + 2 + 3 if pass2 else 13 - 2
    out = [t10 + t3, t11 + t2, t12 + t1, t13 + t0, t13 - t0, t12 - t1, t11 - t2, t10 - t3]
    return np.stack([_descale(o, sh) for o in out], axis=axis)


def _blocks(plane):
    """[H8, W8] -> [H8/8, W8/8, 8, 8]"""
    h, w = plane.shape
    return plane.reshape(h // 8, 8, w // 8, 8).transpose(0, 2, 1, 3)


def _unblocks(b):
    n, m = b.shape[:2]
    return b.transpose(0, 2, 1, 3).reshape(n * 8, m * 8)


def jpeg_reciprocals(qtab):
    """libjpeg-turbo's quantisation by reciprocal for the islow FDCT (whose output carries a factor 8): per entry
    (recip, corr, shift) with |c| / (8 q) rounded = ((|c| + corr) * recip) >> shift."""
    recip, corr, shift = [], [], []
    for q in qtab:
        d = q << 3
        r = 16 + d.bit_length() - 1
        fq, fr = divmod(1 << r, d)
        c = d // 2
        if fr == 0:
            fq, r = fq >> 1, r - 1
        elif fr <= d // 2:
            c += 1
        else:
            fq += 1
        recip.append(fq)
        corr.append(c)
        shift.append(r)
    return recip, corr, shift


def _code(plane, qtab):
    """Level shift, FDCT, quantise (libjpeg-turbo's reciprocal form), dequantise, IDCT, range limit: [H8, W8] uint8."""
    b = _blocks(plane.astype(np.int64) - 128)
    c = _fdct_1d(_fdct_1d(b, 3, False), 2, True)
    recip, corr, shift = (np.array(t, np.int64).reshape(8, 8) for t in jpeg_reciprocals(qtab))
    mag = ((np.abs(c) + corr) * recip) >> shift
    q = np.where(c < 0, -mag, mag)
    r = _idct_1d(_idct_1d(q * np.asarray(qtab, np.int64).reshape(8, 8), 2, False), 3, True)
    return _unblocks(np.clip(r + 128, 0, 255))


def _fancy_up2(c, H, W):
    """h2v2 upsampling of a [ceil(H/2), ceil(W/2)] chroma plane to [H, W]: libjpeg-turbo's triangle filter (3/4, 1/4;
    rows first, then columns with biases 8 and 7), replicated edges; plain 2x2 replication when ceil(W/2) <= 2."""
    ch, cw = c.shape
    c = c.astype(np.int64)
    if cw <= 2:
        return np.repeat(np.repeat(c, 2, 0), 2, 1)[:H, :W]
    up = np.concatenate([c[:1], c[:-1]], 0)
    dn = np.concatenate([c[1:], c[-1:]], 0)
    rows = np.empty((2 * ch, cw), np.int64)
    rows[0::2], rows[1::2] = 3 * c + up, 3 * c + dn
    left = np.concatenate([rows[:, :1], rows[:, :-1]], 1)
    right = np.concatenate([rows[:, 1:], rows[:, -1:]], 1)
    out = np.empty((2 * ch, 2 * cw), np.int64)
    out[:, 0::2] = (3 * rows + left + 8) >> 4
    out[:, 1::2] = (3 * rows + right + 7) >> 4
    return out[:H, :W]


def jpeg_roundtrip_u8(rgb, quality):
    """uint8 RGB [H, W, 3] -> the RGB cv2.imdecode(cv2.imencode('.jpg', BGR, quality)) returns, as uint8."""
    H, W = rgb.shape[:2]
    yt, ct = D.jpeg_quant_tables(quality)
    p = rgb.astype(np.int64)
    R, G, B = p[..., 0], p[..., 1], p[..., 2]
    F = lambda v: int(v * 65536 + 0.5)  # noqa: E731
    half, off = 1 << 15, 128 << 16
    Y = (F(0.299) * R + F(0.587) * G + F(0.114) * B + half) >> 16
    Cb = (-F(0.16874) * R - F(0.33126) * G + F(0.5) * B + off + half - 1) >> 16
    Cr = (F(0.5) * R - F(0.41869) * G - F(0.08131) * B + off + half - 1) >> 16
    # luma: replicate the last row / column out to whole 8x8 blocks
    H8, W8 = -(-H // 8) * 8, -(-W // 8) * 8
    Yp = np.pad(Y, ((0, H8 - H), (0, W8 - W)), mode="edge")
    # chroma: replicate columns out to whole 16-pixel MCUs and one row to an even height, 2x2 average with biases
    # 1, 2, 1, 2, ... along the row, then replicate downsampled rows out to whole blocks
    W16, He = -(-W // 16) * 16, H + (H & 1)
    ch = He // 2
    C8 = -(-ch // 8) * 8
    bias = np.tile(np.array([1, 2], np.int64), W16 // 4)
    dec = []
    for P in (Cb, Cr):
        P = np.pad(P, ((0, He - H), (0, W16 - W)), mode="edge")
        s = (P[0::2, 0::2] + P[0::2, 1::2] + P[1::2, 0::2] + P[1::2, 1::2] + bias) >> 2
        s = np.pad(s, ((0, C8 - ch), (0, 0)), mode="edge")
        dec.append(_fancy_up2(_code(s, ct)[:ch, :-(-W // 2)], H, W))
    y = _code(Yp, yt)[:H, :W]
    cb, cr = dec[0] - 128, dec[1] - 128
    r = y + ((F(1.402) * cr + half) >> 16)
    g = y + ((-F(0.34414) * cb + half - F(0.71414) * cr) >> 16)
    b = y + ((F(1.772) * cb + half) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def single2uint(img):
    return np.uint8((img.clip(0, 1) * 255.).round())


def jpeg_roundtrip(img, quality):
    """add_JPEG_noise given its quality: float32 RGB in -> float32 RGB out (single2uint, JPEG, uint2single)."""
    return (jpeg_roundtrip_u8(single2uint(img), quality) / 255.).astype(np.float32)


# ---------------------------------------------------------------------------------------------- convolution, resize
def mirror_convolve(img, k, stride=1):
    """ndimage.convolve(img, k[..., None], mode='mirror')[::stride, ::stride] in fp64 (rounded to fp32 once)."""
    k = np.asarray(k, np.float64)
    kh, kw = k.shape
    H, W = img.shape[:2]
    rows = D.mirror_index(np.arange(-(kh // 2), H + kh // 2), H)
    cols = D.mirror_index(np.arange(-(kw // 2), W + kw // 2), W)
    p = img.astype(np.float64)[rows][:, cols]
    kf = k[::-1, ::-1]
    out = np.zeros((H, W, img.shape[2]))
    for i in range(kh):
        for j in range(kw):
            out += kf[i, j] * p[i:i + H, j:j + W]
    return out[::stride, ::stride].astype(np.float32)


def apply_taps(img, taps, axis):
    """One separable pass: out[o] = sum_k w[o, k] * img[idx[o, k]] along `axis` (0 rows, 1 columns), accumulated in
    fp32 in tap order."""
    idx, w = taps
    x = np.moveaxis(img.astype(np.float32), axis, 0)
    out = x[idx[:, 0]] * w[:, 0].reshape(-1, *[1] * (x.ndim - 1))
    for k in range(1, idx.shape[1]):
        out = out + x[idx[:, k]] * w[:, k].reshape(-1, *[1] * (x.ndim - 1))
    return np.moveaxis(out.astype(np.float32), 0, axis)
