"""Generate tests/golden/bsrgan/ (the degradation_bsrgan fixtures), offline, from the reference's unmodified
basicsr/data/bsrgan_util.py:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_bsrgan.py

The reference does not run on current SciPy as written; two shims, and nothing else, are applied to its module:
- `scipy.finfo = numpy.finfo` (fspecial_gaussian calls scipy.finfo, which SciPy no longer has);
- `interp2d` (removed from SciPy) is replaced by linear interpolation on the regular grid
  (scipy.interpolate.RegularGridInterpolator), which is what interp2d(kind='linear') evaluates at points of a regular
  grid.  This is the one piece that cannot be checked offline.
Wrappers around cv2.resize, ndimage.convolve, imresize_np, cv2.imencode, np.random.normal and
np.random.multivariate_normal record every operation with its parameters (kernel taps as float64).  Each case is one
.npz: `meta`, a JSON string with the records, the output shapes and a digest of random.getstate() and
np.random.get_state() after each call; `lq{i}`, the final LQ of call i.  Inputs are regenerated from seeds
(`case_input`), not stored.
"""
from __future__ import annotations

import hashlib
import importlib.util
import json
import os
import random
import sys
import types

import cv2
import numpy as np
import scipy
from scipy.interpolate import RegularGridInterpolator

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
OUT = os.path.join(HERE, "bsrgan")

# name, seed, H, W, sf, lq_patchsize, use_crop, calls
CASES = [
    ("sf4_256", 11, 256, 256, 4, 64, False, 1),
    ("sf2_256", 12, 256, 256, 2, 64, False, 1),
    ("sf4_290x322", 13, 290, 322, 4, 64, False, 1),
    ("sf4_crop", 14, 256, 256, 4, 32, True, 1),
    ("seq123_sf4_128", 123, 128, 128, 4, 32, False, 20),     # one stream, as generate_dataset runs
    ("seq7_sf4_64", 7, 64, 64, 4, 16, False, 60),            # more calls, so that every branch is taken twice
]


def case_input(seed, H, W, i=0):
    """The i-th input of a case: a smooth field plus texture, quantised to uint8 / 255 like a loaded PNG."""
    g = np.random.default_rng([seed, i])
    yy, xx = np.mgrid[0:H, 0:W] / max(H, W)
    base = np.stack([0.5 + 0.35 * np.sin(2 * np.pi * (g.random() * 3 * xx + g.random() * 2 * yy) + c) for c in range(3)], -1)
    img = np.clip(base + 0.08 * g.standard_normal((H, W, 3)), 0, 1)
    return (np.round(img * 255).astype(np.uint8).astype(np.float32) / 255.).astype(np.float32)


def rng_digest():
    h = hashlib.sha256(repr(random.getstate()).encode())
    name, keys, pos, has_gauss, cached = np.random.get_state()
    h.update(name.encode() + keys.tobytes() + repr((pos, has_gauss, cached)).encode())
    return h.hexdigest()


def proxy(mod, **over):
    """A stand-in for module `mod` inside the reference's module, with some attributes replaced."""
    ns = types.SimpleNamespace(**{k: getattr(mod, k) for k in dir(mod) if not k.startswith("__")})
    ns.__dict__.update(over)
    return ns


def load_reference(records):
    """The reference's bsrgan_util with the two shims and the recording wrappers; records go to `records`."""
    from scipy import ndimage

    from oracle.ref_shim import REFERENCE_ROOT
    spec = importlib.util.spec_from_file_location("ref_bsrgan_util",
                                                  os.path.join(REFERENCE_ROOT, "basicsr", "data", "bsrgan_util.py"))
    B = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(B)
    scipy.finfo = np.finfo

    def interp2d(x, y, z):
        f = RegularGridInterpolator((np.asarray(y), np.asarray(x)), np.asarray(z), method="linear")
        return lambda xn, yn: f(np.stack(np.meshgrid(yn, xn, indexing="ij"), -1))

    def logged(op, fn, params):
        def call(*a, **kw):
            out = fn(*a, **kw)
            records.append(dict(op=op, **params(out, *a, **kw)))
            return out
        return call

    def hw(x):
        return list(x.shape[:2])

    B.interp2d = interp2d
    B.cv2 = proxy(cv2, resize=logged("cv2.resize", cv2.resize, lambda o, x, dsize, interpolation: dict(
                      dsize=list(dsize), interpolation=int(interpolation), in_shape=hw(x), out_shape=hw(o))),
                  imencode=logged("imencode", cv2.imencode, lambda o, ext, x, p: dict(quality=int(p[1]), in_shape=hw(x))))
    B.ndimage = types.SimpleNamespace(filters=types.SimpleNamespace(convolve=logged(
        "convolve", ndimage.convolve, lambda o, x, k, mode: dict(weights=np.asarray(k[..., 0], np.float64).tolist(),
                                                                 in_shape=hw(x)))))
    B.imresize_np = logged("imresize_np", B.imresize_np, lambda o, x, scale, aa=True: dict(
        scale=float(scale), in_shape=hw(x), out_shape=hw(o)))
    B.np = proxy(np, random=proxy(
        np.random,
        normal=logged("normal", np.random.normal, lambda o, loc, scale, size: dict(scale=float(scale), size=list(size))),
        multivariate_normal=logged("multivariate_normal", np.random.multivariate_normal,
                                   lambda o, mean, cov, size: dict(cov=np.asarray(cov).tolist(), size=list(size)))))
    return B


def load_case(name):
    """(meta, [lq per call]) of a golden case."""
    z = np.load(os.path.join(OUT, name + ".npz"))
    meta = json.loads(str(z["meta"]))
    return meta, [z[f"lq{i}"] for i in range(len(meta["calls"]))]


def branch_counts(calls):
    """How often each branch was taken over lists of per-call records."""
    ops = {}
    for rec in calls:
        keys = ["jpeg_gated_" + ("on" if sum(r["op"] == "imencode" for r in rec) == 2 else "off")]
        first = rec[0]
        if first["op"] == "imresize_np" or (first["op"] == "cv2.resize" and
                                            first["out_shape"] == [first["in_shape"][0] // 2, first["in_shape"][1] // 2]):
            keys.append("downsample1/" + str(first.get("interpolation", "imresize_np")))
        for r in rec:
            key = r["op"] + (f"/{r['interpolation']}" if r["op"] == "cv2.resize" else "")
            if r["op"] == "normal":
                key += f"/{r['size'][-1]}"
            if r["op"] == "convolve":         # the shifted kernel is the only 25x25 one off centre
                k = np.asarray(r["weights"])
                centroid = (k.sum(1) * np.arange(k.shape[0])).sum() / k.sum()
                key += "/shifted" if k.shape[0] == 25 and abs(centroid - 12) > 0.25 else "/blur"
            keys.append(key)
        for k in keys:
            ops[k] = ops.get(k, 0) + 1
    return ops


BRANCHES = ("cv2.resize/1", "cv2.resize/2", "cv2.resize/3", "downsample1/1", "downsample1/2", "downsample1/3",
            "downsample1/imresize_np", "convolve/blur", "convolve/shifted", "normal/3", "normal/1",
            "multivariate_normal", "jpeg_gated_on", "jpeg_gated_off")


def main():
    os.makedirs(OUT, exist_ok=True)
    allrec = []
    for name, seed, H, W, sf, lqp, crop, calls in CASES:
        random.seed(seed)
        np.random.seed(seed)
        per_call, lqs = [], []
        for i in range(calls):
            rec = []
            lq, hq = load_reference(rec).degradation_bsrgan(case_input(seed, H, W, i), sf=sf, lq_patchsize=lqp,
                                                            use_crop=crop)
            per_call.append(dict(records=rec, lq_shape=list(lq.shape), hq_shape=list(hq.shape), rng=rng_digest()))
            lqs.append(np.asarray(lq, np.float32))
            allrec.append(rec)
        meta = dict(name=name, seed=seed, H=H, W=W, sf=sf, lq_patchsize=lqp, use_crop=crop, calls=per_call)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), meta=np.array(json.dumps(meta)),
                            **{f"lq{i}": a for i, a in enumerate(lqs)})
        print(name, [tuple(a.shape) for a in lqs[:3]])
    ops = branch_counts(allrec)
    print(ops)
    for k in BRANCHES:                   # every branch taken at least twice
        assert ops.get(k, 0) >= 2, f"branch {k} taken {ops.get(k, 0)} times"


if __name__ == "__main__":
    main()
