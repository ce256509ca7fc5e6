"""CPU: the BSRGAN degradation's host side (femasr_b200/degrade.py) and its numpy oracles (tests/degrade_oracle.py).

- bsrgan_plan makes the reference's draws: the same operations with the same parameters, taps within 1e-15 relative,
  the same shapes and the same RNG states after every call, on every case of tests/golden/bsrgan/;
- the numpy JPEG round trip equals cv2.imencode / imdecode byte for byte at every quality add_JPEG_noise draws;
- the mirror convolution, the cv2 resize tables and the kernel-tap restatements hold to ndimage, cv2 and SciPy.
"""
from __future__ import annotations

import os
import random
import sys

import cv2
import numpy as np
import pytest

from femasr_b200 import degrade as D
from tests import degrade_oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_golden_bsrgan import CASES, case_input, load_case, rng_digest  # noqa: E402

JPEG_SIZES = [(1, 1), (7, 9), (15, 17), (16, 16), (33, 65), (128, 128), (290, 322), (2, 2), (3, 4), (9, 4)]


def jpeg_content(h, w, kind, seed=0):
    if kind == "random":
        return np.random.default_rng([seed, h, w]).random((h, w, 3)).astype(np.float32)
    yy, xx = np.mgrid[0:h, 0:w]
    return np.stack([0.5 + 0.4 * np.sin(xx / 7.0 + c) * np.cos(yy / 5.0 - c) for c in range(3)], -1).astype(np.float32)


def cv2_jpeg(u8, q):
    ok, enc = cv2.imencode(".jpg", np.ascontiguousarray(u8[:, :, ::-1]), [cv2.IMWRITE_JPEG_QUALITY, q])
    assert ok
    return cv2.imdecode(enc, 1)[:, :, ::-1]


def as_reference_records(plan):
    """degrade.py's records in the vocabulary of the golden's wrappers (no record for the final crop)."""
    out = []
    for r in plan:
        p, op = r["params"], r["op"]
        if op == "cv2.resize":
            out.append(dict(op=op, dsize=list(p["dsize"]), interpolation=p["interpolation"],
                            in_shape=list(r["in_shape"]), out_shape=list(r["out_shape"])))
        elif op == "imresize_np":
            out.append(dict(op=op, scale=p["scale"], in_shape=list(r["in_shape"]), out_shape=list(r["out_shape"])))
        elif op == "convolve":
            out.append(dict(op=op, weights=p["weights"], in_shape=list(r["in_shape"])))
        elif op == "noise":
            h, w = r["in_shape"]
            if p["mode"] == "correlated":
                out.append(dict(op="multivariate_normal", cov=p["cov"], size=[h, w]))
            else:
                out.append(dict(op="normal", scale=p["scale"], size=[h, w, 3 if p["mode"] == "color" else 1]))
        elif op == "imencode":
            out.append(dict(op=op, quality=p["quality"], in_shape=list(r["in_shape"])))
    return out


def assert_same_records(mine, ref, where):
    assert [r["op"] for r in mine] == [r["op"] for r in ref], where
    for k, (a, b) in enumerate(zip(mine, ref)):
        for key, want in b.items():
            if key in ("weights", "cov"):
                got, want = np.asarray(a[key], np.float64), np.asarray(want, np.float64)
                assert got.shape == want.shape, (where, k, key)
                rel = np.abs(got - want).max() / np.abs(want).max()
                assert rel <= 1e-15, (where, k, key, rel)
            elif key != "mode":
                assert a[key] == want, (where, k, key, a[key], want)


@pytest.mark.parametrize("case", [c[0] for c in CASES])
def test_plan_matches_reference_draws(case):
    g = load_case(case)[0]
    random.seed(g["seed"])
    np.random.seed(g["seed"])
    for i, call in enumerate(g["calls"]):
        plan = D.bsrgan_plan(g["H"], g["W"], g["sf"], g["lq_patchsize"], g["use_crop"])
        assert_same_records(as_reference_records(plan), call["records"], f"{case} call {i}")
        assert list(plan[-1]["out_shape"]) == call["lq_shape"][:2]
        assert rng_digest() == call["rng"], f"{case} call {i}: RNG state differs after the call"


def test_case_inputs_are_regenerated_from_seeds():
    a = case_input(11, 256, 256)
    assert a.dtype == np.float32 and a.shape == (256, 256, 3)
    np.testing.assert_array_equal(a, case_input(11, 256, 256))


@pytest.mark.parametrize("h,w", JPEG_SIZES)
@pytest.mark.parametrize("kind", ["random", "smooth"])
def test_jpeg_oracle_equals_cv2(h, w, kind):
    img = jpeg_content(h, w, kind)
    u8 = O.single2uint(img)
    for q in range(30, 96):
        np.testing.assert_array_equal(O.jpeg_roundtrip_u8(u8, q), cv2_jpeg(u8, q), err_msg=f"quality {q}")


def test_jpeg_round_trip_is_add_jpeg_noise():
    img = jpeg_content(33, 65, "random")
    want = (cv2_jpeg(O.single2uint(img), 57) / 255.).astype(np.float32)
    np.testing.assert_array_equal(O.jpeg_roundtrip(img, 57), want)


@pytest.mark.parametrize("h,w,k", [(5, 7, 25), (2, 3, 9), (40, 33, 7), (64, 64, 25), (1, 9, 5)])
def test_mirror_convolution_oracle_equals_ndimage(h, w, k):
    from scipy import ndimage
    rng = np.random.default_rng(k)
    img = rng.random((h, w, 3)).astype(np.float32)
    K = rng.random((k, k))
    np.testing.assert_array_equal(O.mirror_convolve(img, K), ndimage.convolve(img, K[..., None], mode="mirror"))
    np.testing.assert_array_equal(O.mirror_convolve(img, K, 2), ndimage.convolve(img, K[..., None], mode="mirror")[::2, ::2])


@pytest.mark.parametrize("interp", [1, 2, 3])
@pytest.mark.parametrize("H,W", [(256, 256), (100, 77), (13, 9)])
def test_resize_tables_hold_to_cv2(interp, H, W):
    img = np.random.default_rng(H * W).random((H, W, 3)).astype(np.float32)
    for oh, ow in [(H // 2, W // 2), (H // 4, W // 4), (int(H / 2.7), int(W / 2.7)), (H, W), (int(H * 1.7), int(W * 1.7)),
                   (2 * H, 2 * W), (max(1, H // 3), W)]:
        want = np.clip(cv2.resize(img, (ow, oh), interpolation=interp), 0, 1)
        ct, rt = D.cv2_resize_taps(H, W, oh, ow, interp)
        got = np.clip(O.apply_taps(O.apply_taps(img, ct, 1), rt, 0), 0, 1)
        assert np.abs(got - want).max() <= 1e-6, (oh, ow)


def test_matlab_resize_tables():
    idx, w = D.matlab_resize_taps(256, 0.5)
    assert idx.shape[0] == 128 and idx.min() >= 0 and idx.max() < 256
    np.testing.assert_allclose(w.sum(1), 1, atol=1e-6)
    # a constant image stays constant; a ramp stays a ramp in the interior
    ramp = np.tile(np.arange(256, dtype=np.float32)[:, None, None], (1, 4, 3))
    out = O.apply_taps(ramp, (idx, w), 0)
    np.testing.assert_allclose(out[4:-4, 0, 0], 2 * np.arange(4, 124) + 0.5, atol=1e-3)


def test_kernel_taps_hold_to_scipy():
    scipy_stats = pytest.importorskip("scipy.stats")
    from scipy.linalg import orth
    rng = np.random.default_rng(0)
    for _ in range(200):
        a = rng.random((3, 3))
        np.testing.assert_array_equal(D.orth(a), orth(a))
    for _ in range(20):
        th, l1, l2, ks = rng.random() * np.pi, 8 * rng.random() + 0.1, 8 * rng.random() + 0.1, 2 * rng.integers(2, 12) + 3
        v = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]) @ np.array([1.0, 0.0])
        V = np.array([[v[0], v[1]], [v[1], -v[0]]])
        cov = V @ np.diag([l1, l2]) @ np.linalg.inv(V)
        c = ks / 2.0 + 0.5
        want = np.array([[scipy_stats.multivariate_normal.pdf([x - c + 1, y - c + 1], mean=[0, 0], cov=cov)
                          for x in range(ks)] for y in range(ks)])
        want /= want.sum()
        got = D.anisotropic_gaussian(ks, th, l1, l2)
        assert np.abs(got - want).max() / want.max() <= 1e-14


def test_refusals():
    with pytest.raises(ValueError, match="too small"):
        D.bsrgan_plan(100, 100, 4, 72)
    with pytest.raises(NotImplementedError):
        D.degradation_bsrgan(np.zeros((288, 288, 3), np.float32), isp_model=object())
    with pytest.raises(ValueError):
        D.cv2_resize_taps(4, 4, 2, 2, 0)


def test_generate_dataset_script(tmp_path, monkeypatch):
    """Walk order, the HQ_sub/HR -> LR path rewrite, the truncating save and the RNG stream of
    scripts/generate_dataset.py, with the device step replaced by its plan (the shapes and the draws)."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
    import generate_dataset as G
    hq = tmp_path / "HQ_sub"
    for sub, n in (("b_HR", 2), ("a_HR", 1)):
        (hq / sub).mkdir(parents=True)
        for i in range(n):
            cv2.imwrite(str(hq / sub / f"img{i}.png"), np.full((300, 290, 3), 40 * i, np.uint8))
    (hq / "a_HR" / "notes.txt").write_text("not an image")

    def planned(img, sf, use_crop):
        shape = D.bsrgan_plan(img.shape[0], img.shape[1], sf, 72, use_crop)[-1]["out_shape"]
        return np.full(tuple(shape) + (3,), 0.999, np.float32), img

    monkeypatch.setattr(G, "degradation_bsrgan", planned)
    G.main(["--hq", str(hq), "--out", str(tmp_path / "LQ_sub_X4"), "--scale", "4"])
    after = rng_digest()
    files = sorted(p.relative_to(tmp_path / "LQ_sub_X4").as_posix() for p in (tmp_path / "LQ_sub_X4").rglob("*.png"))
    assert files == ["a_LR/img0.png", "b_LR/img0.png", "b_LR/img1.png"]
    for f in files:
        out = cv2.imread(str(tmp_path / "LQ_sub_X4" / f))
        assert out.shape[2] == 3 and int(out.max()) == 254          # 0.999 * 255 truncates to 254
    assert G.walk_images(str(hq))[0].endswith(os.path.join("a_HR", "img0.png"))
    random.seed(123)
    np.random.seed(123)
    for _ in range(3):
        D.bsrgan_plan(300, 290, 4, 72, False)
    assert rng_digest() == after
