"""GPU: the BSRGAN degradation kernels (femasr_b200/csrc/degrade.cu) against cv2 and the numpy oracles, step by step
and end to end on the goldens of tests/golden/bsrgan/, and inside guard bands."""
from __future__ import annotations

import random

import cv2
import numpy as np
import pytest
import torch

from femasr_b200 import degrade as D
from femasr_b200 import lib as L
from tests import degrade_oracle as O
from tests.test_degrade import (CASES, JPEG_SIZES, as_reference_records, assert_same_records, case_input, cv2_jpeg,
                                jpeg_content, load_case, rng_digest)

pytestmark = pytest.mark.gpu
RESIZE_ATOL, IMRESIZE_ATOL, FREE_RUN_PSNR = 1e-6, 2e-6, 40.0


@pytest.fixture(scope="module")
def be():
    """The backend degradation_bsrgan runs its steps on: one method per entry point."""
    dev = torch.device("cuda", 0)
    with torch.cuda.device(dev):
        yield D._Gpu(dev)


def gpu(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def ulps(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.astype(np.float32).view(np.int32).astype(np.int64))


def assert_conv_bar(got, want):
    u = ulps(got, want)
    assert u.max() <= 1 and (u == 0).mean() >= 0.9999, (u.max(), (u == 0).mean())


def imresize_oracle(x):
    h, w = x.shape[:2]
    return np.clip(O.apply_taps(O.apply_taps(x, D.matlab_resize_taps(h, 0.5), 0), D.matlab_resize_taps(w, 0.5), 1), 0, 1)


@pytest.mark.parametrize("h,w", JPEG_SIZES)
@pytest.mark.parametrize("kind", ["random", "smooth"])
def test_jpeg_bit_equal_to_cv2(be, h, w, kind):
    img = jpeg_content(h, w, kind)
    u8 = O.single2uint(img)
    for q in range(30, 96):
        got = be.jpeg(gpu(img), q).cpu().numpy()
        np.testing.assert_array_equal(got, (cv2_jpeg(u8, q) / 255.).astype(np.float32), err_msg=f"quality {q}")
        np.testing.assert_array_equal(got, O.jpeg_roundtrip(img, q), err_msg=f"quality {q}")


@pytest.mark.parametrize("stride", [1, 2, 4])
def test_mirror_convolution_against_fp64_oracle(be, stride):
    rng = np.random.default_rng(stride)
    for k in range(7, 26, 2):
        for (h, w) in [(67, 45), (8, 5)]:
            img = rng.random((h, w, 3)).astype(np.float32)
            K = rng.random((k, k))
            K /= K.sum()
            for clip in (False, True):
                want = O.mirror_convolve(img, K, stride)
                assert_conv_bar(be.conv(gpu(img), K, stride, clip).cpu().numpy(), np.clip(want, 0, 1) if clip else want)


@pytest.mark.parametrize("interp", [1, 2, 3])
def test_resize_against_cv2(be, interp):
    rng = np.random.default_rng(interp)
    worst = 0.0
    for (H, W) in [(256, 256), (101, 77)]:
        img = rng.random((H, W, 3)).astype(np.float32)
        for (oh, ow) in [(int(H / 2.7), int(W / 2.7)), (H // 4, W // 4), (H // 2, W // 2), (H, W),
                         (int(H * 1.7), int(W * 1.7)), (2 * H, 2 * W)]:
            ct, rt = D.cv2_resize_taps(H, W, oh, ow, interp)
            got = be.resize(gpu(img), (rt, ct), (oh, ow), (1, 0), True).cpu().numpy()
            worst = max(worst, float(np.abs(got - np.clip(cv2.resize(img, (ow, oh), interpolation=interp), 0, 1)).max()))
    print(f"resize interp {interp}: max abs vs cv2 {worst:.3g}")
    assert worst <= RESIZE_ATOL


def test_imresize_against_oracle(be):
    rng = np.random.default_rng(5)
    for (H, W) in [(256, 256), (128, 96), (290, 288)]:
        img = rng.random((H, W, 3)).astype(np.float32)
        taps = (D.matlab_resize_taps(H, 0.5), D.matlab_resize_taps(W, 0.5))
        got = be.resize(gpu(img), taps, (-(-H // 2), -(-W // 2)), (0, 1), True).cpu().numpy()
        assert np.abs(got - imresize_oracle(img)).max() <= IMRESIZE_ATOL


@pytest.mark.parametrize("ch", [1, 3])
def test_noise_add_bit_exact(be, ch):
    rng = np.random.default_rng(ch)
    img = rng.random((37, 53, 3)).astype(np.float32)
    f = rng.normal(0, 0.1, (37, 53, ch)).astype(np.float32)
    np.testing.assert_array_equal(be.noise(gpu(img), f).cpu().numpy(), np.clip(img + f, 0.0, 1.0))


def check_step(r):
    """One traced step against cv2 / the oracles on the step's own input."""
    x, y, p = r["input"].cpu().numpy(), r["output"].cpu().numpy(), r["params"]
    if r["op"] == "cv2.resize":
        want = np.clip(cv2.resize(x, tuple(p["dsize"]), interpolation=p["interpolation"]), 0, 1)
        assert np.abs(y - want).max() <= RESIZE_ATOL
    elif r["op"] == "imresize_np":
        assert np.abs(y - imresize_oracle(x)).max() <= IMRESIZE_ATOL
    elif r["op"] == "convolve":
        want = O.mirror_convolve(x, p["weights"], p["stride"])
        assert_conv_bar(y, np.clip(want, 0, 1) if p["stride"] > 1 else want)
    elif r["op"] == "noise":
        np.testing.assert_array_equal(y, np.clip(x + r["field"], 0.0, 1.0))
    elif r["op"] == "imencode":
        np.testing.assert_array_equal(y, O.jpeg_roundtrip(x, p["quality"]))


@pytest.mark.parametrize("case", [c[0] for c in CASES])
def test_step_by_step_and_free_running(be, case):
    g, lqs = load_case(case)
    random.seed(g["seed"])
    np.random.seed(g["seed"])
    worst_psnr, same = np.inf, []
    for i, call in enumerate(g["calls"]):
        trace = []
        lq, hq = D.degradation_bsrgan(case_input(g["seed"], g["H"], g["W"], i), g["sf"], g["lq_patchsize"],
                                      use_crop=g["use_crop"], trace=trace, trace_tensors=True)
        assert rng_digest() == call["rng"], f"call {i}"
        assert_same_records(as_reference_records(trace), call["records"], f"{case} call {i}")
        assert list(lq.shape) == call["lq_shape"] and list(hq.shape) == call["hq_shape"]
        for r in trace:
            check_step(r)
        mse = float(np.mean((lq.astype(np.float64) - lqs[i]) ** 2))
        worst_psnr = min(worst_psnr, 10 * np.log10(1.0 / max(mse, 1e-20)))
        same.append(float(((lq * 255).astype(np.uint8) == (lqs[i] * 255).astype(np.uint8)).mean()))
    print(f"{case}: min PSNR vs the reference's LQ {worst_psnr:.2f} dB, identical uint8 values "
          f"{np.mean(same) * 100:.2f} % (min {np.min(same) * 100:.2f} %)")
    assert worst_psnr >= FREE_RUN_PSNR


def test_tensor_in_tensor_out(be):
    random.seed(3)
    np.random.seed(3)
    lq, hq = D.degradation_bsrgan(gpu(case_input(3, 256, 256)), 4, 32, use_crop=True)
    assert lq.is_cuda and hq.is_cuda and tuple(lq.shape) == (32, 32, 3) and tuple(hq.shape) == (128, 128, 3)
    assert float(lq.min()) >= 0 and float(lq.max()) <= 1


def test_outputs_inside_guard_bands(be):
    """Every kernel writes its whole output and nothing of the NaN guards around it."""
    lib, G, H, W = L.load(), 4096, 45, 61
    rng = np.random.default_rng(9)
    x = gpu(rng.random((H, W, 3)))
    k = np.ascontiguousarray(rng.random((9, 9)))
    noise = gpu(rng.normal(0, 0.1, (H, W, 1)))
    ws = torch.empty(lib.femasr_degrade_jpeg_workspace_bytes(H, W), dtype=torch.uint8, device=x.device)
    ct, rt = (tuple(torch.from_numpy(t).cuda() for t in taps) for taps in D.cv2_resize_taps(H, W, 20, 70, 2))
    q = np.ascontiguousarray(D.jpeg_quant_tables(75), np.int32)
    s = torch.cuda.current_stream().cuda_stream
    calls = [(f"mirror_conv stride {st}", -(-H // st) * -(-W // st),
              lambda y, st=st: lib.femasr_degrade_mirror_conv(x.data_ptr(), y, H, W, k.ctypes.data, 9, 9, st, 1, s))
             for st in (1, 2, 4)]
    calls += [(f"resize_pass axis {a}", n, lambda y, a=a, t=t, o=o: lib.femasr_degrade_resize_pass(
        x.data_ptr(), y, H, W, a, o, t[0].data_ptr(), t[1].data_ptr(), t[0].shape[1], 1, s))
        for a, t, o, n in ((1, ct, 70, H * 70), (0, rt, 20, 20 * W))]
    calls += [("noise_add", H * W, lambda y: lib.femasr_degrade_noise_add(x.data_ptr(), noise.data_ptr(), 1, H, W, y, s)),
              ("jpeg", H * W, lambda y: lib.femasr_degrade_jpeg(x.data_ptr(), y, H, W, q.ctypes.data, ws.data_ptr(), s))]
    for what, pix, launch in calls:
        n = pix * 3
        buf = torch.full((n + 2 * G,), float("nan"), device=x.device)
        L.check(launch(buf[G:].data_ptr()))
        assert bool(torch.isnan(torch.cat([buf[:G], buf[G + n:]])).all()), f"{what}: a guard element was written"
        assert not bool(torch.isnan(buf[G:G + n]).any()), f"{what}: an output element was not written"


def test_refusals(be):
    lib = L.load()
    p = gpu(np.zeros((8, 8, 3))).data_ptr()
    k = np.ones((27, 27))
    assert lib.femasr_degrade_mirror_conv(p, p, 8, 8, k.ctypes.data, 27, 27, 1, 0, None) == -1
    assert lib.femasr_degrade_mirror_conv(p, p, 8, 8, k.ctypes.data, 3, 3, 5, 0, None) == -1
    assert lib.femasr_degrade_noise_add(p, p, 2, 8, 8, p, None) == -1
    q = np.ascontiguousarray(D.jpeg_quant_tables(75), np.int32)
    assert lib.femasr_degrade_jpeg(p, p, 0, 8, q.ctypes.data, p, None) == -1
    assert b"H and W" in lib.femasr_last_error()
    q[0, 5] = 0
    assert lib.femasr_degrade_jpeg(p, p, 8, 8, q.ctypes.data, p, None) == -1
    assert b"quantisation table" in lib.femasr_last_error()
