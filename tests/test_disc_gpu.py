"""GPU: UNetDiscriminatorSN on the engine, on both GEMM paths - the reference's goldens (tests/golden/disc/) through the
public surface, re-upload after an in-place change, the training-mode and geometry refusals, never-iterated u / v, and
the new kernels (4x4 stride-2 convs on both GEMMs, the LeakyReLU epilogue, bilinear x2 staging, spectral sigma, the
Cout = 1 head, the unnormalised im2col) against fp64 / ATen."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from femasr_b200 import lib as L
from femasr_b200.spec import random_disc_state_dict
from tests import disc_oracle as DO
from tests.gpu_util import S, igemm, nhwc, p, pack_weight, tc_igemm, tc_pack, tc_prepare
from tests.test_disc import DISC_GOLDEN, DISC_IDS, load_disc_case

pytestmark = pytest.mark.gpu
# output max-abs error / max|ref|: gemm_path 0 is fp32 SIMT, gemm_path 1 the K-sliced 3-product split-fp16 GEMM
OUT_RTOL = {0: 2e-5, 1: 2e-4}


def make_net(sd, cuda, gemm_path, skip=True):
    from basicsr.archs.discriminator_arch import UNetDiscriminatorSN
    net = UNetDiscriminatorSN(3, num_feat=64, skip_connection=skip, gemm_path=gemm_path)
    net.load_state_dict(sd, strict=True)
    return net.to(cuda).eval()


def rel(got, want):
    return ((got.double().cpu() - want.double()).abs().max() / want.double().abs().max()).item()


@pytest.mark.parametrize("gemm_path", [0, 1])
@pytest.mark.parametrize("path", DISC_GOLDEN, ids=DISC_IDS)
def test_disc_golden_through_public_surface(cuda, path, gemm_path):
    g, sd = load_disc_case(path)
    net = make_net(sd, cuda, gemm_path, bool(g["skip"]))
    x = torch.from_numpy(g["input"]).to(cuda)
    want = torch.from_numpy(g["out"])
    if int(g["power_iterations"]) == 0 and gemm_path == 1:
        with pytest.raises(L.FemasrError, match="never power-iterated"):
            net(x)
        return
    out = net(x)
    assert out.shape == want.shape and out.dtype == torch.float32 and not out.requires_grad
    err = rel(out, want)
    print(f"{path.split('/')[-1]} gemm_path {gemm_path}: output max-abs / max|ref| = {err:.3e}")
    assert err <= OUT_RTOL[gemm_path]


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_reupload_tracks_oracle(cuda, gemm_path):
    sd = random_disc_state_dict(80)
    net = make_net(sd, cuda, gemm_path)
    x = torch.rand(2, 3, 32, 48, generator=torch.Generator().manual_seed(81))
    y0 = net(x.to(cuda))
    assert rel(y0, DO.forward(sd, x)) <= OUT_RTOL[gemm_path]
    other = random_disc_state_dict(82)
    sd2 = dict(sd)
    sd2["conv3.weight_u"] = sd["conv3.weight_u"] * 1.5                # sigma x 1.5 (u stays aligned with W v)
    sd2["conv6.weight_v"] = sd["conv6.weight_v"] * 0.8                # sigma x 0.8
    sd2["conv0.weight"] = other["conv0.weight"]
    net.conv3.weight_u.copy_(sd2["conv3.weight_u"])                   # buffers: _version changes, the layer repacks
    net.conv6.weight_v.copy_(sd2["conv6.weight_v"])
    net.conv0.weight.copy_(sd2["conv0.weight"])
    y1 = net(x.to(cuda))
    want = DO.forward(sd2, x)
    assert rel(y1, want) <= OUT_RTOL[gemm_path]
    assert rel(y0, want) > 10 * OUT_RTOL[gemm_path]


def test_training_mode_and_geometry_raise(cuda):
    net = make_net(random_disc_state_dict(83), cuda, 1)
    net.train()
    with pytest.raises(L.FemasrError, match=r"\.eval\(\)"):
        net(torch.rand(1, 3, 16, 16, device=cuda))
    net.eval()
    with pytest.raises(L.FemasrError, match="multiples of 8"):
        net(torch.rand(1, 3, 16, 20, device=cuda))


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("H,W", [(8, 8), (24, 40), (64, 64)])
def test_conv4x4_stride2_both_gemms(cuda, H, W):
    g = torch.Generator().manual_seed(90 + H)
    B, Cin, Cout = 2, 128, 256
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 4, 4, generator=g) * 0.03
    want = F.conv2d(x.double(), w.double(), stride=2, padding=1).permute(0, 2, 3, 1)
    xd, wd = nhwc(x).to(cuda), w.to(cuda)
    y0 = igemm(xd, pack_weight(wd), None, B, H, W, Cin, Cout, ksize=4, stride=2)
    hi, lo = tc_prepare(xd)
    y1 = tc_igemm(hi, lo, tc_pack(wd), None, Cout, ksize=4, stride=2, slice_kb=4)
    y2 = tc_igemm(hi, lo, tc_pack(wd), None, Cout, ksize=4, stride=2)
    # y2: one pass through the tensor core's truncating accumulator (the engine slices, like y1)
    for y, bar in ((y0, 1e-5), (y1, 1e-5), (y2, OUT_RTOL[1])):
        assert y.shape == want.shape
        assert rel(y, want) <= bar


def test_lrelu_epilogue_both_gemms(cuda):
    g = torch.Generator().manual_seed(95)
    B, H, W, Cin, Cout = 2, 12, 20, 64, 128
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) * 0.05
    b = torch.randn(Cout, generator=g) * 0.5
    r = torch.randn(B, H, W, Cout, generator=g)
    want = F.leaky_relu(F.conv2d(x.double(), w.double(), b.double(), padding=1), 0.2).permute(0, 2, 3, 1) + r.double()
    xd, wd, bd, rd = nhwc(x).to(cuda), w.to(cuda), b.to(cuda), r.to(cuda)
    y0 = igemm(xd, pack_weight(wd), bd, B, H, W, Cin, Cout, act=L.ACT_LRELU, res1=rd)
    hi, lo = tc_prepare(xd)
    y1 = tc_igemm(hi, lo, tc_pack(wd), bd, Cout, act=L.ACT_LRELU, res1=rd)
    for y in (y0, y1):
        assert rel(y, want) <= 2e-5
    neg = (want - r.double()) < 0
    assert neg.double().mean() > 0.3                                   # the negative slope is exercised


@pytest.mark.parametrize("H,W", [(1, 1), (5, 9), (16, 16)])
def test_bilinear_staging_against_interpolate(cuda, H, W):
    g = torch.Generator().manual_seed(96)
    B, Cc = 2, 64
    x = torch.randn(B, H, W, Cc, generator=g) * 3
    want = F.interpolate(x.permute(0, 3, 1, 2).double(), scale_factor=2, mode="bilinear", align_corners=False)
    want = want.permute(0, 2, 3, 1)
    xd = x.to(cuda)
    lib = L.load()
    y = torch.empty(B, 2 * H, 2 * W, Cc, device=cuda)
    L.check(lib.femasr_bilinear_up2(p(xd), p(y), B, H, W, Cc, S()))
    hi = torch.empty(B, 2 * H, 2 * W, Cc, dtype=torch.float16, device=cuda)
    lo = torch.empty_like(hi)
    L.check(lib.femasr_tc_prepare(p(xd), p(hi), p(lo), L.PRO_BILINEAR2, None, None, None, None, B, H, W, Cc, 0, 0.0, S()))
    aten = F.interpolate(xd.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    assert rel(y, want) <= 1e-6
    assert (y - aten).abs().max().item() <= 1e-6 * aten.abs().max().item()
    assert torch.equal(hi, y.half())                                   # |y| < 65504: the staging is the split of y
    assert torch.equal(lo, (y - hi.float()).half())


def test_spectral_sigma_against_fp64(cuda):
    g = torch.Generator().manual_seed(97)
    lib = L.load()
    for co, k in ((128, 64 * 16), (64, 512 * 9), (512, 256 * 16)):
        w = torch.randn(co, k, generator=g) * 0.02
        u = F.normalize(torch.randn(co, generator=g), dim=0)
        v = F.normalize(torch.randn(k, generator=g), dim=0)
        out = torch.empty(2, device=cuda)
        wd, ud, vd = w.to(cuda), u.to(cuda), v.to(cuda)
        L.check(lib.femasr_spectral_sigma(p(wd), p(ud), p(vd), co, k, p(out), S()))
        wv = w.double().numpy() @ v.double().numpy()
        want = np.array([u.double().numpy() @ wv, np.linalg.norm(wv)])
        got = out.double().cpu().numpy()
        assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()
        out2 = torch.empty(2, device=cuda)
        L.check(lib.femasr_spectral_sigma(p(wd), p(ud), p(vd), co, k, p(out2), S()))
        assert torch.equal(out, out2)                                  # fixed order
        wn = torch.empty_like(wd)
        L.check(lib.femasr_spectral_normalize(p(wd), p(out), p(wn), wd.numel(), S()))
        assert torch.equal(wn, wd / out[0])                            # fp32 division, like weight_orig / sigma


@pytest.mark.parametrize("mma", [0, 1])
def test_head_cout1_and_cout3(cuda, mma):
    g = torch.Generator().manual_seed(98)
    B, H, W = 2, 19, 70
    x = torch.randn(B, 64, H, W, generator=g)
    lib = L.load()
    xd = nhwc(x).to(cuda)
    for co in (1, 3):
        w = torch.randn(co, 64, 3, 3, generator=g) * 0.05
        b = torch.randn(co, generator=g)
        want = F.conv2d(x.double(), w.double(), b.double(), padding=1)
        wp, bd = pack_weight(w.to(cuda)), b.to(cuda)
        y = torch.empty(B, co, H, W, device=cuda)
        L.check(lib.femasr_out_conv3x3_n(p(xd), p(wp), p(bd), p(y), B, H, W, 64, co, mma, S()))
        assert rel(y, want) <= 1e-5
        if co == 3:                                                    # the out_conv entry points are this kernel
            y3 = torch.empty_like(y)
            fn = lib.femasr_out_conv3x3_mma if mma else lib.femasr_out_conv3x3
            L.check(fn(p(xd), p(wp), p(bd), p(y3), B, H, W, 64, S()))
            assert torch.equal(y, y3)


def test_unnormalised_im2col(cuda):
    g = torch.Generator().manual_seed(99)
    B, H, W = 2, 9, 14
    x = torch.rand(B, 3, H, W, generator=g)
    cols = F.unfold(x, 3, padding=1).view(B, 3, 9, H * W)
    want = torch.zeros(B, H * W, 64)
    want[:, :, :27] = cols.permute(0, 3, 2, 1).reshape(B, H * W, 27)      # k = tap * 3 + ci
    want = want.view(B * H * W, 64)
    lib = L.load()
    xd = x.to(cuda)
    f32 = torch.empty(B * H * W, 64, device=cuda)
    L.check(lib.femasr_vgg_im2col(p(xd), None, None, None, None, p(f32), B, H, W, S()))
    assert torch.equal(f32.cpu(), want)
    assert lib.femasr_vgg_im2col(p(xd), p(xd), None, None, None, p(f32), B, H, W, S()) == -1   # mean without std
