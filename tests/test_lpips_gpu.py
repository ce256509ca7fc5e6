"""GPU: LPIPS v0.1 on the engine, both nets on both GEMM paths - the goldens (tests/golden/lpips/) through
femasr_b200.lpips.LPIPS, exact zero and exact symmetry, retPerLayer, re-upload after an in-place change, the geometry
refusals, the new kernels (5x5 conv on both GEMMs, the 3x3/2 pool staging, the K = 363 im2col, the head) against ATen /
fp64, and scripts/validate_lpips.py on generated PNG pairs."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from femasr_b200 import lib as L
from femasr_b200.spec import random_lpips_state_dict
from tests import lpips_oracle as LO
from tests.gpu_util import S, igemm, nhwc, p, pack_weight, tc_igemm, tc_pack, tc_prepare
from tests.test_lpips import LPIPS_GOLDEN, LPIPS_IDS, load_lpips_case

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# absolute error of d per image: gemm_path 0 is fp32 SIMT, gemm_path 1 the split-fp16 tensor-core GEMM (half a unit of
# the 4th decimal LPIPS is reported to)
D_ATOL = {0: 2e-6, 1: 5e-5}


def make(net, sd, cuda, gemm_path):
    from femasr_b200.lpips import LPIPS
    with pytest.warns(UserWarning):
        m = LPIPS(net, gemm_path=gemm_path)
    m.load_state_dict(sd, strict=True)
    return m.to(cuda)


@pytest.mark.parametrize("gemm_path", [0, 1])
@pytest.mark.parametrize("path", LPIPS_GOLDEN, ids=LPIPS_IDS)
def test_lpips_golden_through_public_surface(cuda, path, gemm_path):
    g, net, sd, in0, in1, normalize = load_lpips_case(path)
    m = make(net, sd, cuda, gemm_path)
    d, res = m(in0.to(cuda), in1.to(cuda), retPerLayer=True, normalize=normalize)
    B = in0.shape[0]
    assert d.shape == (B, 1, 1, 1) and d.dtype == torch.float32 and not d.requires_grad
    assert len(res) == 5 and all(r.shape == (B, 1, 1, 1) for r in res)
    err = np.abs(d.view(-1).cpu().numpy() - g["d"]).max()
    rerr = np.abs(torch.stack([r.view(-1) for r in res]).cpu().numpy() - g["r"]).max()
    print(f"{os.path.basename(path)} gemm_path {gemm_path}: |d - golden| max {err:.3e}, |r_k - golden| max {rerr:.3e}")
    assert err <= D_ATOL[gemm_path]
    # retPerLayer: d is the left-to-right float sum of the five r_k
    acc = res[0].clone()
    for r in res[1:]:
        acc = acc + r
    assert torch.equal(acc, d)
    assert torch.equal(m(in0.to(cuda), in1.to(cuda), normalize=normalize), d)


@pytest.mark.parametrize("gemm_path", [0, 1])
@pytest.mark.parametrize("net,H,W", [("alex", 67, 93), ("vgg", 32, 48)])
def test_zero_and_symmetry_exact(cuda, net, H, W, gemm_path):
    m = make(net, random_lpips_state_dict(net, 30), cuda, gemm_path)
    gen = torch.Generator().manual_seed(31)
    x0 = torch.rand(3, 3, H, W, generator=gen).to(cuda)
    x1 = torch.rand(3, 3, H, W, generator=gen).to(cuda)
    assert torch.equal(m(x0, x0.clone(), normalize=True), torch.zeros(3, 1, 1, 1, device=cuda))
    d01, r01 = m(x0, x1, retPerLayer=True, normalize=True)
    d10, r10 = m(x1, x0, retPerLayer=True, normalize=True)
    assert torch.equal(d01, d10)
    assert all(torch.equal(a, b) for a, b in zip(r01, r10))
    # a pair's distance does not depend on the other pairs of the batch
    assert torch.equal(m(x0[1:2], x1[1:2], normalize=True), d01[1:2])


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_reupload_tracks_oracle(cuda, gemm_path):
    sd = random_lpips_state_dict("alex", 40)
    m = make("alex", sd, cuda, gemm_path)
    gen = torch.Generator().manual_seed(41)
    x0, x1 = torch.rand(2, 3, 48, 64, generator=gen), torch.rand(2, 3, 48, 64, generator=gen)
    d0 = m(x0.to(cuda), x1.to(cuda), normalize=True).view(-1).cpu()
    assert (d0 - LO.forward("alex", sd, x0, x1, normalize=True).view(-1)).abs().max() <= D_ATOL[gemm_path]
    sd2 = dict(sd)
    sd2["lin2.model.1.weight"] = sd["lin2.model.1.weight"] * 3.0
    sd2["net.slice2.3.weight"] = random_lpips_state_dict("alex", 42)["net.slice2.3.weight"]
    getattr(m.lin2.model, "1").weight.copy_(sd2["lin2.model.1.weight"])      # in place: _version changes, re-upload
    getattr(m.net.slice2, "3").weight.copy_(sd2["net.slice2.3.weight"])
    d1 = m(x0.to(cuda), x1.to(cuda), normalize=True).view(-1).cpu()
    want = LO.forward("alex", sd2, x0, x1, normalize=True).view(-1)
    assert (d1 - want).abs().max() <= D_ATOL[gemm_path]
    assert (d0 - want).abs().max() > 100 * D_ATOL[gemm_path]


def test_geometry_refusals(cuda):
    ma = make("alex", random_lpips_state_dict("alex", 50), cuda, 1)
    mv = make("vgg", random_lpips_state_dict("vgg", 51), cuda, 1)
    with pytest.raises(L.FemasrError, match="at least 31"):
        ma(torch.rand(1, 3, 30, 64, device=cuda), torch.rand(1, 3, 30, 64, device=cuda))
    with pytest.raises(L.FemasrError, match="multiples of 16"):
        mv(torch.rand(1, 3, 32, 40, device=cuda), torch.rand(1, 3, 32, 40, device=cuda))
    with pytest.raises(L.FemasrError, match="different shapes"):
        ma(torch.rand(1, 3, 32, 32, device=cuda), torch.rand(1, 3, 32, 48, device=cuda))
    assert ma(torch.rand(1, 3, 31, 31, device=cuda), torch.rand(1, 3, 31, 31, device=cuda)).shape == (1, 1, 1, 1)


# ------------------------------------------------------------------------------------------------ kernels
def rel(got, want):
    return ((got.double().cpu() - want.double()).abs().max() / want.double().abs().max()).item()


@pytest.mark.parametrize("H,W", [(31, 31), (15, 22), (84, 127)])
def test_conv5x5_both_gemms(cuda, H, W):
    g = torch.Generator().manual_seed(60 + H)
    B, Cin, Cout = 2, 64, 192
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 5, 5, generator=g) * 0.03
    b = torch.randn(Cout, generator=g)
    want = F.relu(F.conv2d(x.double(), w.double(), b.double(), padding=2)).permute(0, 2, 3, 1)
    xd, wd, bd = nhwc(x).to(cuda), w.to(cuda), b.to(cuda)
    y0 = igemm(xd, pack_weight(wd), bd, B, H, W, Cin, Cout, ksize=5, act=L.ACT_RELU)
    hi, lo = tc_prepare(xd)
    y1 = tc_igemm(hi, lo, tc_pack(wd), bd, Cout, ksize=5, act=L.ACT_RELU)
    y2 = tc_igemm(hi, lo, tc_pack(wd), bd, Cout, ksize=5, act=L.ACT_RELU, slice_kb=4)
    for y, bar in ((y0, 1e-5), (y1, 2e-4), (y2, 1e-5)):
        assert y.shape == want.shape
        assert rel(y, want) <= bar


@pytest.mark.parametrize("H,W", [(63, 63), (31, 31), (3, 4), (335, 507)])
def test_pool3s2_staging_against_max_pool2d(cuda, H, W):
    g = torch.Generator().manual_seed(70)
    B, Cc = 2, 64
    x = torch.randn(B, H, W, Cc, generator=g) * 3
    xd = x.to(cuda)
    want = F.max_pool2d(xd.permute(0, 3, 1, 2), 3, 2).permute(0, 2, 3, 1).contiguous()
    lib = L.load()
    y = torch.empty_like(want)
    L.check(lib.femasr_maxpool3s2(p(xd), p(y), B, H, W, Cc, S()))
    assert torch.equal(y, want)                                        # exact: a max
    hi = torch.empty(want.shape, dtype=torch.float16, device=cuda)
    lo = torch.empty_like(hi)
    L.check(lib.femasr_tc_prepare(p(xd), p(hi), p(lo), L.PRO_MAXPOOL3S2, None, None, None, None, B, H, W, Cc, 0, 0.0, S()))
    assert torch.equal(hi, want.half())                                # the staging is the split of the pooled tensor
    assert torch.equal(lo, (want - hi.float()).half())


@pytest.mark.parametrize("normalize", [0, 1])
def test_im2col_k363_against_unfold(cuda, normalize):
    g = torch.Generator().manual_seed(80)
    B, H, W = 2, 37, 45
    x0, x1 = torch.rand(B, 3, H, W, generator=g), torch.rand(B, 3, H, W, generator=g)
    shift = torch.tensor([-0.030, -0.088, -0.188])
    scale = torch.tensor([0.458, 0.448, 0.450])
    Ho, Wo = (H + 4 - 11) // 4 + 1, (W + 4 - 11) // 4 + 1
    rows = []
    for x in (x0, x1):
        t = 2 * x - 1 if normalize else x
        t = (t - shift.view(1, 3, 1, 1)) / scale.view(1, 3, 1, 1)
        cols = F.unfold(t, 11, padding=2, stride=4).view(B, 3, 121, Ho * Wo)
        rows.append(cols.permute(0, 3, 2, 1).reshape(B * Ho * Wo, 363))     # k = tap * 3 + ci
    want = torch.zeros(2 * B * Ho * Wo, 384)
    want[:, :363] = torch.cat(rows)
    lib = L.load()
    xd0, xd1, sd, scd = x0.to(cuda), x1.to(cuda), shift.to(cuda), scale.to(cuda)
    f32 = torch.empty(2 * B * Ho * Wo, 384, device=cuda)
    L.check(lib.femasr_vgg_im2col_ex(p(xd0), p(xd1), B, H, W, 11, 4, 2, 384, p(sd), p(scd), normalize, None, None,
                                     p(f32), S()))
    assert torch.equal(f32.cpu(), want)
    hi = torch.empty(2 * B * Ho * Wo, 384, dtype=torch.float16, device=cuda)
    lo = torch.empty_like(hi)
    L.check(lib.femasr_vgg_im2col_ex(p(xd0), p(xd1), B, H, W, 11, 4, 2, 384, p(sd), p(scd), normalize, p(hi), p(lo),
                                     None, S()))
    assert torch.equal(hi, f32.half()) and torch.equal(lo, (f32 - hi.float()).half())
    w = torch.randn(64, 3, 11, 11, generator=g).to(cuda)
    wp = torch.empty(64, 384, device=cuda)
    L.check(lib.femasr_vgg_pad_weight_ex(p(w), p(wp), 64, 11, 384, S()))
    assert torch.equal(wp[:, :363].cpu(), w.permute(0, 2, 3, 1).reshape(64, 363).cpu()) and not wp[:, 363:].any()


@pytest.mark.parametrize("C,HW", [(64, 3969), (192, 961), (512, 256), (256, 1)])
def test_head_against_fp64(cuda, C, HW):
    g = torch.Generator().manual_seed(90 + C)
    B = 3
    f = torch.relu(torch.randn(2 * B, HW, C, generator=g))
    f[1, 0] = 0.0                                                      # an all-zero feature vector (norm + 1e-10)
    w = torch.rand(C, generator=g) * 0.3
    fd = f.double()
    n = fd / (fd.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)
    want = ((n[:B] - n[B:]).pow(2) * w.double()).sum(-1).mean(-1)
    lib = L.load()
    fc, wc = f.to(cuda), w.to(cuda)
    r = torch.zeros(5, B, device=cuda)
    r[:2] = torch.rand(2, B, generator=g).to(cuda)
    dist = torch.empty(B, device=cuda)
    scratch = torch.empty(lib.femasr_lpips_head_scratch_bytes(B, HW), dtype=torch.uint8, device=cuda)
    L.check(lib.femasr_lpips_head(p(fc), p(wc), B, HW, C, p(r), 2, p(dist), p(scratch), S()))
    got = r[2].double().cpu()
    assert (got - want).abs().max().item() <= 1e-6 * want.abs().max().item()
    assert torch.equal(dist, (r[0] + r[1]) + r[2])
    r2 = r.clone()
    L.check(lib.femasr_lpips_head(p(fc), p(wc), B, HW, C, p(r2), 2, None, p(scratch), S()))
    assert torch.equal(r2, r)                                          # fixed order: the same bits every run


def test_validate_script_on_png_pairs(cuda, tmp_path):
    cv2 = pytest.importorskip("cv2")
    from femasr_b200.spec import random_state_dict
    g = torch.Generator().manual_seed(100)
    lq, gt = tmp_path / "lq", tmp_path / "gt"
    lq.mkdir(); gt.mkdir()
    for i, (h, w) in enumerate(((16, 24), (16, 24), (24, 16))):
        cv2.imwrite(str(lq / f"im{i}.png"), (torch.rand(h, w, 3, generator=g) * 255).byte().numpy())
        cv2.imwrite(str(gt / f"im{i}.png"), (torch.rand(4 * h, 4 * w, 3, generator=g) * 255).byte().numpy())
    torch.save({"params": random_state_dict(4, 256, seed=3, init="perturbed")}, tmp_path / "net_g.pth")
    sd = random_lpips_state_dict("alex", 101)
    torch.save(sd, tmp_path / "lpips_alex.pth")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "validate_lpips.py"), "--lq", str(lq), "--gt", str(gt),
                          "-w", str(tmp_path / "net_g.pth"), "--lpips", "alex", "--lpips-weights", str(tmp_path / "lpips_alex.pth"),
                          "--codebook", "32,1024,256", "--scale", "4"],
                         capture_output=True, text=True, cwd=ROOT)
    assert out.returncode == 0, out.stderr
    vals = {ln.split()[0]: float(ln.split()[1]) for ln in out.stdout.splitlines() if ln.startswith("im")}
    assert sorted(vals) == ["im0.png", "im1.png", "im2.png"]
    # the same flow on the oracle side: the engine's SR output (uint8) against the GT, LPIPS by the ATen restatement
    from basicsr.archs.femasr_arch import FeMaSRNet
    net = FeMaSRNet(codebook_params=[[32, 1024, 256]], LQ_stage=True, scale_factor=4).eval()
    net.load_state_dict(torch.load(tmp_path / "net_g.pth")["params"], strict=True)
    net = net.to(cuda)
    for name, v in vals.items():
        img = torch.from_numpy(cv2.imread(str(lq / name))).to(cuda)[None]
        sr = net.sr_uint8(img)[0].cpu().flip(-1).permute(2, 0, 1).float() / 255.0
        ref = torch.from_numpy(cv2.imread(str(gt / name))).flip(-1).permute(2, 0, 1).float() / 255.0
        want = LO.forward("alex", sd, sr[None], ref[None], normalize=True).item()
        assert abs(v - want) <= 1e-4, (name, v, want)
    assert "mean lpips (alex) over 3 images" in out.stdout
