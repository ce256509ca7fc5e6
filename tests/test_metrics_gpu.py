"""GPU: PSNR / SSIM on the engine - the goldens (tests/golden/metrics/) through femasr_b200.metrics, the device against
the CPU oracle on fresh seeded inputs, exact identities, exact symmetry, batch invariance, the refusals, and
scripts/validate.py on generated PNG pairs against the oracle and scripts/validate_lpips.py."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from femasr_b200 import lib as L
from tests import metrics_oracle as MO
from tests.test_metrics import (METRICS_GOLDEN, METRICS_IDS, PSNR_GOLDEN_ATOL, SSIM_GOLDEN_ATOL, LQ_CONFIG,
                                load_metrics_case)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# Device against the oracle (dB; SSIM units).  Both bars are below one fp32 ulp of the score, so they effectively ask for
# the same fp32 value: the fp64 sums of the separable device filter and of the oracle's 2-D conv2d run in different
# orders and agree to about 1e-15 relative, so only a score lying within that of an fp32 rounding boundary could differ
# by one ulp.  A failure by exactly one ulp would be such a rounding flip, not a kernel error.
PSNR_ATOL, SSIM_ATOL = 1e-6, 1e-10
MODES = [(False, "yiq"), (True, "yiq"), (True, "ycbcr")]
MODE_IDS = ["rgb", "yiq", "ycbcr"]


def metrics(ty, crop, space):
    from femasr_b200.metrics import PSNR, SSIM
    return PSNR(ty, crop, space), SSIM(ty, crop, space)


@pytest.mark.parametrize("path", METRICS_GOLDEN, ids=METRICS_IDS)
def test_goldens_through_public_surface(cuda, path):
    from femasr_b200.metrics import create_metric
    g, x, y, opts = load_metrics_case(path)
    p = create_metric("psnr", **opts)(x.to(cuda), y.to(cuda))
    s = create_metric("ssim", better="higher", **opts)(x.to(cuda), y.to(cuda))
    B = x.shape[0]
    assert p.shape == (B,) and s.shape == (B,) and p.dtype == s.dtype == torch.float32
    perr = np.abs(p.cpu().double().numpy() - g["psnr"]).max()
    serr = np.abs(s.cpu().double().numpy() - g["ssim"]).max()
    print(f"{os.path.basename(path)}: |psnr - golden| {perr:.2e} dB, |ssim - golden| {serr:.2e}")
    assert perr <= PSNR_GOLDEN_ATOL and serr <= SSIM_GOLDEN_ATOL
    if B == 1:
        assert isinstance(p.item(), float)


@pytest.mark.parametrize("ty,space", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("B,H,W,crop", [(3, 37, 53, 0), (2, 200, 301, 4), (1, 11, 19, 0), (1, 1344 // 4, 2032 // 4, 4)])
def test_device_against_oracle(cuda, ty, space, B, H, W, crop):
    g = torch.Generator().manual_seed(H * 7 + W)
    x = torch.rand(B, 3, H, W, generator=g)
    y = (x + 0.03 * torch.randn(B, 3, H, W, generator=g)).clamp(0, 1)
    y[-1] = torch.rand(3, H, W, generator=g)                         # one unrelated pair
    mp, ms = metrics(ty, crop, space)
    p, s = mp(x.to(cuda), y.to(cuda)).cpu(), ms(x.to(cuda), y.to(cuda)).cpu()
    wp, ws = MO.psnr(x, y, ty, crop, space), MO.ssim(x, y, ty, crop, space)
    print(f"{B}x{H}x{W} crop {crop} {space if ty else 'rgb'}: |dpsnr| {(p.double() - wp.double()).abs().max():.2e} dB, "
          f"|dssim| {(s.double() - ws.double()).abs().max():.2e}")
    assert (p.double() - wp.double()).abs().max() <= PSNR_ATOL
    assert (s.double() - ws.double()).abs().max() <= SSIM_ATOL


@pytest.mark.parametrize("ty,space", MODES, ids=MODE_IDS)
def test_identities_symmetry_and_batch_invariance(cuda, ty, space):
    g = torch.Generator().manual_seed(5)
    x = torch.rand(3, 3, 67, 93, generator=g).to(cuda)
    y = (x + 0.05 * torch.randn(3, 3, 67, 93, generator=g).to(cuda)).clamp(0, 1)
    for m in metrics(ty, 4, space):
        same = 80.0 if m._name == "psnr" else 1.0
        assert torch.equal(m(x, x.clone()), torch.full((3,), same, device=cuda))
        xy, yx = m(x, y), m(y, x)
        assert torch.equal(xy, yx)
        for b in range(3):
            assert torch.equal(m(x[b:b + 1], y[b:b + 1]), xy[b:b + 1])         # image b alone == inside the batch
        assert torch.equal(m(x, y), xy)                                      # the same bits every run


def test_refusals_through_public_surface(cuda):
    from femasr_b200.metrics import PSNR, SSIM
    x = torch.rand(2, 3, 32, 40, device=cuda)
    with pytest.raises(L.FemasrError, match="crop"):
        PSNR(crop_border=16)(x, x)
    with pytest.raises(L.FemasrError, match="crop"):
        SSIM(crop_border=-1)(x, x)
    with pytest.raises(L.FemasrError, match="11x11"):
        SSIM(crop_border=11)(x, x)
    with pytest.raises(L.FemasrError, match="one shape"):
        PSNR()(x, x[:, :, :31])
    with pytest.raises(L.FemasrError, match="one shape"):
        SSIM()(x[:, :1], x[:, :1])
    with pytest.raises(L.FemasrError, match="fp32"):
        PSNR()(x.double(), x.double())
    with pytest.raises(L.FemasrError, match="no CPU fallback"):
        SSIM()(x, x.cpu())
    big = torch.zeros(65536, 3, 1, 1, device=cuda)
    with pytest.raises(L.FemasrError, match="65535"):
        PSNR()(big, big)
    assert PSNR(crop_border=15)(x, x).tolist() == [80.0, 80.0]              # a 2x10 cropped image is fine for PSNR
    assert SSIM(crop_border=10)(x, x).tolist() == [1.0, 1.0]                # 12x20: SSIM's smallest sides are 11


def test_lpips_metric_matches_lpips_module(cuda):
    from femasr_b200.metrics import create_metric
    from femasr_b200.spec import random_lpips_state_dict
    with pytest.warns(UserWarning):
        m = create_metric("lpips")
    m.net.load_state_dict(random_lpips_state_dict("alex", 3), strict=True)
    m = m.to(cuda)
    g = torch.Generator().manual_seed(9)
    x, y = torch.rand(2, 3, 64, 64, generator=g).to(cuda), torch.rand(2, 3, 64, 64, generator=g).to(cuda)
    assert torch.equal(m(x, y), m.net(x, y, normalize=True).view(2))


def test_validate_script_on_png_pairs(cuda, tmp_path):
    cv2 = pytest.importorskip("cv2")
    pytest.importorskip("yaml")
    from basicsr.archs.femasr_arch import FeMaSRNet
    from femasr_b200.spec import random_lpips_state_dict, random_state_dict
    g = torch.Generator().manual_seed(110)
    lq, gt = tmp_path / "lq", tmp_path / "gt"
    lq.mkdir(); gt.mkdir()
    for i, (h, w) in enumerate(((16, 24), (16, 24), (24, 16), (16, 24))):
        cv2.imwrite(str(lq / f"im{i}.png"), (torch.rand(h, w, 3, generator=g) * 255).byte().numpy())
        cv2.imwrite(str(gt / f"im{i}.png"), (torch.rand(4 * h, 4 * w, 3, generator=g) * 255).byte().numpy())
    torch.save({"params": random_state_dict(4, 256, seed=3, init="perturbed")}, tmp_path / "net_g.pth")
    torch.save(random_lpips_state_dict("alex", 111), tmp_path / "lpips_alex.pth")
    (tmp_path / "opt.yml").write_text(LQ_CONFIG.replace("[32, 1024, 512]", "[32, 1024, 256]"))
    common = ["--lq", str(lq), "--gt", str(gt), "-w", str(tmp_path / "net_g.pth"), "--lpips-weights",
              str(tmp_path / "lpips_alex.pth")]
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "validate.py"), "-opt", str(tmp_path / "opt.yml"),
                          *common, "--batch", "2"], capture_output=True, text=True, cwd=ROOT)
    assert out.returncode == 0, out.stderr
    print(out.stdout)
    lines = out.stdout.splitlines()
    rows = {ln.split()[0]: dict(zip(ln.split()[1::2], map(float, ln.split()[2::2]))) for ln in lines if ln.startswith("im")}
    assert sorted(rows) == [f"im{i}.png" for i in range(4)] and all(list(r) == ["psnr", "ssim", "lpips"] for r in rows.values())
    assert lines[-2].startswith("mean over 4 images: psnr ") and lines[-1] == "key metric: lpips"
    ref = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "validate_lpips.py"), *common, "--lpips", "alex",
                          "--codebook", "32,1024,256", "--scale", "4"], capture_output=True, text=True, cwd=ROOT)
    assert ref.returncode == 0, ref.stderr
    ref_lines = {ln.split()[0]: ln.split()[1] for ln in ref.stdout.splitlines() if ln.startswith("im")}
    for name in rows:
        assert f"{rows[name]['lpips']:.6f}" == ref_lines[name]
    net = FeMaSRNet(codebook_params=[[32, 1024, 256]], LQ_stage=True, scale_factor=4).eval()
    net.load_state_dict(torch.load(tmp_path / "net_g.pth")["params"], strict=True)
    net = net.to(cuda)
    from femasr_b200.folders import rgb01
    for name, r in rows.items():
        # the tensors validate.py scores: sr_uint8's output and the GT, both converted to [0, 1] on the device by rgb01
        img = torch.from_numpy(cv2.imread(str(lq / name))).to(cuda)[None]
        sr = rgb01(net.sr_uint8(img)).cpu()
        ref_gt = rgb01(torch.from_numpy(cv2.imread(str(gt / name))).to(cuda)[None]).cpu()
        # printed to 6 decimals: half a unit of the last digit plus the device-oracle bar
        assert abs(MO.psnr(sr, ref_gt, True, 4, "yiq").item() - r["psnr"]) <= 5e-7 + PSNR_ATOL
        assert abs(MO.ssim(sr, ref_gt, True, 4, "yiq").item() - r["ssim"]) <= 5e-7 + SSIM_ATOL
