"""CPU: PSNR / SSIM (femasr_b200.metrics) - the oracle (tests/metrics_oracle.py) against the goldens
(tests/golden/metrics/), its exact identities, create_metric's mapping and refusals, the C entry points' argument
refusals without a GPU, and scripts/validate.py's reading of both training configs' val blocks."""
import ctypes as C
import glob
import importlib.util
import os

import numpy as np
import pytest
import torch

from tests import metrics_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
METRICS_GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "metrics", "*.npz")))
METRICS_IDS = [os.path.basename(p)[:-4] for p in METRICS_GOLDEN]
PSNR_GOLDEN_ATOL, SSIM_GOLDEN_ATOL = 1e-5, 1e-7      # dB; SSIM units


def load_metrics_case(path):
    """(record, x, y, metric options) of a golden file; x, y [B,3,H,W] fp32 = uint8 / 255."""
    g = np.load(path)
    space = str(g["color_space"])
    opts = dict(test_y_channel=space != "rgb", crop_border=int(g["crop_border"]),
                color_space=space if space != "rgb" else "yiq")
    return g, torch.from_numpy(g["x_u8"]).float() / 255.0, torch.from_numpy(g["y_u8"]).float() / 255.0, opts


def load_validate_script():
    spec = importlib.util.spec_from_file_location("validate_script", os.path.join(ROOT, "scripts", "validate.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_goldens_cover_the_configs():
    seen = set()
    for path in METRICS_GOLDEN:
        g, x, _y, opts = load_metrics_case(path)
        seen.add((str(g["color_space"]), opts["crop_border"], x.shape[0]))
    assert {s for s, _c, _b in seen} == {"rgb", "yiq", "ycbcr"}
    assert {c for _s, c, _b in seen} == {0, 4} and {b for *_, b in seen} == {1, 3}
    assert ("yiq", 4, 3) in seen and ("ycbcr", 4, 1) in seen           # the LQ and HQ configs' settings


@pytest.mark.parametrize("path", METRICS_GOLDEN, ids=METRICS_IDS)
def test_oracle_matches_goldens(path):
    g, x, y, opts = load_metrics_case(path)
    p = MO.psnr(x, y, **opts).double().numpy()
    s = MO.ssim(x, y, **opts).double().numpy()
    assert np.abs(p - g["psnr"]).max() <= PSNR_GOLDEN_ATOL
    assert np.abs(s - g["ssim"]).max() <= SSIM_GOLDEN_ATOL
    assert 10 < g["psnr"].min() and g["psnr"].max() < 35 and 0.1 < g["ssim"].min() and g["ssim"].max() < 0.9


def test_oracle_identities():
    x = torch.rand(2, 3, 23, 29, generator=torch.Generator().manual_seed(1))
    for space in ("yiq", "ycbcr"):
        for ty in (False, True):
            assert torch.equal(MO.psnr(x, x.clone(), ty, 2, space), torch.full((2,), 80.0))
            assert torch.equal(MO.ssim(x, x.clone(), ty, 2, space), torch.ones(2))


def test_create_metric_mapping_and_refusals():
    from femasr_b200.lpips import LPIPS
    from femasr_b200.metrics import PSNR, SSIM, LPIPSMetric, create_metric
    p = create_metric("psnr", crop_border=4, test_y_channel=True, better="higher")
    assert isinstance(p, PSNR) and (p.test_y_channel, p.crop_border, p.color_space) == (True, 4, "yiq")
    assert not PSNR().test_y_channel and SSIM().test_y_channel                       # pyiqa's defaults
    s = create_metric("ssim", crop_border=4, test_y_channel=True, color_space="ycbcr")
    assert isinstance(s, SSIM) and s.color_space == "ycbcr" and s.crop_border == 4
    with pytest.warns(UserWarning, match="untrained"):
        la = create_metric("lpips", better="lower")
    with pytest.warns(UserWarning, match="untrained"):
        lv = create_metric("lpips-vgg")
    assert isinstance(la, LPIPSMetric) and isinstance(la.net, LPIPS)
    assert la.net.pnet_type == "alex" and lv.net.pnet_type == "vgg"
    with pytest.raises(ValueError, match="'niqe'"):
        create_metric("niqe")
    with pytest.raises(TypeError, match="'data_range'"):
        create_metric("psnr", data_range=255)
    with pytest.raises(TypeError, match="'net'"):
        create_metric("lpips", net="squeeze")
    with pytest.raises(NotImplementedError, match="as_loss"):
        create_metric("lpips-vgg", as_loss=True)
    with pytest.raises(NotImplementedError, match="downsample"):
        create_metric("ssim", downsample=True)
    with pytest.raises(ValueError, match="'lab'"):
        create_metric("psnr", test_y_channel=True, color_space="lab")


def test_cpu_tensors_are_refused():
    from femasr_b200.lib import FemasrError
    from femasr_b200.metrics import PSNR, SSIM
    x = torch.rand(1, 3, 16, 16)
    for m in (PSNR(), SSIM()):
        with pytest.raises(FemasrError, match="no CPU fallback"):
            m(x, x)


def test_entry_point_refusals(built_lib):
    from femasr_b200 import lib as L
    lib = L.load()
    ptr = C.c_void_p(256)                     # never dereferenced: every case below is refused first
    for kind, fn in ((L.METRIC_PSNR, lib.femasr_psnr), (L.METRIC_SSIM, lib.femasr_ssim)):
        name = b"psnr" if kind == L.METRIC_PSNR else b"ssim"
        assert lib.femasr_metric_scratch_bytes(kind, 2, 64, 48, 4) > 0
        cases = [((None, ptr, 1, 32, 32, 0, 0, ptr, ptr), b"null"),
                 ((ptr, ptr, 1, 32, 32, 0, 0, None, ptr), b"null"),
                 ((ptr, ptr, 1, 32, 32, 0, 0, ptr, None), b"null"),
                 ((ptr, ptr, 0, 32, 32, 0, 0, ptr, ptr), b"65535"),
                 ((ptr, ptr, 65536, 32, 32, 0, 0, ptr, ptr), b"65535"),
                 ((ptr, ptr, 1, 32, 32, -1, 0, ptr, ptr), b"crop"),
                 ((ptr, ptr, 1, 32, 40, 16, 0, ptr, ptr), b"crop"),
                 ((ptr, ptr, 1, 40, 32, 16, 0, ptr, ptr), b"crop"),
                 ((ptr, ptr, 1, 32, 32, 0, 3, ptr, ptr), b"mode")]
        for args, why in cases:
            assert fn(*args, None) == -1                                     # FEMASR_ERR_ARG
            msg = lib.femasr_last_error()
            assert name in msg and why in msg, (args, msg)
            B, H, W, crop = args[2:6]
            if why != b"null" and why != b"mode":
                assert lib.femasr_metric_scratch_bytes(kind, B, H, W, crop) == 0
    # SSIM needs an 11x11 cropped image; PSNR takes a single pixel
    assert lib.femasr_ssim(ptr, ptr, 1, 18, 40, 4, 0, ptr, ptr, None) == -1
    assert b"11x11" in lib.femasr_last_error()
    assert lib.femasr_metric_scratch_bytes(L.METRIC_SSIM, 1, 18, 40, 4) == 0
    assert lib.femasr_metric_scratch_bytes(L.METRIC_SSIM, 1, 19, 19, 4) > 0
    assert lib.femasr_metric_scratch_bytes(L.METRIC_PSNR, 1, 9, 9, 4) > 0
    assert lib.femasr_metric_scratch_bytes(2, 1, 64, 64, 0) == 0


LQ_CONFIG = """
scale: &upscale 4
network_g:
  type: FeMaSRNet
  gt_resolution: 256
  norm_type: 'gn'
  act_type: 'silu'
  scale_factor: *upscale
  codebook_params:
    - [32, 1024, 512]
  LQ_stage: true
  frozen_module_keywords: ['quantize', 'decoder', 'after_quant_group', 'out_conv']
val:
  val_freq: !!float 5e3
  save_img: true
  key_metric: lpips
  metrics:
    psnr: # metric name, can be arbitrary
      type: psnr
      crop_border: 4
      test_y_channel: true
    ssim:
      type: ssim
      crop_border: 4
      test_y_channel: true
    lpips:
      type: lpips
      better: lower
"""

HQ_CONFIG = """
network_g:
  type: FeMaSRNet
  gt_resolution: 256
  norm_type: 'gn'
  act_type: 'silu'
  use_semantic_loss: true
  codebook_params:
    - [32, 1024, 512]
  LQ_stage: false
  use_quantize: true
val:
  val_freq: !!float 5e3
  save_img: false
  key_metric: lpips
  metrics:
    psnr: # metric name, not used in this codebase
      type: psnr
      crop_border: 4
      test_y_channel: true
      color_space: ycbcr
    ssim:
      type: ssim
      crop_border: 4
      test_y_channel: true
      color_space: ycbcr
    lpips:
      type: lpips
      better: lower
"""


@pytest.mark.parametrize("config,space", [(LQ_CONFIG, "yiq"), (HQ_CONFIG, "ycbcr")], ids=["lq", "hq"])
def test_validate_reads_config_val_blocks(tmp_path, config, space):
    pytest.importorskip("yaml")
    from femasr_b200.metrics import PSNR, SSIM, LPIPSMetric
    v = load_validate_script()
    path = tmp_path / "opt.yml"
    path.write_text(config)
    opt = v.load_options(str(path))
    key, plan = v.metric_plan(opt)
    assert key == "lpips"
    assert plan == [("psnr", "psnr", {"crop_border": 4, "test_y_channel": True, **({"color_space": "ycbcr"} if space == "ycbcr" else {})}),
                    ("ssim", "ssim", {"crop_border": 4, "test_y_channel": True, **({"color_space": "ycbcr"} if space == "ycbcr" else {})}),
                    ("lpips", "lpips", {})]
    lp = tmp_path / "lpips.pth"
    from femasr_b200.spec import random_lpips_state_dict
    torch.save(random_lpips_state_dict("alex", 0), lp)
    metrics = v.build_metrics(plan, [str(lp)], torch.device("cpu"))
    assert isinstance(metrics["psnr"], PSNR) and isinstance(metrics["ssim"], SSIM)
    assert isinstance(metrics["lpips"], LPIPSMetric)
    for m in (metrics["psnr"], metrics["ssim"]):
        assert (m.test_y_channel, m.crop_border, m.color_space) == (True, 4, space)
    assert torch.equal(metrics["lpips"].net.state_dict()["lin2.model.1.weight"], torch.load(lp)["lin2.model.1.weight"])
    with pytest.raises(SystemExit, match="--lpips-weights"):
        v.build_metrics(plan, None, torch.device("cpu"))
