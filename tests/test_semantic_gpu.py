"""GPU: the HQ stage's semantic loss (use_semantic_loss=True) on the engine, on both GEMM paths - the reference's goldens
(tests/golden/semantic/) through the public surface, the vgg / semantic stage taps against the oracle, the main path left
bit-identical by the branch, CUDA-graph replay, the configurations where the reference raises, and the four new kernels
(ReLU epilogue, max-pool staging, normalising im2col, squared-difference rows) against ATen / fp64."""
import ctypes as C
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from femasr_b200 import lib as L
from femasr_b200.spec import random_state_dict
from tests import semantic_oracle as SO
from tests.golden_util import indices_of
from tests.gpu_util import S, igemm, nhwc, p, pack_weight, tc_igemm, tc_pack, tc_prepare
from tests.test_semantic import SEM_GOLDEN, SEM_IDS, load_sem_case

pytestmark = pytest.mark.gpu
# gemm_path 1 runs the VGG convs in ONE pass on the tensor cores, whose fp32 accumulator truncates: measured on an H100,
# relu4_4 comes out biased by -7.8e-5 (relative, the same sign everywhere) and the loss, a mean of squares, by about twice
# that (-1.6e-4 on hq_e512_sem_fwd_default, -8.7e-5 on hq_e512_sem_fwd).  K slices of 256 (measured with
# FEMASR_SEM_SLICE_KB=4, a study knob since removed) cut both tenfold; the branch only feeds a scalar loss, so the
# one-pass GEMM is kept and the bar covers its bias.
SEM_RTOL = {0: 2e-5, 1: 3e-4}


def make_net(scale, e_dim, sd, cuda, gemm_path, sem=True):
    from basicsr.archs.femasr_arch import FeMaSRNet
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)          # no VGG file here: weights come from sd
        net = FeMaSRNet(codebook_params=[[32, 1024, e_dim]], LQ_stage=scale != 1, scale_factor=scale,
                        use_semantic_loss=sem, gemm_path=gemm_path)
    net.load_state_dict(sd, strict=True)
    return net.to(cuda).eval()


def rel(got, want):
    return ((got.double().cpu() - want.double()).abs().max() / want.double().abs().max()).item()


@pytest.mark.parametrize("gemm_path", [0, 1])
@pytest.mark.parametrize("path", SEM_GOLDEN, ids=SEM_IDS)
def test_semantic_golden_through_public_surface(cuda, path, gemm_path):
    g, sd, _cbs = load_sem_case(path)
    scale, e_dim = int(g["scale"]), int(g["e_dim"])
    net = make_net(scale, e_dim, sd, cuda, gemm_path)
    x = torch.from_numpy(g["input"]).to(cuda)
    with torch.no_grad():
        if str(g["entry"]) == "forward":
            out, loss, sem, idx = net(x)
            mism = int((idx[0].cpu().numpy() != indices_of(g)[0]).sum())
            assert mism == 0, f"{mism} index mismatches"
            np.testing.assert_allclose(loss.item(), float(g["loss"]), rtol=2e-5)
            np.testing.assert_allclose(sem.item(), float(g["sem"]), rtol=SEM_RTOL[gemm_path])
        else:
            out = net.test(x)
    err = np.abs(out.cpu().numpy() - g["out"]).max()
    assert err <= 1e-3, f"output max-abs {err:.3e}"


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_semantic_taps_against_oracle(cuda, gemm_path):
    sd = random_state_dict(1, 512, seed=41, init="perturbed", semantic=True)
    net = make_net(1, 512, sd, cuda, gemm_path)
    x = torch.rand((2, 3, 64, 64), generator=torch.Generator().manual_seed(42))
    taps = {}
    with torch.no_grad():
        _out, _loss, wsem, _idx = SO.encode_and_decode(sd, x, 1, taps, semantic=True)
    eng = net._native(cuda)
    _y, _l, _i, sem, got = eng.forward(x.to(cuda), taps=["vgg", "semantic"], want_sem=True)
    errs = {n: rel(got[n].permute(0, 3, 1, 2), taps[n]) for n in ("vgg", "semantic")}
    print("relative stage errors:", {k: f"{v:.2e}" for k, v in errs.items()}, "sem", sem.item(), wsem.item())
    for n, v in errs.items():
        assert v <= 2e-4, f"stage {n}: relative max error {v:.3e}"
    assert abs(sem.item() - wsem.item()) <= SEM_RTOL[gemm_path] * abs(wsem.item())


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_branch_leaves_main_path_bit_identical(cuda, gemm_path):
    sd = random_state_dict(1, 512, seed=43, init="perturbed", semantic=True)
    base = {k: v for k, v in sd.items() if not k.startswith(("vgg_feat_extractor.", "conv_semantic."))}
    x = torch.rand((2, 3, 64, 64), generator=torch.Generator().manual_seed(44)).to(cuda)
    on = make_net(1, 512, sd, cuda, gemm_path)
    off = make_net(1, 512, base, cuda, gemm_path, sem=False)
    toggled = make_net(1, 512, sd, cuda, gemm_path)
    toggled.use_semantic_loss = False
    with torch.no_grad():
        runs = [net(x) for net in (on, off, toggled)]
    assert runs[0][2].item() > 0
    assert runs[1][2].item() == 0 and runs[2][2].item() == 0
    for out, loss, _sem, idx in runs[1:]:
        assert torch.equal(out, runs[0][0]) and torch.equal(loss, runs[0][1]) and torch.equal(idx[0], runs[0][3][0])


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_semantic_loss_stable_through_cuda_graph(cuda, gemm_path):
    sd = random_state_dict(1, 512, seed=45, init="perturbed", semantic=True)
    net = make_net(1, 512, sd, cuda, gemm_path)
    eng = net._native(cuda)
    if not eng.use_graph:
        pytest.skip("CUDA graphs disabled (FEMASR_CUDA_GRAPH=0)")
    x = torch.rand((1, 3, 64, 64), generator=torch.Generator().manual_seed(46)).to(cuda)
    sems, froms = [], []
    with torch.no_grad():
        for _ in range(3):                 # eager (first sighting), capture + replay, replay
            sems.append(net(x)[2].item())
            froms.append(eng.last_from_graph)
    assert froms == [False, True, True]
    assert sems[0] > 0 and sems[0] == sems[1] == sems[2]


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_lq_net_with_flag(cuda, gemm_path):
    """LQ x4 with the flag: test / test_tile / sr_uint8 never run VGG (femasr_arch.py:451-452, 467) and equal the
    flagless net bit for bit; forward raises like the reference (z_quant at H/2, relu4_4 at H/8)."""
    sd = random_state_dict(4, 512, seed=47, init="perturbed", semantic=True)
    base = {k: v for k, v in sd.items() if not k.startswith(("vgg_feat_extractor.", "conv_semantic."))}
    flag = make_net(4, 512, sd, cuda, gemm_path)
    plain = make_net(4, 512, base, cuda, gemm_path, sem=False)
    x = torch.rand((1, 3, 40, 24), generator=torch.Generator().manual_seed(48)).to(cuda)
    u8 = torch.randint(0, 256, (2, 24, 32, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(49)).to(cuda)
    with torch.no_grad():
        assert torch.equal(flag.test(x), plain.test(x))
        assert torch.equal(flag.test_tile(x, 16, 4), plain.test_tile(x, 16, 4))
        assert torch.equal(flag.sr_uint8(u8), plain.sr_uint8(u8))
        with pytest.raises(L.FemasrError, match="relu4_4"):
            flag(torch.rand((1, 3, 32, 32), device=cuda))
    hq256 = make_net(1, 256, random_state_dict(1, 256, seed=50, semantic=True), cuda, gemm_path)
    with torch.no_grad(), pytest.raises(L.FemasrError, match="512 channels"):
        hq256(torch.rand((1, 3, 64, 64), device=cuda))
    with torch.no_grad():
        hq256.test(torch.rand((1, 3, 40, 40), device=cuda))        # no loss requested: no error


def test_workspace_bytes_sem_without_sem_is_workspace_bytes(cuda):
    sd = random_state_dict(1, 512, seed=51, semantic=True)
    eng = make_net(1, 512, sd, cuda, 1)._native(cuda)
    lib = L.load()
    for B, H, W in ((1, 64, 64), (8, 256, 256)):
        a, b, s = C.c_size_t(), C.c_size_t(), C.c_size_t()
        L.check(lib.femasr_net_workspace_bytes(eng._h, B, H, W, C.byref(a)))
        L.check(lib.femasr_net_workspace_bytes_sem(eng._h, B, H, W, 0, C.byref(b)))
        L.check(lib.femasr_net_workspace_bytes_sem(eng._h, B, H, W, 1, C.byref(s)))
        assert a.value == b.value and s.value >= a.value


# ------------------------------------------------------------------------------------------------ kernels
def _split(v):
    c = v.clamp(-65504, 65504)
    hi = c.half()
    return hi, (c - hi.float()).half()


def test_relu_epilogue_both_gemms(cuda):
    g = torch.Generator().manual_seed(60)
    B, H, W, Cin, Cout = 2, 12, 20, 64, 128
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) * 0.05
    b = torch.randn(Cout, generator=g) * 0.5
    want = F.relu(F.conv2d(x.double(), w.double(), b.double(), padding=1)).permute(0, 2, 3, 1)
    xd, wd, bd = nhwc(x).to(cuda), w.to(cuda), b.to(cuda)
    y0 = igemm(xd, pack_weight(wd), bd, B, H, W, Cin, Cout, act=L.ACT_RELU)
    hi, lo = tc_prepare(xd)
    y1 = tc_igemm(hi, lo, tc_pack(wd), bd, Cout, act=L.ACT_RELU)
    for y in (y0, y1):
        assert (y >= 0).all()
        assert rel(y, want) <= 2e-5
    assert (want == 0).double().mean() > 0.3                    # the clamp is exercised


def test_maxpool_staging_is_split_of_max_pool(cuda):
    g = torch.Generator().manual_seed(61)
    B, H, W, Cc = 2, 18, 10, 128
    x = torch.randn(B, H, W, Cc, generator=g) * 3
    x[0, 0, 0, :8] = 1e5                                          # beyond fp16: the split clamps like tc_prepare
    xd = x.to(cuda)
    pooled = F.max_pool2d(x.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1).contiguous()
    hi, lo = torch.empty(B, H // 2, W // 2, Cc, dtype=torch.float16, device=cuda), None
    lo = torch.empty_like(hi)
    lib = L.load()
    L.check(lib.femasr_tc_prepare(p(xd), p(hi), p(lo), L.PRO_MAXPOOL2, None, None, None, None, B, H, W, Cc, 0, 0.0, S()))
    whi, wlo = _split(pooled)
    assert torch.equal(hi.cpu(), whi) and torch.equal(lo.cpu(), wlo)
    y = torch.empty(B, H // 2, W // 2, Cc, device=cuda)
    L.check(lib.femasr_maxpool2(p(xd), p(y), B, H, W, Cc, S()))
    assert torch.equal(y.cpu(), pooled)


def test_normalising_im2col_against_aten(cuda):
    g = torch.Generator().manual_seed(62)
    B, H, W = 2, 9, 14
    x = torch.rand(B, 3, H, W, generator=g)
    mean = torch.tensor([0.485, 0.456, 0.406])
    std = torch.tensor([0.229, 0.224, 0.225])
    norm = (x - mean.view(1, 3, 1, 1)) / std.view(1, 3, 1, 1)
    cols = F.unfold(norm, 3, padding=1).view(B, 3, 9, H * W)             # [B, ci, tap, pix]
    want = torch.zeros(B, H * W, 64)
    want[:, :, :27] = cols.permute(0, 3, 2, 1).reshape(B, H * W, 27)      # k = tap * 3 + ci
    want = want.view(B * H * W, 64)
    lib = L.load()
    xd, md, sdv = x.to(cuda), mean.to(cuda), std.to(cuda)
    f32 = torch.empty(B * H * W, 64, device=cuda)
    L.check(lib.femasr_vgg_im2col(p(xd), p(md), p(sdv), None, None, p(f32), B, H, W, S()))
    assert torch.equal(f32.cpu(), want)
    hi = torch.empty(B * H * W, 64, dtype=torch.float16, device=cuda)
    lo = torch.empty_like(hi)
    L.check(lib.femasr_vgg_im2col(p(xd), p(md), p(sdv), p(hi), p(lo), None, B, H, W, S()))
    whi, wlo = _split(want)
    assert torch.equal(hi.cpu(), whi) and torch.equal(lo.cpu(), wlo)
    # conv1_1 as the padded-weight GEMM equals the 3x3 conv of the normalised image
    w = torch.randn(64, 3, 3, 3, generator=g) * 0.2
    wp = torch.empty(64, 64, device=cuda)
    L.check(lib.femasr_vgg_pad_weight(p(w.to(cuda)), p(wp), 64, S()))
    y = F.conv2d(norm.double(), w.double(), padding=1).permute(0, 2, 3, 1).reshape(-1, 64)
    assert rel(f32 @ wp.t(), y) <= 1e-5


def test_sq_diff_rows_against_fp64(cuda):
    g = torch.Generator().manual_seed(63)
    N, Cc = 1000, 512
    a, b = torch.randn(N, Cc, generator=g), torch.randn(N, Cc, generator=g)
    ad, bd = a.to(cuda), b.to(cuda)
    rows = torch.empty(N, device=cuda)
    lib = L.load()
    L.check(lib.femasr_sq_diff_rows(p(ad), p(bd), p(rows), N, Cc, S()))
    want = ((a.double() - b.double()) ** 2).sum(1)
    assert ((rows.double().cpu() - want).abs() / want).max().item() <= 1e-5
    rows2 = torch.empty_like(rows)
    L.check(lib.femasr_sq_diff_rows(p(ad), p(bd), p(rows2), N, Cc, S()))
    assert torch.equal(rows, rows2)                               # fixed order: deterministic
    out = torch.empty((), device=cuda)
    L.check(lib.femasr_sum_scaled(p(rows), p(out), N, 1.0 / (N * Cc), S()))
    assert abs(out.item() - F.mse_loss(a.double(), b.double()).item()) <= 1e-5 * out.item()
