"""The ping-pong schedule of the tensor-core implicit GEMM (tc_igemm_kernel's PP): each consumer warpgroup owns whole
128-row tiles and the two take turns on the tensor cores.  plan_tiles runs every BN-64 launch that is not K-sliced on it.

Every launch class the schedule runs (BN 64: F8 columns with and without residuals and GroupNorm partials, the F8
tap-order schedule, the F8 sub-pixel up conv, the plain 3x3, 4x4 stride-2 and 5x5 taps, linears with GELU and split
output or a residual, the im2col first-conv GEMM) is covered, plus the edge tilings: a ragged 127 x 127 map, fewer
tiles than SMs, an odd number of tiles per CTA, and a single tile.  The outputs are checked against fp64 with
tests/test_gemm_matrix_gpu.py's bars, every GroupNorm partial row must be written, and the partials must sum to the
output's per-group sums."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import gpu_util as G
from tests.test_gemm_matrix_gpu import tile_shape

pytestmark = pytest.mark.gpu

GELU, LRELU = 1, 3


def columns_apply(H, W):
    """plan_tiles (tc_gemm.cu): the column schedule's 8 x 16 tiles cover the map with no more tiles than tc_tile_shape's."""
    wt, ht = tile_shape(H, W)
    return math.ceil(W / 8) * math.ceil(H / 16) == math.ceil(W / wt) * math.ceil(H / ht)


def cases(sms):
    """name -> (B, H, W, Cin, Cout, ksize, stride, up, f8, res1, res2, gn, act, split); sms: the device's SM count."""
    odd = 3 * sms * 128                   # 3 tiles per CTA: warpgroup 0 takes two and warpgroup 1 one
    return {
        "f8-cols-64to64-gn": (2, 48, 48, 64, 64, 3, 1, 0, 1, False, False, True, 0, False),
        "f8-cols-128to64-res-res2-gn": (2, 48, 48, 128, 64, 3, 1, 0, 1, True, True, True, 0, False),
        "f8-taps-ragged127-64to64-res-gn": (1, 127, 127, 64, 64, 3, 1, 0, 1, True, False, True, 0, False),
        "f8-up-128to64": (1, 40, 24, 128, 64, 3, 1, 1, 1, False, False, False, 0, False),
        "bn64-3x3-64to64-gn": (2, 13, 37, 64, 64, 3, 1, 0, 0, True, False, True, 0, False),
        "bn64-4x4s2-lrelu": (2, 27, 75, 64, 64, 4, 2, 0, 0, False, False, False, LRELU, False),
        "bn64-5x5-res": (1, 23, 29, 64, 64, 5, 1, 0, 0, True, False, False, 0, False),
        "linear-256to192-gelu-split": (1, 1, 4000, 256, 192, 1, 1, 0, 0, False, False, False, GELU, True),
        "linear-256to64-res": (1, 1, 3000, 256, 64, 1, 1, 0, 0, True, False, False, 0, False),
        "im2col-gemm-64to64-split": (2, 33, 47, 64, 64, 1, 1, 0, 0, False, False, False, 0, True),
        "fewer-tiles-than-sms": (1, 16, 24, 128, 64, 3, 1, 0, 0, True, False, True, 0, False),
        "odd-tiles-per-cta": (1, 1, odd, 256, 64, 1, 1, 0, 0, True, False, False, 0, False),
        "one-tile": (1, 1, 100, 64, 64, 1, 1, 0, 0, False, False, False, 0, False),
    }


def data(name, c):
    B, H, W, Cin, Cout, k, stride, up, f8, res1, res2, gn, act, split = c
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = torch.randn(B, Cin, H, W, generator=g)
    if not f8:
        hi = x.half()
        x = hi.float() + (x - hi.float()).half().float()      # exactly what the split planes hold
    w = torch.randn(Cout, Cin, k, k, generator=g) * 0.03
    b = torch.randn(Cout, generator=g)
    Ho, Wo = ((H + 2 - k) // 2 + 1, (W + 2 - k) // 2 + 1) if stride == 2 else (H * (1 + up), W * (1 + up))
    r1 = torch.randn(B, Cout, Ho, Wo, generator=g) if res1 else None
    r2 = torch.randn(B, Cout, Ho, Wo, generator=g) if res2 else None
    return x, w, b, r1, r2


def run(name, c, cuda):
    """The launch: {output (fp32, or the hi and lo planes), GroupNorm partials} on the CPU."""
    B, H, W, Cin, Cout, k, stride, up, f8, res1, res2, gn, act, split = c
    x, w, b, r1, r2 = data(name, c)
    xd = G.nhwc(x).to(cuda)
    if f8:
        hi, lo = G.tc_prepare_f8(xd)
        blob = G.tc_pack_f8(w.to(cuda), up2=bool(up))
    else:
        hi, lo = G.tc_prepare(xd)
        blob = G.tc_pack_up2(w.to(cuda)) if up else G.tc_pack(w.to(cuda))
    part = None
    if gn:
        part = torch.full((B, G.tc_gn_rows(B, H, W, Cin, Cout, upsample=up), 32, 2), float("nan"), device=cuda)
    dev = lambda t: None if t is None else G.nhwc(t).to(cuda)
    out = G.tc_igemm(hi, lo, blob, b.to(cuda), Cout, k, act=act, res1=dev(r1), res2=dev(r2), upsample=up, stride=stride,
                     split_out=split, gn_partial=part, f8=f8)
    torch.cuda.synchronize()
    res = {"hi": out[0].cpu(), "lo": out[1].cpu()} if split else {"y": out.cpu()}
    if gn:
        res["gn"] = part.cpu()
    return res


def reference(name, c):
    B, H, W, Cin, Cout, k, stride, up, f8, res1, res2, gn, act, split = c
    x, w, b, r1, r2 = data(name, c)
    v = x.double()
    if up:
        v = v.repeat_interleave(2, 2).repeat_interleave(2, 3)
    y = F.conv2d(v, w.double(), b.double(), stride=stride, padding={1: 0, 3: 1, 4: 1, 5: 2}[k])
    if act == GELU:
        y = F.gelu(y)
    elif act == LRELU:
        y = F.leaky_relu(y, 0.2)
    for r in (r1, r2):
        if r is not None:
            y = y + r.double()
    return y.permute(0, 2, 3, 1).contiguous()


def bar(c):
    """test_gemm_matrix_gpu.tc_bar: one pass 2e-5, F8 1.5e-4, GELU + 1e-5."""
    f8, act = c[8], c[12]
    return (1.5e-4 if f8 else 2e-5) + (1e-5 if act == GELU else 0.0)


def test_tc_pingpong_case_shapes():
    """The cases exercise what their names say (the tiling rule of plan_tiles, CPU only)."""
    cs = cases(132)
    for name in ("f8-cols-64to64-gn", "f8-cols-128to64-res-res2-gn"):
        assert columns_apply(*cs[name][1:3]), name
    assert not columns_apply(127, 127) and tile_shape(127, 127) == (128, 1)     # the TMA clips every tile's last row
    B, H, W = cs["fewer-tiles-than-sms"][:3]
    wt, ht = tile_shape(H, W)
    assert B * math.ceil(H / ht) * math.ceil(W / wt) < 132
    assert cs["odd-tiles-per-cta"][2] // 128 == 3 * 132 and cs["one-tile"][2] <= 128


NAMES = list(cases(132))


@pytest.mark.parametrize("name", NAMES)
def test_tc_pingpong_against_fp64(cuda, name):
    c = cases(torch.cuda.get_device_properties(cuda).multi_processor_count)[name]
    got = run(name, c, cuda)
    y = got["y"] if "y" in got else got["hi"].float() + got["lo"].float()
    want = reference(name, c)
    e = ((y.double() - want).abs().max() / want.abs().max()).item()
    print(f"{name}: rel err {e:.2e}")
    assert e <= bar(c)
    if "gn" in got:
        gn = got["gn"]
        assert not torch.isnan(gn).any(), "every GroupNorm partial row is written"
        B, Cout = c[0], c[4]
        s = gn[..., 0].double().sum(1)            # per (image, channel group) over all tiles and quarters
        ss = gn[..., 1].double().sum(1)
        yg = y.double().reshape(B, -1, 32, Cout // 32)
        assert ((s - yg.sum((1, 3))).abs() <= 1e-5 * yg.abs().sum((1, 3)) + 1e-6).all()
        assert ((ss - (yg * yg).sum((1, 3))).abs() <= 1e-5 * (yg * yg).sum((1, 3)) + 1e-6).all()
