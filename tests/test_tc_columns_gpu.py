"""The column schedule of the tensor-core implicit GEMM (stride-1 3x3 convs in F8 mode: 8 x 16 tiles, one activation
column box per (channel chunk, dx) for the three taps dy) against fp64, at sides that are not multiples of 16 or 8, one
to four channel chunks, BN 64 and 128, with and without a residual and GroupNorm partials.

The schedule runs where its 8 x 16 tiling needs no more tiles than tc_tile_shape's; every case asserts that, and the
GroupNorm partial rows are checked one by one against the 8 x 4 pixel quarter of the 8 x 16 tile each one covers, which
only the column tiling produces at these shapes."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import gpu_util as G
from tests.test_gemm_matrix_gpu import assert_canaries, guarded, rel_err, tile_shape

pytestmark = pytest.mark.gpu

# B, H, W, Cin, Cout, residual, GroupNorm partials
CASES = [
    (2, 30, 15, 64, 64, False, True),        # 1 chunk, BN 64
    (3, 30, 15, 128, 64, True, False),       # 2 chunks, BN 64
    (1, 47, 31, 192, 128, True, True),       # 3 chunks, BN 128
    (2, 33, 23, 256, 256, True, True),       # 4 chunks, BN 128 x 2 n-tiles
    (1, 47, 31, 256, 128, False, False),
]


def columns_apply(H, W):
    """plan_tiles (tc_gemm.cu): the column schedule's 8 x 16 tiles cover the map with no more tiles than tc_tile_shape's."""
    wt, ht = tile_shape(H, W)
    return math.ceil(W / 8) * math.ceil(H / 16) == math.ceil(W / wt) * math.ceil(H / ht)


@pytest.mark.parametrize("B,H,W,Cin,Cout,res,gn", CASES, ids=[f"{c[0]}x{c[1]}x{c[2]}-{c[3]}to{c[4]}" +
                                                             ("-res" if c[5] else "") + ("-gn" if c[6] else "")
                                                             for c in CASES])
def test_column_schedule_against_fp64(cuda, B, H, W, Cin, Cout, res, gn):
    assert columns_apply(H, W) and tile_shape(H, W) != (8, 16) and H % 16 and W % 8
    g = torch.Generator().manual_seed(B * 1000003 + H * 1009 + W * 31 + Cin + Cout)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) * 0.03
    b = torch.randn(Cout, generator=g)
    r = torch.randn(B, Cout, H, W, generator=g) if res else None
    want = F.conv2d(x.double(), w.double(), b.double(), padding=1)
    if res:
        want = want + r.double()
    want = want.permute(0, 2, 3, 1).contiguous()

    hi, x8 = G.tc_prepare_f8(G.nhwc(x).to(cuda))
    buf, y = guarded((B, H, W, Cout), torch.float32, cuda)
    part = None
    if gn:
        rows = G.tc_gn_rows(B, H, W, Cin, Cout)
        assert rows == 4 * math.ceil(W / 8) * math.ceil(H / 16)
        pbuf, part = guarded((B, rows, 32, 2), torch.float32, cuda)
    G.tc_igemm(hi, x8, G.tc_pack_f8(w.to(cuda)), b.to(cuda), Cout, 3, res1=None if r is None else G.nhwc(r).to(cuda),
               y=y, gn_partial=part, f8=1)
    assert_canaries(buf, "y")
    e = rel_err(y, want)
    print(f"column schedule {B}x{H}x{W} {Cin}->{Cout} res={res} gn={gn}: rel err {e:.2e}")
    assert e <= 1.5e-4

    if gn:
        assert_canaries(pbuf, "partials")
        # row (b, tile ty * tiles_x + tx, quarter q): image rows 16 ty + 4 q ... + 3, columns 8 tx ... + 7, per group
        cpg = Cout // 32
        tx_n, ty_n = math.ceil(W / 8), math.ceil(H / 16)
        yp = torch.zeros(B, ty_n * 16, tx_n * 8, Cout, dtype=torch.float64)
        yp[:, :H, :W] = y.double().cpu()
        blocks = yp.view(B, ty_n, 4, 4, tx_n, 8, 32, cpg).permute(0, 1, 4, 2, 6, 3, 5, 7).reshape(B, ty_n * tx_n * 4, 32, -1)
        s, ss = blocks.sum(-1), (blocks * blocks).sum(-1)
        got = part.double().cpu()
        mag = blocks.abs().sum(-1)
        assert ((got[..., 0] - s).abs() <= 1e-5 * mag + 1e-6).all(), "sum partials of the 8 x 4 quarters"
        assert ((got[..., 1] - ss).abs() <= 1e-5 * ss + 1e-6).all(), "sum of squares partials of the 8 x 4 quarters"
