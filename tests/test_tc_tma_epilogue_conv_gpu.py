"""The TMA epilogue of the F8 column-schedule 3x3 convs (tc_igemm_kernel's TMAE with COLS): the cooperative BN-128 convs
behind the VQ write each finished tile into shared memory and store it by TMA over the NHWC output, with the residual
tile loaded by TMA and the GroupNorm partials computed from the same values.  Only how the bytes travel changes, so
every output and every GroupNorm partial row must equal the register epilogue's byte for byte.  plan_tiles takes the TMA
epilogue only when the output and the residual are 16-byte aligned, so each case runs twice: on aligned buffers (TMA
epilogue) and with the output and residual placed 8 bytes past a 16-byte boundary (register epilogue).  The res2 cases
take the register epilogue both times; they check that it still agrees with itself across the alignments and with fp64.

Covered: 128->128 and 256->256 without a residual (with GroupNorm partials), with an in-place residual (y == res1, with
partials) and with an in-place residual plus res2 (no partials), on 16x16 maps at batch 3, 48x32, a 12x16 map at batch 2
(the tiles' last four rows lie outside the image) and 256x256 at batch 1 (512 or 1024 tiles, more than one per SM, so the
next tile's residual loads under the k-loop).  Every output lies inside a sentinel-filled guard allocation whose bytes
outside the output must survive, every GroupNorm partial row must be written, and the aligned run is checked against
fp64 with tests/test_gemm_matrix_gpu.py's F8 bar."""
import pytest
import torch

from tests import gpu_util as G

pytestmark = pytest.mark.gpu

GUARD = 4096                        # guard elements on each side of an output (16-byte multiples: TMA alignment)
SENT32 = 0x7FC0DEAD                 # a NaN pattern no kernel writes
EPILOGUES = {"tma": 0, "register": 8}  # bytes the output and residual sit past a 16-byte boundary
MAPS = {"16x16-b3": (3, 16, 16), "48x32-b1": (1, 48, 32), "12x16-b2": (2, 12, 16), "256x256-b1": (1, 256, 256)}
KINDS = ("gn", "inplace-gn", "inplace-res2")


def cases():
    """name -> (B, H, W, C, kind); Cin = Cout = C"""
    return {f"{c}-{kind}-{m}": (*MAPS[m], c, kind) for c in (128, 256) for kind in KINDS for m in MAPS}


def data(name, c):
    B, H, W, C, kind = c
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = torch.randn(B, H, W, C, generator=g)
    w = torch.randn(C, C, 3, 3, generator=g) * 0.03
    b = torch.randn(C, generator=g)
    r = torch.randn(B, H, W, C, generator=g) if kind.startswith("inplace") else None
    r2 = torch.randn(B, H, W, C, generator=g) if kind.endswith("res2") else None
    return x, w, b, r, r2


def start(shift):
    return GUARD + shift // 4


def guarded(n, shift, cuda):
    """(whole guard allocation, the n-element fp32 output inside it)"""
    buf = torch.full((n + 2 * GUARD,), SENT32, dtype=torch.int32, device=cuda).view(torch.float32)
    return buf, buf[start(shift):start(shift) + n]


def run(name, c, shift, cuda):
    """The launch with its output and residual `shift` bytes past a 16-byte boundary: outputs, GroupNorm partial rows and
    guard checks on the CPU."""
    B, H, W, C, kind = c
    x, w, b, r, r2 = data(name, c)
    hi, x8 = G.tc_prepare_f8(x.to(cuda))
    blob = G.tc_pack_f8(w.to(cuda))
    n = B * H * W * C
    shape = (B, H, W, C)
    ybuf, yv = guarded(n, shift, cuda)
    y = yv.view(shape)
    r1 = None
    if r is not None:
        y.copy_(r.to(cuda))
        r1 = y
    res2 = None
    if r2 is not None:
        r2buf, r2v = guarded(n, shift, cuda)
        res2 = r2v.view(shape)
        res2.copy_(r2.to(cuda))
    part = None
    if kind.endswith("gn"):
        part = torch.full((B * G.tc_gn_rows(B, H, W, C, C) * 64,), SENT32, dtype=torch.int32, device=cuda).view(torch.float32)
    G.tc_igemm(hi, x8, blob, b.to(cuda), C, 3, res1=r1, res2=res2, y=y, gn_partial=part, f8=1)
    torch.cuda.synchronize()
    ints = ybuf.view(torch.int32)
    off = start(shift)
    guard_ok = {"y": bool((ints[:off] == SENT32).all() and (ints[off + n:] == SENT32).all())}
    if res2 is not None:
        r2ints = r2buf.view(torch.int32)
        guard_ok["res2"] = bool((r2ints[:off] == SENT32).all() and (r2ints[off + n:] == SENT32).all()) and \
            torch.equal(res2.cpu(), r2)
    out = {"y": y.cpu()}
    if part is not None:
        out["gn_partial"] = part.cpu()
    return {"out": out, "guard_ok": guard_ok}


@pytest.fixture(scope="module")
def runs(cuda):
    """{name: {epilogue: results}}"""
    return {name: {e: run(name, c, shift, cuda) for e, shift in EPILOGUES.items()} for name, c in cases().items()}


def same_bytes(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.view(torch.int32), b.view(torch.int32))


NAMES = list(cases())


@pytest.mark.parametrize("name", NAMES)
def test_tc_tma_epilogue_conv_equals_register_epilogue(runs, name):
    tma, reg = runs[name]["tma"]["out"], runs[name]["register"]["out"]
    assert tma.keys() == reg.keys()
    for key in tma:
        assert same_bytes(tma[key], reg[key]), f"{name} {key}: {int((tma[key] != reg[key]).sum())} elements differ"


@pytest.mark.parametrize("epilogue", list(EPILOGUES))
@pytest.mark.parametrize("name", NAMES)
def test_tc_tma_epilogue_conv_writes_only_the_output(runs, name, epilogue):
    bad = [k for k, ok in runs[name][epilogue]["guard_ok"].items() if not ok]
    assert not bad, f"{name}: bytes outside the output changed in {bad}"


@pytest.mark.parametrize("epilogue", list(EPILOGUES))
@pytest.mark.parametrize("name", [n for n in NAMES if "gn" in n])
def test_tc_tma_epilogue_conv_writes_every_gn_partial_row(runs, name, epilogue):
    part = runs[name][epilogue]["out"]["gn_partial"]
    unwritten = int((part.view(torch.int32) == SENT32).sum())
    assert unwritten == 0, f"{name}: {unwritten} GroupNorm partial values not written"


@pytest.mark.parametrize("name", NAMES)
def test_tc_tma_epilogue_conv_against_fp64(runs, name, cuda):
    B, H, W, C, kind = cases()[name]
    x, w, b, r, r2 = data(name, cases()[name])
    want = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).to(cuda, torch.float64), w.to(cuda, torch.float64),
                                      b.to(cuda, torch.float64), padding=1).permute(0, 2, 3, 1)
    for extra in (r, r2):
        if extra is not None:
            want = want + extra.to(cuda, torch.float64)
    y = runs[name]["tma"]["out"]["y"].to(cuda, torch.float64)
    e = ((y - want).abs().max() / want.abs().max()).item()
    print(f"{name}: rel err {e:.2e}")
    assert e <= 1.5e-4                                 # test_gemm_matrix_gpu.tc_bar: F8 cross terms
