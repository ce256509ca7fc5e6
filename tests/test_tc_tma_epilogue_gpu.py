"""The TMA epilogue of the tensor-core implicit GEMM (tc_igemm_kernel's TMAE): the cooperative BN-128 linears write each
finished tile into shared memory and store it by TMA, with the residual tile loaded by TMA.  Only how the bytes travel
changes, not the rule per element, so every output must equal the register epilogue's byte for byte.  plan_tiles takes
the TMA epilogue only when the outputs and the residual are 16-byte aligned (the tensor maps' global addresses), so each
case runs twice: on aligned buffers (TMA epilogue) and with the outputs and a separate residual placed 8 bytes past a
16-byte boundary (register epilogue; 8 rather than 4 because that epilogue stores float2).

Covered: qkv (fp32 out), proj with a separate and with an aliased residual (y == res1), fc1 (GELU, split fp16 out), fc2
(K-sliced, aliased residual) and a ReLU 1x1, on 64x64, 24x40 and 7x9 maps at batch 1-3 and on a 4000-token row, so
that tiles cross image boundaries and the last tile is ragged.  Every output lies inside a sentinel-filled guard
allocation whose bytes outside the output must survive.  The outputs are checked against fp64 with
tests/test_gemm_matrix_gpu.py's bars."""
import pytest
import torch

from tests import gpu_util as G

pytestmark = pytest.mark.gpu

RELU, GELU = 2, 1
GUARD = 4096                        # guard elements on each side of an output (16-byte multiples: TMA alignment)
SENT32, SENT16 = 0x7FC0DEAD, 0x7E5A  # NaN patterns no kernel writes
EPILOGUES = {"tma": 0, "register": 8}  # bytes the outputs and a separate residual sit past a 16-byte boundary


def cases():
    """name -> (B, H, W, Cin, Cout, act, res: None | 'sep' | 'alias', split, slice_kb)"""
    return {
        "qkv-64x64-b2": (2, 64, 64, 256, 768, 0, None, False, 0),
        "qkv-4000-tokens": (1, 1, 4000, 256, 768, 0, None, False, 0),
        "proj-res-24x40-b3": (3, 24, 40, 256, 256, 0, "sep", False, 0),
        "proj-res-alias-7x9-b2": (2, 7, 9, 256, 256, 0, "alias", False, 0),
        "proj-res-alias-64x64-b1": (1, 64, 64, 256, 256, 0, "alias", False, 0),
        "fc1-gelu-split-24x40-b2": (2, 24, 40, 256, 1024, GELU, None, True, 0),
        "fc1-gelu-split-4000-tokens": (1, 1, 4000, 256, 1024, GELU, None, True, 0),
        "fc2-sliced-res-alias-64x64-b2": (2, 64, 64, 1024, 256, 0, "alias", False, 4),
        "fc2-sliced-res-alias-4000-tokens": (1, 1, 4000, 1024, 256, 0, "alias", False, 4),
        "relu-256to128-7x9-b3": (3, 7, 9, 256, 128, RELU, None, False, 0),
    }


def data(name, c):
    B, H, W, Cin, Cout, act, res, split, slice_kb = c
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = torch.randn(B, Cin, H, W, generator=g)
    hi = x.half()
    x = hi.float() + (x - hi.float()).half().float()          # exactly what the split planes hold
    w = torch.randn(Cout, Cin, 1, 1, generator=g) * 0.03
    b = torch.randn(Cout, generator=g)
    r = torch.randn(B, H, W, Cout, generator=g) if res else None
    return x, w, b, r


def start(dtype, shift):
    """index of the output in its guard allocation: GUARD elements plus `shift` bytes"""
    return GUARD + shift // dtype.itemsize


def guarded(n, dtype, sentinel, shift, cuda):
    """(whole guard allocation, the n-element output inside it)"""
    idt = torch.int32 if dtype == torch.float32 else torch.int16
    buf = torch.full((n + 2 * GUARD,), sentinel, dtype=idt, device=cuda).view(dtype)
    return buf, buf[start(dtype, shift):start(dtype, shift) + n]


def run(name, c, shift, cuda):
    """The launch with its outputs `shift` bytes past a 16-byte boundary: {outputs, guard_ok} on the CPU."""
    B, H, W, Cin, Cout, act, res, split, slice_kb = c
    x, w, b, r = data(name, c)
    hi, lo = G.tc_prepare(G.nhwc(x).to(cuda))
    blob = G.tc_pack(w.to(cuda))
    n = B * H * W * Cout
    shape = (B, H, W, Cout)
    bufs = {}
    r1 = y = planes = None
    if split:
        bufs["hi"], oh = guarded(n, torch.float16, SENT16, shift, cuda)
        bufs["lo"], ol = guarded(n, torch.float16, SENT16, shift, cuda)
        planes = (oh.view(shape), ol.view(shape))
    else:
        bufs["y"], yv = guarded(n, torch.float32, SENT32, shift, cuda)
        y = yv.view(shape)
    if res == "alias":
        y.copy_(r.to(cuda))
        r1 = y
    elif res == "sep":
        bufs["r"], rv = guarded(n, torch.float32, SENT32, shift, cuda)
        r1 = rv.view(shape)
        r1.copy_(r.to(cuda))
    G.tc_igemm(hi, lo, blob, b.to(cuda), Cout, 1, act=act, res1=r1, y=y, out_planes=planes, slice_kb=slice_kb)
    torch.cuda.synchronize()
    out = {"hi": planes[0].cpu(), "lo": planes[1].cpu()} if split else {"y": y.cpu()}
    guard_ok = {}
    for k, buf in bufs.items():
        off = start(buf.dtype, shift)
        ints = buf.view(torch.int32 if buf.dtype == torch.float32 else torch.int16)
        s = SENT32 if buf.dtype == torch.float32 else SENT16
        guard_ok[k] = bool((ints[:off] == s).all() and (ints[off + n:] == s).all())
    if res == "sep":
        guard_ok["r_unchanged"] = torch.equal(r1.cpu(), r)
    return {"out": out, "guard_ok": guard_ok}


@pytest.fixture(scope="module")
def runs(cuda):
    """{name: {epilogue: results}}"""
    return {name: {e: run(name, c, shift, cuda) for e, shift in EPILOGUES.items()} for name, c in cases().items()}


def same_bytes(a, b):
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.is_floating_point:
        it = {torch.float16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}[a.dtype]
        return torch.equal(a.view(it), b.view(it))
    return torch.equal(a, b)


NAMES = list(cases())


@pytest.mark.parametrize("name", NAMES)
def test_tc_tma_epilogue_equals_register_epilogue(runs, name):
    tma, reg = runs[name]["tma"]["out"], runs[name]["register"]["out"]
    assert tma.keys() == reg.keys()
    for key in tma:
        assert same_bytes(tma[key], reg[key]), f"{name} {key}: {int((tma[key] != reg[key]).sum())} elements differ"


@pytest.mark.parametrize("epilogue", list(EPILOGUES))
@pytest.mark.parametrize("name", NAMES)
def test_tc_tma_epilogue_writes_only_the_output(runs, name, epilogue):
    bad = [k for k, ok in runs[name][epilogue]["guard_ok"].items() if not ok]
    assert not bad, f"{name}: bytes outside the output changed in {bad}"


@pytest.mark.parametrize("name", NAMES)
def test_tc_tma_epilogue_against_fp64(runs, name):
    c = cases()[name]
    B, H, W, Cin, Cout, act, res, split, slice_kb = c
    got = runs[name]["tma"]["out"]
    y = got["y"] if "y" in got else got["hi"].float() + got["lo"].float()
    x, w, b, r = data(name, c)
    want = torch.einsum("bchw,oc->bhwo", x.double(), w[:, :, 0, 0].double()) + b.double()
    if act == GELU:
        want = torch.nn.functional.gelu(want)
    elif act == RELU:
        want = want.clamp_min(0)
    if r is not None:
        want = want + r.double()
    e = ((y.double() - want).abs().max() / want.abs().max()).item()
    print(f"{name}: rel err {e:.2e}")
    assert e <= 2e-5 + (1e-5 if act == GELU else 0.0)      # test_gemm_matrix_gpu.tc_bar: one pass, GELU
