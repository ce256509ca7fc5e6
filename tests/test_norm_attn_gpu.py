"""GPU: the kernels that feed every conv - GroupNorm statistics (femasr_gn_stats and the tensor-core epilogue partials +
femasr_gn_finalize_rows), GN + SiLU operand staging (femasr_tc_prepare exact / fast SiLU, femasr_tc_prepare_f8),
LayerNorm (femasr_ln_stats, femasr_tc_prepare LN) and window attention (femasr_window_attention, _mma) - against one
float64 ATen reference per operation, at the map sizes the engine launches for the configurations of
tests/test_engine_plan.py and at each kernel's edges, with offset-heavy inputs.

Each bar is a multiple of what ATen fp32 reaches on the same input (computed here and printed next to the kernel's error);
the multiples come from one measured H100 run with headroom (DESIGN.md section 6, "Normalisation and attention matrix").
A group or row "of mean/std R" holds R * s + a per-channel offset + noise of std s."""
import math

import pytest
import torch
import torch.nn.functional as F

from femasr_b200 import lib as L
from femasr_b200.spec import relative_position_index
from oracle import femasr_oracle as O
from tests import gpu_util as G
from tests.test_engine_plan import CONFIGS, DIV, SHAPES

pytestmark = pytest.mark.gpu

EPS_GN, EPS_LN = 1e-6, 1e-5
GN_CHUNK = 512                     # pixels per gn_partial_kernel block (norm.cu)


# ------------------------------------------------------------------------------------------------ engine shapes
def engine_maps():
    """(C, H, W, kind) of every GroupNorm map and (H, W) of every Swin map Ctx::forward / decode_loop launch for CONFIGS at
    SHAPES (engine.cu: down block i -> H / 2^(i+1) with chan(256 / scale / 2^(i+1)); up branches and decoder up_blocks ->
    2, 4, 8 x the latent).  kind "down" maps come from a stride-2 conv, "up" maps from an upsampled one."""
    chan = {8: 256, 16: 256, 32: 256, 64: 256, 128: 128, 256: 64, 512: 32}
    gn, swin = set(), set()
    for scale, _cbs, _sem, _tap in CONFIGS.values():
        d = {4: 1, 2: 2, 1: 3}[scale]
        m = 8 if scale == 1 else 8 * DIV[scale]         # check_geometry: the Swin map (LQ) or the input (HQ) in 8x8 windows
        for (B, H, W) in SHAPES:
            if B == 0 or H % m or W % m:
                continue
            for i in range(d):
                gn.add((chan[(256 // scale) >> (i + 1)], H >> (i + 1), W >> (i + 1), "down"))
            h, w = H >> d, W >> d
            if scale != 1:
                swin.add((h, w))
            for k, c in ((1, 256), (2, 128), (3, 64)):
                gn.add((c, h << k, w << k, "up"))
    return sorted(gn), sorted(swin)


GN_ENGINE, SWIN_ENGINE = engine_maps()
# edges of gn_partial_kernel / gn_finalize_kernel: HW below, at and above GN_CHUNK, odd sizes, > 32 chunks (lane loop wraps)
GN_EDGES = [(7, 73), (16, 32), (27, 19), (5, 7), (37, 29), (120, 160)]
assert [h * w for h, w in GN_EDGES[:3]] == [511, 512, 513] and 120 * 160 > 32 * GN_CHUNK
GN_CASES = ([pytest.param(c, h, w, k, 1, id=f"engine-{c}-{h}x{w}-{k}") for c, h, w, k in GN_ENGINE] +
            [pytest.param(c, h, w, "down", 3, id=f"edge-{c}-{h}x{w}-b3") for h, w in GN_EDGES for c in (64, 128, 256)])

KINDS = ("centred", "r3", "r10", "r30", "r100", "constant", "outlier")
RATIO = {"r3": 3, "r10": 10, "r30": 30, "r100": 100}


def rnd(g, *shape):
    return torch.randn(*shape, generator=g)


def kinds_tensor(g, B, C, H, W):
    """[B, C, H, W] fp32; group j is of kind KINDS[j % 7] in every image."""
    cpg = C // 32
    x = torch.empty(B, C, H, W)
    for j in range(32):
        k = KINDS[j % len(KINDS)]
        sl = slice(j * cpg, (j + 1) * cpg)
        s = 1.5
        if k == "centred":
            x[:, sl] = 2.0 * rnd(g, B, cpg, H, W)
        elif k in RATIO:
            off = (torch.rand(B, cpg, 1, 1, generator=g) - 0.5) * s
            x[:, sl] = RATIO[k] * s + off + s * rnd(g, B, cpg, H, W)
        elif k == "constant":
            x[:, sl] = 0.7 + 0.1 * j
        else:                   # one 1e4 outlier per image, away from the group's first element
            v = rnd(g, B, cpg, H, W)
            i = 1 + int(torch.randint(cpg * H * W - 1, (1,), generator=g))
            v.view(B, -1)[:, i] = 1e4
            x[:, sl] = v
    return x


def group_stats64(x):
    """fp64 per-(image, group) mean and rstd of [B, C, H, W]."""
    B = x.shape[0]
    v = x.double().reshape(B, 32, -1)
    return v.mean(-1), 1.0 / torch.sqrt(v.var(-1, unbiased=False) + EPS_GN)


def per_kind(err_bg):
    """{kind: largest value} of a [B, 32] error table."""
    return {k: err_bg[:, [j for j in range(32) if KINDS[j % 7] == k]].max().item() for k in KINDS}


def gn_errors(x, sc, sh, gamma, beta):
    """Per-kind (output error, rstd relative error) of the tables, next to ATen fp32's on the same x.  The output error of
    a group is max |x * scale + shift - group_norm64(x)| over its elements; the fold is evaluated in fp64 so that only the
    tables are measured."""
    B, C = x.shape[:2]
    cpg = C // 32
    want = F.group_norm(x.double(), 32, gamma.double(), beta.double(), EPS_GN)
    got = x.double() * sc.double()[:, :, None, None] + sh.double()[:, :, None, None]
    ref32 = F.group_norm(x, 32, gamma, beta, EPS_GN).double()
    red = lambda e: e.reshape(B, 32, -1).max(-1).values
    _, r64 = group_stats64(x)
    r_got = (sc.double() / gamma.double()).view(B, 32, cpg)[..., 0]
    _, _, r32 = torch.ops.aten.native_group_norm(x, gamma, beta, B, C, x.shape[2] * x.shape[3], 32, EPS_GN)
    return (per_kind(red((got - want).abs())), per_kind(red((ref32 - want).abs())),
            per_kind((r_got - r64).abs() / r64), per_kind((r32.double().view(B, 32) - r64).abs() / r64))


# bars: {kind: (output, rstd)} as multiples of ATen fp32's error on the same groups, None = printed only; the floor keeps
# an exact ATen from demanding 0.  Measured maxima of the ratios on an H100 (DESIGN.md): gn_stats output / rstd 3.0 / 3.1,
# outlier groups 9.3 / 5.3 (the fp32 per-thread sums hold the 1e8 square next to O(1) ones); epilogue partials 14.3 / 45.1
# at mean/std 10, 63 / 234 at 30 and 115 / 708 at 100, and a constant group's rstd 0.26 off (var = fp32 rounding of the
# squares, against eps = 1e-6) although its output stays within 2.7x of ATen's.
GN_STATS_BAR = {k: (6.0, 6.0) for k in KINDS} | {"outlier": (16.0, 12.0)}
GN_EPI_BAR = {k: (25.0, 90.0) for k in ("centred", "r3", "r10", "outlier")} | {"constant": (6.0, None), "r30": None,
                                                                               "r100": None}
FLOOR = 1e-7
WORST = {}


def note(key, e, ref, what):
    if key not in WORST or e > WORST[key][0]:
        WORST[key] = (e, ref, what)


def check_gn(name, x, sc, sh, gamma, beta, bars, what):
    out, out32, rs, rs32 = gn_errors(x, sc, sh, gamma, beta)
    for k in KINDS:
        print(f"{name} {what} {k:8s}: output {out[k]:.2e} (ATen fp32 {out32[k]:.2e}), rstd {rs[k]:.2e} (ATen fp32 {rs32[k]:.2e})")
        note(f"{name} output {k}", out[k], out32[k], what)
        note(f"{name} rstd {k}", rs[k], rs32[k], what)
    for k, (bo, br) in ((k, v) for k, v in bars.items() if v is not None):
        assert out[k] <= bo * max(out32[k], FLOOR), f"{name} {what} {k}: output error {out[k]:.3e} vs ATen fp32 {out32[k]:.3e}"
        assert br is None or rs[k] <= br * max(rs32[k], FLOOR), f"{name} {what} {k}: rstd error {rs[k]:.3e} vs ATen fp32 {rs32[k]:.3e}"


def affine(g, C, cuda):
    gamma, beta = 1 + 0.2 * rnd(g, C), 0.2 * rnd(g, C)
    return gamma, beta, gamma.to(cuda), beta.to(cuda)


# ------------------------------------------------------------------------------------------------ GroupNorm statistics
@pytest.mark.parametrize("C_,H,W,kind,B", GN_CASES)
def test_gn_stats(cuda, C_, H, W, kind, B):
    """femasr_gn_stats on every kind of group, and image b of a batch == the image alone, bit for bit."""
    g = torch.Generator().manual_seed(C_ * 7919 + H * 31 + W)
    x = kinds_tensor(g, B, C_, H, W)
    gamma, beta, gd, bd = affine(g, C_, cuda)
    xg = G.nhwc(x).to(cuda)
    sc, sh = G.gn_tables(xg, gd, bd)
    check_gn("gn_stats", x, sc.cpu(), sh.cpu(), gamma, beta, GN_STATS_BAR, f"C {C_} {B}x{H}x{W}")
    for b in range(B) if B > 1 else ():
        s1, h1 = G.gn_tables(xg[b:b + 1].contiguous(), gd, bd)
        assert torch.equal(s1, sc[b:b + 1]) and torch.equal(h1, sh[b:b + 1]), f"image {b} of {B} differs from the image alone"


def epilogue_data(g, xk, up, cuda):
    """A 3x3 conv (upsampled for up) from 64 channels whose stored output is conv(N(0,1)) + bias + res1 with res1 = xk, so
    every group of the output has the kind of the same group of xk; the constant groups get zero weights and bias."""
    B, C, Ho, Wo = xk.shape
    H, W = (Ho // 2, Wo // 2) if up else (Ho, Wo)
    w, b = 0.02 * rnd(g, C, 64, 3, 3), 0.3 * rnd(g, C)
    cpg = C // 32
    for j in range(32):
        if KINDS[j % 7] == "constant":
            w[j * cpg:(j + 1) * cpg] = 0
            b[j * cpg:(j + 1) * cpg] = 0
    blob = G.tc_pack_up2(w.to(cuda)) if up else G.tc_pack(w.to(cuda))
    return dict(x=rnd(g, B, H, W, 64).to(cuda), blob=blob, b=b.to(cuda), res=G.nhwc(xk).to(cuda), H=H, W=W, C=C, up=up,
                Ho=Ho, Wo=Wo)


def epilogue_run(d, b0, b1):
    """femasr_tc_igemm with GroupNorm partials on images [b0, b1) into NaN-filled outputs: (y, partial rows)."""
    n, C, dev = b1 - b0, d["C"], d["x"].device
    hi, lo = G.tc_prepare(d["x"][b0:b1])
    rows = G.tc_gn_rows(n, d["H"], d["W"], 64, C, upsample=d["up"])
    part = torch.full((n, rows, 32, 2), float("nan"), device=dev)
    y = torch.full((n, d["Ho"], d["Wo"], C), float("nan"), device=dev)
    G.tc_igemm(hi, lo, d["blob"], d["b"], C, 3, res1=d["res"][b0:b1], upsample=d["up"], gn_partial=part, y=y)
    assert not torch.isnan(part).any() and not torch.isnan(y).any(), "not every output or partial row was written"
    return y, part


@pytest.mark.parametrize("C_,H,W,kind,B", GN_CASES)
def test_gn_epilogue_partials(cuda, C_, H, W, kind, B):
    """The tensor-core conv epilogue's fp32 (sum, sumsq) rows + femasr_gn_finalize_rows against fp64 GroupNorm of the
    stored output: pinned up to mean/std 10, printed at 30 and 100.  Maps an upsampled conv produces run as one (Cout 64 is
    two channels per group); the rows of image b of a batch == the image alone, bit for bit."""
    up = int(kind == "up")
    g = torch.Generator().manual_seed(C_ * 104729 + H * 37 + W)
    xk = kinds_tensor(g, B, C_, H, W)
    gamma, beta, gd, bd = affine(g, C_, cuda)
    d = epilogue_data(g, xk, up, cuda)
    y, part = epilogue_run(d, 0, B)
    sc, sh = torch.empty(B, C_, device=cuda), torch.empty(B, C_, device=cuda)
    L.check(L.load().femasr_gn_finalize_rows(G.p(part), G.p(gd), G.p(bd), G.p(sc), G.p(sh), B, part.shape[1], H * W, C_,
                                             EPS_GN, G.S()))
    what = f"C {C_} {B}x{H}x{W}{' up' if up else ''}"
    check_gn("epilogue", G.nchw(y).cpu(), sc.cpu(), sh.cpu(), gamma, beta, GN_EPI_BAR, what)
    for b in range(B) if B > 1 else ():
        y1, p1 = epilogue_run(d, b, b + 1)
        assert torch.equal(y1, y[b:b + 1]) and torch.equal(p1, part[b:b + 1]), f"image {b} of {B} differs from the image alone"


# ------------------------------------------------------------------------------------------------ GN + SiLU staging
STAGE_CASES = [(1, 32, 32, 256), (1, 64, 64, 128), (1, 128, 128, 64), (3, 13, 37, 256), (3, 5, 7, 64), (3, 27, 19, 128)]
FAST_SILU_REL = 4e-7               # include/femasr_b200.h: the fast SiLU's relative error bound


def tables64(x, gamma, beta, cuda):
    """The scale/shift tables computed in fp64 from fp64 statistics, rounded once to fp32."""
    B, C = x.shape[:2]
    mean, rstd = group_stats64(x)
    sc = rstd.repeat_interleave(C // 32, 1) * gamma.double()
    sh = beta.double() - sc * mean.repeat_interleave(C // 32, 1)
    return sc.float().to(cuda), sh.float().to(cuda)


# x ATen fp32's max-abs error of silu(group_norm(x)); measured: 1.0 on femasr_gn_stats' tables, 6.8 (exact) / 1.5 (fast) on
# fp64 tables, where ATen's own statistics error is the yardstick and the kernel has none
STAGE_BAR = {"exact": 12.0, "fast": 12.0}


@pytest.mark.parametrize("tables", ["gn_stats", "fp64"])
@pytest.mark.parametrize("B,H,W,C_", STAGE_CASES, ids=[f"{b}x{h}x{w}x{c}" for b, h, w, c in STAGE_CASES])
def test_gn_silu_staging(cuda, B, H, W, C_, tables):
    """femasr_tc_prepare (exact and fast SiLU) and femasr_tc_prepare_f8: hi + lo against fp64 silu(group_norm(x)); the F8
    hi plane bit-equal to femasr_tc_prepare's in the same mode; the e4m3 plane decodes to the staged value."""
    g = torch.Generator().manual_seed(B * 1000 + H * 10 + C_)
    x = kinds_tensor(g, B, C_, H, W)
    gamma, beta, gd, bd = affine(g, C_, cuda)
    xg = G.nhwc(x).to(cuda)
    sc, sh = G.gn_tables(xg, gd, bd) if tables == "gn_stats" else tables64(x, gamma, beta, cuda)
    want = G.nhwc(F.silu(F.group_norm(x.double(), 32, gamma.double(), beta.double(), EPS_GN)))
    ref32 = (G.nhwc(F.silu(F.group_norm(x, 32, gamma, beta, EPS_GN))).double() - want).abs().max().item()
    for mode, form in ((L.PRO_GN_SILU, "exact"), (L.PRO_GN_SILU_FAST, "fast")):
        hi, lo = G.tc_prepare(xg, mode, sc, sh)
        got = hi.double().cpu() + lo.double().cpu()
        e = (got - want).abs().max().item()
        what = f"{form} SiLU, {tables} tables, {B}x{H}x{W}x{C_}"
        print(f"staging {what}: max-abs {e:.2e} (ATen fp32 {ref32:.2e})")
        note(f"staging {form} {tables}", e, ref32, what)
        assert e <= STAGE_BAR[form] * max(ref32, FLOOR), f"staging {what}: max-abs {e:.3e} vs ATen fp32 {ref32:.3e}"
        hi8, x8 = G.tc_prepare_f8(xg, mode, sc, sh)
        assert torch.equal(hi8, hi), f"F8 staging {what}: hi plane differs from femasr_tc_prepare's"
        v = (hi.float() + lo.float()).cpu()          # the staged fp32 value to 2^-22 relative
        lo8, val8 = f8_decode(x8.cpu(), C_)
        e4 = lambda t: (t.abs() * 2.0 ** -3 + 2.0 ** -9)                 # e4m3 rounding: half of 2^-3 relative, subnormals
        assert ((val8 - v * 0.25).abs() <= e4(v * 0.25)).all(), f"F8 staging {what}: value part"
        d = (v - hi.float().cpu()) * 1024.0
        assert ((lo8 - d).abs() <= e4(d)).all(), f"F8 staging {what}: lo part"


def f8_decode(x8, C):
    """The F8 plane [B,H,W,C] (2 bytes per channel) -> (lo part, value part) as fp32 [B,H,W,C]: per pixel and 64-channel
    chunk 128 bytes, e4m3((v - hi) * 2^10) of the chunk's channels at (c / 64) * 128 + c % 64, e4m3(v * 2^-2) at + 64."""
    b = x8.view(torch.uint8).view(*x8.shape[:3], C // 64, 2, 64)
    dec = lambda t: t.contiguous().view(torch.float8_e4m3fn).float().reshape(*x8.shape[:3], C)
    return dec(b[..., 0, :]), dec(b[..., 1, :])


def f8_bytes(x, C):
    """CPU emulation of femasr_tc_prepare_f8 in mode NONE: the expected bytes of the F8 plane of fp32 NHWC x."""
    a = x.clamp(-65504.0, 65504.0)
    hi = a.half().float()
    q = lambda t: t.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).view(torch.uint8)
    lo8, val8 = q((a - hi) * 1024.0), q(a * 0.25)
    out = torch.stack([lo8.view(*x.shape[:3], C // 64, 64), val8.view(*x.shape[:3], C // 64, 64)], -2)
    return out.reshape(*x.shape[:3], 2 * C)


@pytest.mark.parametrize("C_", [64, 256, 512])
def test_f8_plane_bytes(cuda, C_):
    """femasr_tc_prepare_f8 (mode NONE) byte-exact against a torch.float8_e4m3fn emulation, over magnitudes from e4m3
    subnormals to fp16 saturation: both parts saturate at +-448, the hi plane at +-65504."""
    B, H, W = 2, 7, 9
    g = torch.Generator().manual_seed(C_)
    mag = torch.exp(torch.empty(B, H, W, C_).uniform_(math.log(1e-4), math.log(2e5), generator=g))
    x = (mag * torch.sign(rnd(g, B, H, W, C_))).float()
    x[0, 0, 0, :4] = torch.tensor([1792.0, 2047.0, 65504.0, -1e6])
    hi, x8 = G.tc_prepare_f8(x.to(cuda))
    assert torch.equal(hi.cpu(), x.clamp(-65504.0, 65504.0).half()), "F8 hi plane"
    got = x8.cpu().view(torch.uint8).view(B, H, W, 2 * C_)
    want = f8_bytes(x, C_)
    bad = int((got != want).sum())
    assert bad == 0, f"{bad} of {want.numel()} F8 bytes differ from the emulation"
    lo8, val8 = f8_decode(x8.cpu(), C_)
    assert (val8.abs() == 448).any() and (lo8.abs() == 448).any(), "the input should saturate both parts somewhere"


# ------------------------------------------------------------------------------------------------ LayerNorm
LN_KINDS = KINDS
LN_M = sorted({b * h * w for (h, w) in SWIN_ENGINE for b in (1, 3)}) + [17, 33, 1023, 4097]
LN_BAR = (4.0, 4.0, 4.0)           # x ATen fp32: mean (in std units), rstd (relative), staged output (max-abs); measured 1.6 / 1.1 / 1.6


def ln_rows(g, M):
    """[M, 256]; row r is of kind LN_KINDS[r % 7]."""
    x = torch.empty(M, 256)
    off = (torch.rand(256, generator=g) - 0.5) * 1.5
    for r, k in enumerate(LN_KINDS):
        n = len(range(r, M, 7))
        if k == "centred":
            v = 2.0 * rnd(g, n, 256)
        elif k in RATIO:
            v = RATIO[k] * 1.5 + off + 1.5 * rnd(g, n, 256)
        elif k == "constant":
            v = torch.full((n, 256), 0.3)
        else:
            v = rnd(g, n, 256)
            v[torch.arange(n), torch.randint(256, (n,), generator=g)] = 1e4
        x[r::7] = v
    return x


def ln_kind_max(e):
    return {k: e[r::7].max().item() if e[r::7].numel() else 0.0 for r, k in enumerate(LN_KINDS)}


@pytest.mark.parametrize("M", LN_M)
def test_layernorm(cuda, M):
    """femasr_ln_stats (mean, rstd) and femasr_tc_prepare(FEMASR_PRO_LN) (hi + lo) against fp64 F.layer_norm, per row kind;
    M odd and M = 1 mod 16 leave the staging kernel's last warp with one row."""
    g = torch.Generator().manual_seed(M)
    x = ln_rows(g, M)
    gamma, beta = 1 + 0.2 * rnd(g, 256), 0.2 * rnd(g, 256)
    xd = x.double()
    m64, r64 = xd.mean(1), 1.0 / torch.sqrt(xd.var(1, unbiased=False) + EPS_LN)
    _, m32, r32 = torch.ops.aten.native_layer_norm(x, [256], None, None, EPS_LN)
    mu, rs = G.ln_stats(x.to(cuda), EPS_LN)
    want = F.layer_norm(xd, (256,), gamma.double(), beta.double(), EPS_LN)
    ref32 = (F.layer_norm(x, (256,), gamma, beta, EPS_LN).double() - want).abs().max(1).values
    hi = torch.full((M, 256), float("nan"), dtype=torch.float16, device=cuda)
    lo = torch.full_like(hi, float("nan"))
    xg, gd, bd = x.to(cuda), gamma.to(cuda), beta.to(cuda)
    L.check(L.load().femasr_tc_prepare(G.p(xg), G.p(hi), G.p(lo), L.PRO_LN, None, None, G.p(gd), G.p(bd), 1, 1, M, 256, 0,
                                       EPS_LN, G.S()))
    assert not torch.isnan(hi).any() and not torch.isnan(lo).any(), "LN staging: not every row was written"
    got = hi.double().cpu() + lo.double().cpu()
    errs = {
        "mean": (ln_kind_max((mu.cpu().double() - m64).abs() * r64), ln_kind_max((m32.view(-1).double() - m64).abs() * r64)),
        "rstd": (ln_kind_max((rs.cpu().double() - r64).abs() / r64), ln_kind_max((r32.view(-1).double() - r64).abs() / r64)),
        "staged": (ln_kind_max((got - want).abs().max(1).values), ln_kind_max(ref32)),
    }
    for i, (name, (e, e32)) in enumerate(errs.items()):
        for k in LN_KINDS:
            print(f"layernorm M {M} {name} {k:8s}: {e[k]:.2e} (ATen fp32 {e32[k]:.2e})")
            note(f"layernorm {name} {k}", e[k], e32[k], f"M {M}")
            assert e[k] <= LN_BAR[i] * max(e32[k], FLOOR), f"layernorm M {M} {name} {k}: {e[k]:.3e} vs ATen fp32 {e32[k]:.3e}"


# ------------------------------------------------------------------------------------------------ window attention
from tests.test_gemm_matrix_gpu import assert_canaries, guarded  # noqa: E402


def attention_ref(qkv, table, B, H, W, shift, dtype):
    """network_swinir.py WindowAttention + SwinTransformerBlock's roll / partition / mask, in `dtype`: [B, H*W, 256]."""
    t = qkv.to(dtype).view(B, H, W, 768)
    if shift:
        t = torch.roll(t, (-shift, -shift), (1, 2))
    q, k, v = O.window_partition(t, 8).reshape(-1, 64, 3, 8, 32).permute(2, 0, 3, 1, 4)
    attn = (q * 32 ** -0.5) @ k.transpose(-2, -1)
    attn = attn + table.to(dtype)[relative_position_index().view(-1)].view(64, 64, 8).permute(2, 0, 1).unsqueeze(0)
    if shift:
        mask = O.shift_mask(H, W, 8, shift, dtype)
        nW = mask.shape[0]
        attn = (attn.view(-1, nW, 8, 64, 64) + mask[None, :, None]).view(-1, 8, 64, 64)
    o = O.window_reverse((attn.softmax(-1) @ v).transpose(1, 2).reshape(-1, 64, 256), 8, H, W)
    if shift:
        o = torch.roll(o, (shift, shift), (1, 2))
    return o.reshape(B, H * W, 256)


# the engine's Swin maps at B = 1, a ragged batch, a one-window-high map (still shifted and masked), W = 8, non-square
ATTN_MAPS = [(1, h, w) for h, w in SWIN_ENGINE] + [(3, 24, 40), (2, 8, 64), (1, 40, 8), (3, 16, 8)]
ATTN_INPUTS = [(1.0, 0.5), (4.0, 0.5), (12.0, 0.5), (4.0, 20.0)]         # (qkv scale, rel-pos table std)
ATTN_CASES = [pytest.param(B, H, W, s, qs, ts, id=f"{B}x{H}x{W}-shift{s}-q{qs:g}-t{ts:g}")
              for B, H, W in ATTN_MAPS for s in (0, 4) for qs, ts in ATTN_INPUTS]
ATTN_BAR = {"simt": 4.0, "mma": 4.0}        # x ATen fp32's max-abs error over max |out|; measured 1.6 / 2.3


def attention_run(lib, kind, qkv, bias, B, H, W, shift, planes=False):
    """One launch into NaN-filled guarded outputs: fp32 out, or the mma kernel's (hi, lo) planes."""
    dev = qkv.device
    if planes:
        bh, oh = guarded((B, H * W, 256), torch.float16, dev)
        bl, ol = guarded((B, H * W, 256), torch.float16, dev)
        L.check(lib.femasr_window_attention_mma(G.p(qkv), G.p(bias), None, G.p(oh), G.p(ol), B, H, W, 256, 8, shift, G.S()))
        assert_canaries(bh, "attention hi plane")
        assert_canaries(bl, "attention lo plane")
        return oh, ol
    buf, out = guarded((B, H * W, 256), torch.float32, dev)
    if kind == "simt":
        L.check(lib.femasr_window_attention(G.p(qkv), G.p(bias), G.p(out), B, H, W, 256, 8, shift, G.S()))
    else:
        L.check(lib.femasr_window_attention_mma(G.p(qkv), G.p(bias), G.p(out), None, None, B, H, W, 256, 8, shift, G.S()))
    assert_canaries(buf, f"attention {kind}")
    return out


@pytest.mark.parametrize("B,H,W,shift,qs,ts", ATTN_CASES)
def test_window_attention(cuda, B, H, W, shift, qs, ts):
    """Both window-attention kernels against fp64: peaked softmax (qkv x 12: logit gaps of the order of the -100 mask), large
    relative-position entries; the mma kernel's split planes == the split of its fp32 output; image b == the image alone."""
    lib = L.load()
    g = torch.Generator().manual_seed(B * 7 + H * 131 + W + shift + int(qs * 10 + ts))
    qkv = qs * rnd(g, B, H * W, 768)
    table = ts * rnd(g, 225, 8)
    want = attention_ref(qkv, table, B, H, W, shift, torch.float64)
    scale = want.abs().max().item()
    ref32 = (attention_ref(qkv, table, B, H, W, shift, torch.float32).double() - want).abs().max().item() / scale
    qg, tg = qkv.to(cuda), table.to(cuda)
    full = torch.empty(8, 64, 64, device=cuda)
    frag = torch.empty(8 * 64 * 64, device=cuda)
    L.check(lib.femasr_expand_rel_bias(G.p(tg), G.p(full), 8, G.S()))
    L.check(lib.femasr_expand_rel_bias_mma(G.p(tg), G.p(frag), 8, G.S()))
    what = f"{B}x{H}x{W} shift {shift} qkv x{qs:g} table std {ts:g}"
    outs = {}
    for kind, bias in (("simt", full), ("mma", frag)):
        out = attention_run(lib, kind, qg, bias, B, H, W, shift)
        e = (out.double().cpu() - want).abs().max().item() / scale
        print(f"attention {kind} {what}: rel max-abs {e:.2e} (ATen fp32 {ref32:.2e})")
        note(f"attention {kind}", e, ref32, what)
        assert e <= ATTN_BAR[kind] * max(ref32, FLOOR), f"attention {kind} {what}: {e:.3e} vs ATen fp32 {ref32:.3e}"
        outs[kind] = out
    oh, ol = attention_run(lib, "mma", qg, frag, B, H, W, shift, planes=True)
    y = outs["mma"]
    assert torch.equal(oh, y.half()) and torch.equal(ol, (y - oh.float()).half()), f"{what}: planes != split of the fp32 output"
    for b in range(B) if B > 1 else ():
        one = qg[b:b + 1]
        assert torch.equal(attention_run(lib, "simt", one, full, 1, H, W, shift), outs["simt"][b:b + 1]), f"simt image {b}"
        assert torch.equal(attention_run(lib, "mma", one, frag, 1, H, W, shift), y[b:b + 1]), f"mma image {b}"


def test_zz_largest_errors(cuda):
    """Runs last in this file: the largest error of every measured quantity next to ATen fp32's on that input."""
    for key, (e, ref, what) in sorted(WORST.items()):
        print(f"largest {key}: {e:.2e} (ATen fp32 {ref:.2e}, ratio {e / max(ref, FLOOR):.2f}) at {what}")
