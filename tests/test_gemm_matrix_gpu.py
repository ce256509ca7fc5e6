"""GPU: both implicit GEMMs (femasr_tc_igemm, femasr_igemm_simt) against fp64 ATen in the COMBINATIONS Ctx::conv
(femasr_b200/csrc/engine.cu) launches, at tile edges, plus exact invariants of the tensor-core kernel's persistent tile loop.

One table of conv classes (CLASSES), one runner (run_case), one reference (reference).  A class is what Ctx::conv composes:
kernel size, stride, fused upsample, prologue, activation, bias, residuals, output form, GroupNorm partials, operand form,
numerics and channels.  CLASSES holds every class Ctx::forward, decode_loop, swin, resblock, up_block, quantise
(before_quant), semantic_loss, vgg_stack, alex and disc emit on gemm_path 1 for the configurations of
tests/test_engine_plan.py (CONFIGS and HEADS); the numerics column follows Ctx::numerics.  The quantiser's z . E^T is not a
conv there: with the fused VQ (the default) it is femasr_vq_match_tc, which tests/test_vq_fused_gpu.py covers.

Every class runs at three spatial shapes chosen for the kernel's 128-pixel tiles (Wt x Ht, tc_tile_shape in tc_gemm.cu,
mirrored by tile_shape below): an exact fit, a ragged multi-tile batch of 2 with odd sizes, and wide rows with Wt = 128.
ACCEPTED is a second table: calls the engine never makes but the ABIs accept, each pinned as right or refused."""
import dataclasses
import math

import pytest
import torch
import torch.nn.functional as F

from femasr_b200 import lib as L
from tests import gpu_util as G

pytestmark = pytest.mark.gpu

NONE, GELU, RELU, LRELU = L.ACT_NONE, L.ACT_GELU, L.ACT_RELU, L.ACT_LRELU


@dataclasses.dataclass(frozen=True)
class Cls:
    name: str
    ch: tuple                 # ((Cin, Cout), ...): the channel pairs the engine launches this class with
    k: int = 3
    stride: int = 1
    up: int = 0
    pro: str = "none"         # none | gn (GroupNorm(32, 1e-6) + SiLU) | ln (LayerNorm(1e-5))
    act: int = NONE
    bias: bool = True
    res1: str = "none"        # none | sep (its own tensor) | alias (the output buffer)
    res2: bool = False
    out: str = "f32"          # f32 | split (fp16 hi/lo planes)
    gn: bool = False          # GroupNorm partials of the output
    operand: str = "staged"   # staged (femasr_tc_prepare / _f8 from fp32) | planes (a producer wrote split planes)
    num: str = "one"          # one (one pass) | slice (slice_kb 4) | f8 (F8 cross terms; GN + SiLU staged with the fast SiLU)
    kb: tuple = None          # ACCEPTED only: (kb_begin, kb_count)


R = dict(pro="gn", gn=True)                        # resblock conv.2
R5 = dict(pro="gn", res1="alias")                  # resblock conv.5
V = dict(act=RELU, operand="planes")               # VGG / AlexNet conv on a producer's planes
D = dict(act=LRELU, bias=False)                    # discriminator spectral-norm conv
CLASSES = [
    # forward: in_conv as a 1x1 GEMM over im2col rows (K = 48 -> 64), written as the down conv's operand planes
    Cls("in_conv", ((64, 256), (64, 128), (64, 64)), k=1, operand="planes", out="split"),
    # forward: down convs; block 0 reads in_conv's planes (x4 256->256, x2 128->256, HQ 64->128), later blocks stage fp32
    Cls("down_planes", ((64, 128), (128, 256), (256, 256)), stride=2, gn=True, operand="planes", num="slice"),
    Cls("down_staged", ((128, 256), (256, 256)), stride=2, gn=True, num="slice"),
    # resblock in front of the last quantiser (encoder; up branches and decoder levels of multi-scale nets)
    Cls("res2_precise", ((128, 128), (256, 256)), num="slice", **R),
    Cls("res5_precise_gn", ((128, 128), (256, 256)), num="slice", gn=True, **R5),
    Cls("res5_precise", ((128, 128), (256, 256)), num="slice", **R5),
    # resblock behind the last quantiser (decoder; up branches of single-codebook nets)
    Cls("res2_f8", ((256, 256), (128, 128), (64, 64)), num="f8", **R),
    Cls("res5_f8_gn", ((256, 256), (128, 128), (64, 64)), num="f8", gn=True, **R5),
    Cls("res5_f8", ((256, 256), (128, 128), (64, 64)), num="f8", **R5),
    # resblock, last of a decoder up_block in the LQ stage: the next level's skip add (decode_loop's `extra`) as res2
    Cls("res5_f8_skip", ((256, 256), (128, 128)), num="f8", res2=True, **R5),
    # up_block: nearest x2 + conv3x3 as four sub-pixel phases, with the first resblock's statistics
    Cls("up_precise", ((256, 256), (256, 128)), up=1, gn=True, num="slice"),
    Cls("up_f8", ((256, 256), (256, 128), (128, 64)), up=1, gn=True, num="f8"),
    # swin: qkv and fc1 stage LayerNorm; proj and fc2 read planes (attention output, fc1's split output)
    Cls("swin_qkv", ((256, 768),), k=1, pro="ln"),
    Cls("swin_proj", ((256, 256),), k=1, operand="planes", res1="sep"),
    Cls("swin_fc1", ((256, 1024),), k=1, pro="ln", act=GELU, out="split"),
    Cls("swin_fc2", ((1024, 256),), k=1, operand="planes", res1="alias", num="slice"),
    Cls("swin_conv", ((256, 256),), res1="alias", num="slice"),
    # quantise: before_quant on the encoder feature (256 channels) or on cat(feature, decoder stream) (512 / 256)
    Cls("before_quant", ((256, 256), (256, 512), (256, 128)), k=1),
    Cls("before_quant_cat", ((512, 128), (512, 256)), k=1, num="slice"),
    # decode_loop: after_quant; behind the last quantiser F8 (384 / 768: concatenated codebooks), else K-sliced
    Cls("after_quant_f8", ((256, 256), (512, 256), (384, 256), (384, 128), (768, 128)), num="f8"),
    Cls("after_quant_precise", ((256, 256), (512, 256), (768, 256)), num="slice"),
    # semantic_loss: conv_semantic
    Cls("conv_semantic", ((512, 512),), k=1, act=RELU),
    # vgg_stack (VGG19 to relu4_4, LPIPS' VGG16): conv 0 over im2col rows; fp32 output in front of a pool / at a tap
    Cls("vgg_conv0", ((64, 64),), k=1, out="split", **V),
    Cls("vgg_split", ((64, 128), (128, 256), (256, 256), (256, 512), (512, 512)), out="split", **V),
    Cls("vgg_f32", ((64, 64), (128, 128), (256, 256), (512, 512)), **V),
    # alex: conv1 over K = 363 -> 384 im2col rows, conv2 5x5 and conv3 on pooled planes, conv4 / conv5 stage fp32
    Cls("alex_conv1", ((384, 64),), k=1, **V),
    Cls("alex_conv2", ((64, 192),), k=5, **V),
    Cls("alex_conv3", ((192, 384),), **V),
    Cls("alex_conv45", ((384, 256), (256, 256)), act=RELU),
    # disc: conv0 over im2col rows (bias); conv1-3 4x4 stride 2; conv4-6 on bilinear planes, with / without the skip;
    # conv6 -> conv7 -> conv8 hand split planes on
    Cls("disc_conv0", ((64, 64),), k=1, act=LRELU, operand="planes"),
    Cls("disc_down", ((64, 128), (128, 256), (256, 512)), k=4, stride=2, num="slice", **D),
    Cls("disc_up_skip", ((512, 256), (256, 128)), operand="planes", res1="sep", num="slice", **D),
    Cls("disc_up", ((512, 256), (256, 128)), operand="planes", num="slice", **D),
    Cls("disc_conv6_skip", ((128, 64),), operand="planes", res1="sep", out="split", num="slice", **D),
    Cls("disc_conv6", ((128, 64),), operand="planes", out="split", num="slice", **D),
    Cls("disc_conv7", ((64, 64),), operand="planes", out="split", num="slice", **D),
    Cls("disc_conv8", ((64, 64),), operand="planes", num="slice", **D),
]

# Calls the engine never makes but the ABIs accept: (class, femasr_tc_igemm is right | refused).  femasr_igemm_simt must be
# right in every row it can express.
A = ((64, 64),)
ACCEPTED = [(Cls(f"act{act}_k{k}", A, k=k, stride=2 if k == 4 else 1, act=act), "right") for k in (1, 3, 4, 5)
            for act in (NONE, GELU, RELU, LRELU) if (k, act) != (5, LRELU)] + [
    # the 5x5 instantiations have no LeakyReLU epilogue: femasr_tc_igemm used to return the pre-activation values
    (Cls("act3_k5", A, k=5, act=LRELU), "refused"),
    (Cls("res2_alone", A, res2=True), "right"),
    (Cls("res5_f8_gn_skip", ((64, 64), (256, 256)), num="f8", gn=True, res2=True, **R5), "right"),
    (Cls("gn_split", ((128, 128),), gn=True, out="split"), "right"),
    (Cls("gn_stride2", ((64, 64), (128, 256)), stride=2, gn=True), "right"),
    (Cls("f8_k1", ((128, 128),), k=1, num="f8"), "right"),
    (Cls("f8_stride2", ((128, 128),), stride=2, num="f8"), "right"),
    (Cls("f8_slice", A, num="f8+slice"), "refused"),
    (Cls("f8_lrelu", A, act=LRELU, num="f8"), "refused"),
    # cpg = Cout / 32 = 6, 10, 12: the epilogue's shuffle reduction handles 2, 4, 8
    (Cls("gn_cout192", ((64, 192),), gn=True), "refused"),
    (Cls("gn_cout320", ((64, 320),), gn=True), "refused"),
    (Cls("gn_cout384", ((64, 384),), gn=True), "refused"),
    (Cls("gn_k1", A, k=1, gn=True), "refused"),
    (Cls("kb_range_sliced", ((128, 128),), num="slice", kb=(3, 11)), "right"),
    (Cls("kb_range", ((128, 128),), kb=(5, 6)), "right"),
    (Cls("up_k1", A, k=1, up=1), "refused"),
    (Cls("k4_stride1", A, k=4), "refused"),
    (Cls("k5_stride2", A, k=5, stride=2), "refused"),
]
SIMT_REFUSES = {"up_k1", "k4_stride1", "k5_stride2"}        # the rows femasr_igemm_simt refuses as well
# femasr_igemm_simt alone: its k-step is 16 channels, and Cin % 16 is all its argument check asks
SIMT_ONLY = [Cls("simt_cin48", ((48, 64),), res1="sep"), Cls("simt_cin80", ((80, 128),), k=1, act=GELU)]


# ------------------------------------------------------------------------------------------------ shapes
def tile_shape(H, W):
    """tc_tile_shape (tc_gemm.cu): the widest power-of-two Wt <= 128 that pads the fewest pixels; Ht = 128 / Wt."""
    best = None
    for wt in (128, 64, 32, 16, 8):
        ht = 128 // wt
        cost = math.ceil(W / wt) * wt * math.ceil(H / ht) * ht
        if best is None or cost < best[0]:
            best = (cost, wt, ht)
    return best[1], best[2]


def out_dims(c, H, W):
    if c.stride == 2:
        return (H + 2 - c.k) // 2 + 1, (W + 2 - c.k) // 2 + 1
    return (2 * H, 2 * W) if c.up else (H, W)


def tile_grid(c, B, H, W):
    """The grid femasr_tc_igemm tiles: the output for stride 2, the low-res input for upsample, all tokens as one row for k 1."""
    if c.k == 1:
        return 1, B * H * W
    return out_dims(c, H, W) if c.stride == 2 else (H, W)


def shapes_of(c):
    """(B, H, W) of the conv INPUT: exact fit, ragged multi-tile, wide rows."""
    if c.k == 1:
        return [(1, 8, 16), (1, 7, 111), (2, 5, 200)]
    if c.stride == 2 and c.k == 3:
        return [(1, 15, 31), (2, 26, 73), (1, 10, 399)]        # -> 8x16, 13x37, 5x200; odd and even input sizes
    if c.stride == 2:                                            # 4x4: odd input sizes, which only the ABI accepts
        return [(1, 16, 32), (2, 27, 75), (1, 10, 400)]        # -> 8x16, 13x37, 5x200
    return [(1, 8, 16), (2, 13, 37), (1, 5, 200)]


def check_shapes(c):
    """The three shapes must stay an exact fit, a ragged multi-tile case and a Wt = 128 case under the tiling rule."""
    exact, ragged, wide = [(tile_grid(c, *s), s[0]) for s in shapes_of(c)]
    (h, w), _ = exact
    wt, ht = tile_shape(h, w)
    assert h % ht == 0 and w % wt == 0 and (h // ht) * (w // wt) == 1, (c.name, "exact", wt, ht)
    (h, w), b = ragged
    wt, ht = tile_shape(h, w)
    ntiles = b * math.ceil(h / ht) * math.ceil(w / wt)
    assert ntiles > 2 and w % wt != 0 and (c.k == 1 or h % ht != 0), (c.name, "ragged", wt, ht)
    (h, w), _ = wide
    wt, ht = tile_shape(h, w)
    assert (wt, ht) == (128, 1) and w % 128 != 0 and w > 128, (c.name, "wide", wt, ht)


for _c in CLASSES + SIMT_ONLY:         # (ACCEPTED rows run at the ragged shape only)
    check_shapes(_c)

CASES = [pytest.param(c, ci, co, si, id=f"{c.name}-{ci}x{co}-{('fit', 'ragged', 'wide')[si]}")
         for c in CLASSES for (ci, co) in c.ch for si in range(3)]
ACCEPTED_CASES = [pytest.param(c, ci, co, verdict, id=f"{c.name}-{ci}x{co}") for c, verdict in ACCEPTED for (ci, co) in c.ch]
SIMT_CASES = [pytest.param(c, ci, co, si, id=f"{c.name}-{ci}x{co}-{si}") for c in SIMT_ONLY for (ci, co) in c.ch
              for si in range(3)]


# ------------------------------------------------------------------------------------------------ reference and data
def reference(c, x, w, b, gamma, beta, res1, res2):
    """y = act(conv(pro(x)) + bias) + res1 + res2 in float64 on the CPU; x NCHW, residuals NCHW like y."""
    v = x.double()
    if c.pro == "gn":
        v = F.silu(F.group_norm(v, 32, gamma.double(), beta.double(), 1e-6))
    elif c.pro == "ln":
        v = F.layer_norm(v.permute(0, 2, 3, 1), (v.shape[1],), gamma.double(), beta.double(), 1e-5).permute(0, 3, 1, 2)
    if c.up:
        v = v.repeat_interleave(2, 2).repeat_interleave(2, 3)
    w = w.double()
    if c.kb:          # k-blocks of 64 over k = tap * Cin + c: every weight outside the range counts as zero
        co, ci, kh, kw = w.shape
        k = (torch.arange(kh * kw).view(1, kh * kw, 1) * ci + torch.arange(ci).view(1, 1, ci)) // 64
        keep = (k >= c.kb[0]) & (k < c.kb[0] + c.kb[1])
        w = (w.permute(0, 2, 3, 1).reshape(co, kh * kw, ci) * keep).reshape(co, kh, kw, ci).permute(0, 3, 1, 2)
    y = F.conv2d(v, w, None if b is None else b.double(), stride=c.stride, padding={1: 0, 3: 1, 4: 1, 5: 2}[c.k])
    if c.act == GELU:
        y = F.gelu(y)
    elif c.act == RELU:
        y = F.relu(y)
    elif c.act == LRELU:
        y = F.leaky_relu(y, 0.2)
    for r in (res1, res2):
        if r is not None:
            y = y + r.double()
    return y


def rnd(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g) * scale


def split_exact(x):
    """x rounded so that fp16(x) + fp16(x - fp16(x)) == x: planes a producer wrote hold exactly these values."""
    hi = x.half()
    return hi.float() + (x - hi.float()).half().float()


def make_data(c, cin, cout, shape, cuda, seed):
    """The tensors of one (class, shape), made once: CPU fp32 values, their device copies, and the fp64 reference."""
    B, H, W = shape
    g = torch.Generator().manual_seed(seed)
    d = dict(B=B, H=H, W=W, cin=cin, cout=cout)
    x = rnd(g, B, cin, H, W, scale=2.0) + 0.5 if c.pro != "none" else rnd(g, B, cin, H, W)
    if c.operand == "planes":
        x = split_exact(x)
    w = rnd(g, cout, cin, c.k, c.k, scale=0.03)
    b = rnd(g, cout) if c.bias else None
    gamma = beta = None
    if c.pro != "none":
        gamma, beta = 1 + 0.2 * rnd(g, cin), 0.2 * rnd(g, cin)
    Ho, Wo = out_dims(c, H, W)
    res1 = rnd(g, B, cout, Ho, Wo) if c.res1 != "none" else None
    res2 = rnd(g, B, cout, Ho, Wo) if c.res2 else None
    d["want"] = reference(c, x, w, b, gamma, beta, res1, res2).permute(0, 2, 3, 1).contiguous()      # NHWC like y
    dev = lambda t: None if t is None else t.to(cuda)
    d.update(x=G.nhwc(x).to(cuda), w=w.to(cuda), b=dev(b), gamma=dev(gamma), beta=dev(beta), Ho=Ho, Wo=Wo,
             res1=None if res1 is None else G.nhwc(res1).to(cuda), res2=None if res2 is None else G.nhwc(res2).to(cuda))
    if c.pro == "gn":
        d["sc"], d["sh"] = G.gn_tables(d["x"], d["gamma"], d["beta"])
    return d


def rel_err(got, want64):
    return ((got.double().cpu() - want64).abs().max() / want64.abs().max()).item()


def describe(got, want64, c, B, H, W):
    """Where the largest error sits: for the report of a case over its bar."""
    e = (got.double().cpu() - want64).abs()
    i = int(e.argmax())
    b, y, x, ch = (int(v) for v in torch.unravel_index(torch.tensor(i), e.shape))
    wt, ht = tile_shape(*tile_grid(c, B, H, W))
    return f"worst at image {b} y {y} x {x} channel {ch} (tiles {wt}x{ht}); errors over half of it: {int((e > e.max() / 2).sum())}"


# ------------------------------------------------------------------------------------------------ guard bands
GUARD = 2048                     # elements in front of and behind every output the kernels write
SENTINEL = 1234.5                # exactly representable in fp16 and fp32


def guarded(shape, dtype, device, fill=float("nan")):
    """(whole buffer, view of `shape` inside it): guard bands of SENTINEL around a tensor pre-filled with `fill`."""
    n = math.prod(shape)
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=dtype, device=device)
    view = buf[GUARD:GUARD + n].view(shape)
    view.fill_(fill)
    return buf, view


def assert_canaries(buf, what):
    inner = buf[GUARD:-GUARD]
    assert not torch.isnan(inner).any(), f"{what}: not every element was written"
    assert bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[-GUARD:] == SENTINEL).all()), f"{what}: wrote outside the tensor"


# ------------------------------------------------------------------------------------------------ the two kernels
def tc_operand(c, d):
    """The operand planes and weight blob femasr_tc_igemm reads for class c, staged as Ctx::conv stages them."""
    f8 = c.num.startswith("f8")
    if f8:
        mode = L.PRO_GN_SILU_FAST if c.pro == "gn" else L.PRO_NONE
        hi, lo = G.tc_prepare_f8(d["x"], mode, d.get("sc"), d.get("sh"))
        blob = G.tc_pack_f8(d["w"], up2=bool(c.up))
    else:
        if c.pro == "gn":
            hi, lo = G.tc_prepare(d["x"], L.PRO_GN_SILU, d["sc"], d["sh"])
        elif c.pro == "ln":
            hi, lo = G.tc_prepare(d["x"], L.PRO_LN, gamma=d["gamma"], beta=d["beta"], eps=1e-5)
        else:
            hi, lo = G.tc_prepare(d["x"])
        blob = G.tc_pack_up2(d["w"]) if c.up else G.tc_pack(d["w"])
    return hi, lo, blob


def tc_call(c, d, op, alias=False, split=None):
    """One femasr_tc_igemm launch into guarded outputs.  Returns (y or (hi, lo) views, partial view or None, buffers)."""
    hi, lo, blob = op
    B, Ho, Wo, cout = d["B"], d["Ho"], d["Wo"], d["cout"]
    split = (c.out == "split") if split is None else split
    bufs, kw = {}, {}
    res1 = d["res1"]
    if split:
        bufs["out_hi"], oh = guarded((B, Ho, Wo, cout), torch.float16, hi.device)
        bufs["out_lo"], ol = guarded((B, Ho, Wo, cout), torch.float16, hi.device)
        kw["out_planes"] = (oh, ol)
    else:
        bufs["y"], y = guarded((B, Ho, Wo, cout), torch.float32, hi.device)
        if alias:
            y.copy_(res1)
            res1 = y
        kw["y"] = y
    part = None
    if c.gn:
        rows = G.tc_gn_rows(B, d["H"], d["W"], d["cin"], cout, upsample=c.up, stride=c.stride)
        bufs["gn_partial"], part = guarded((B, rows, 32, 2), torch.float32, hi.device)
    if c.kb:
        kw.update(kb_begin=c.kb[0], kb_count=c.kb[1])
    G.tc_igemm(hi, lo, blob, d["b"], cout, c.k, act=c.act, res1=res1, res2=d["res2"], upsample=c.up, stride=c.stride,
               gn_partial=part, slice_kb=4 if "slice" in c.num else 0, f8=int(c.num.startswith("f8")), **kw)
    return (kw["out_planes"] if split else kw["y"]), part, bufs


def simt_call(c, d, alias=False):
    B, H, W = d["B"], d["H"], d["W"]
    buf, y = guarded((B, d["Ho"], d["Wo"], d["cout"]), torch.float32, d["x"].device)
    res1 = d["res1"]
    if alias:
        y.copy_(res1)
        res1 = y
    kw = {}
    if c.pro == "gn":
        kw = dict(prologue=L.PRO_GN_SILU, pro_a=d["sc"], pro_b=d["sh"])
    elif c.pro == "ln":
        mu, rs = G.ln_stats(d["x"].view(-1, d["cin"]))
        kw = dict(prologue=L.PRO_LN, pro_a=mu, pro_b=rs, gamma=d["gamma"], beta=d["beta"])
    G.igemm(d["x"], G.pack_weight(d["w"]), d["b"], B, H, W, d["cin"], d["cout"], ksize=c.k, stride=c.stride, upsample=c.up,
            act=c.act, res1=res1, res2=d["res2"], y=y, **kw)
    return y, buf


def tc_bar(c):
    """Relative bar against fp64 (DESIGN.md section 4): one pass 2e-5; K-sliced 2e-6, 1e-5 for the 4x4 stride-2 convs
    (tests/test_disc_gpu.py); F8 1.5e-4.  GELU adds test_tc_split_output's 1e-5, the fast SiLU staging 2e-6."""
    bar = {"one": 2e-5, "slice": 1e-5 if c.k == 4 else 2e-6, "f8": 1.5e-4}[c.num]
    if c.act == GELU:
        bar += 1e-5
    if c.num == "f8" and c.pro == "gn":
        bar += 2e-6
    return bar


SIMT_BAR = 1e-5
WORST = {}       # numerics -> (largest relative error seen, case): printed by test_zz_largest_errors


def note(num, e, what):
    if e > WORST.get(num, (0.0, ""))[0]:
        WORST[num] = (e, what)


def check_simt(c, d, what):
    """femasr_igemm_simt on the same tensors: accuracy, canaries, in-place equality."""
    want = d["want"]
    y, buf = simt_call(c, d)
    assert_canaries(buf, f"simt {what}")
    e = rel_err(y, want)
    note("simt", e, what)
    assert e <= SIMT_BAR, f"simt {what}: rel err {e:.3e} > {SIMT_BAR:.1e}; {describe(y, want, c, d['B'], d['H'], d['W'])}"
    if c.res1 == "alias":
        y2, buf2 = simt_call(c, d, alias=True)
        assert_canaries(buf2, f"simt {what} in place")
        assert torch.equal(y2, y), f"simt {what}: in-place residual differs from out of place"
    return e


def check_tc(c, d, what):
    """femasr_tc_igemm: accuracy, canaries, split-output bits, GroupNorm partials, in-place equality."""
    lib = L.load()
    want, B, cout = d["want"], d["B"], d["cout"]
    op = tc_operand(c, d)
    out, part, bufs = tc_call(c, d, op)
    for k, buf in bufs.items():
        assert_canaries(buf, f"{what} {k}")
    y32 = out
    if c.out == "split":
        oh, ol = out
        y32, _, bufs32 = tc_call(c, d, op, split=False)
        assert_canaries(bufs32["y"], f"{what} y (fp32 rerun)")
        assert torch.equal(oh, y32.half()), f"{what}: out_hi != fp16(y)"
        assert torch.equal(ol, (y32 - oh.float()).half()), f"{what}: out_lo != fp16(y - hi)"
        got = oh.double() + ol.double()
    else:
        got = y32
    e = rel_err(got, want)
    note(c.num, e, what)
    bar = tc_bar(c)
    assert e <= bar, f"{what}: rel err {e:.3e} > {bar:.1e}; {describe(got, want, c, B, d['H'], d['W'])}"
    if c.gn:
        # summed over rows in fp64, the partials are the per-(image, group) sum and sum of squares of the stored output
        cpg = cout // 32
        v = y32.double().view(B, -1, 32, cpg)
        s, ss = v.sum((1, 3)), (v * v).sum((1, 3))
        ps = part.double().sum(1)
        count = v.shape[1] * cpg
        assert ((ps[..., 1] - ss).abs() <= 1e-6 * ss).all(), f"{what}: sum of squares partials"
        assert ((ps[..., 0] - s).abs() <= 1e-6 * count).all(), f"{what}: sum partials"
        g = torch.Generator().manual_seed(7)
        gamma, beta = (1 + 0.2 * rnd(g, cout)).to(y32.device), (0.2 * rnd(g, cout)).to(y32.device)
        sc, sh = torch.empty(B, cout, device=y32.device), torch.empty(B, cout, device=y32.device)
        L.check(lib.femasr_gn_finalize_rows(G.p(part), G.p(gamma), G.p(beta), G.p(sc), G.p(sh), B, part.shape[1],
                                            d["Ho"] * d["Wo"], cout, 1e-6, G.S()))
        sc2, sh2 = G.gn_tables(y32.contiguous(), gamma, beta)
        assert (sc - sc2).abs().max().item() <= 2e-6 * sc2.abs().max().item(), f"{what}: finalize_rows scale"
        assert (sh - sh2).abs().max().item() <= 2e-6 * max(1.0, sh2.abs().max().item()), f"{what}: finalize_rows shift"
    if c.res1 == "alias":
        out2, part2, bufs2 = tc_call(c, d, op, alias=True, split=False)
        assert_canaries(bufs2["y"], f"{what} y in place")
        assert torch.equal(out2, y32), f"{what}: in-place residual differs from out of place"
        if c.gn:
            assert torch.equal(part2, part), f"{what}: partials of the in-place call differ"
    return e


def run_case(cuda, c, cin, cout, si, seed):
    shape = shapes_of(c)[si]
    what = f"{c.name} {cin}->{cout} at {shape}"
    d = make_data(c, cin, cout, shape, cuda, seed)
    e_tc = check_tc(c, d, what)
    e_simt = check_simt(c, d, what)
    print(f"{what} [{c.num}]: tc rel err {e_tc:.2e} (bar {tc_bar(c):.1e}), simt {e_simt:.2e}")


@pytest.mark.parametrize("c,cin,cout,si", CASES)
def test_engine_class(cuda, c, cin, cout, si):
    run_case(cuda, c, cin, cout, si, seed=1000 + si)


@pytest.mark.parametrize("c,cin,cout,si", SIMT_CASES)
def test_simt_cin_multiple_of_16(cuda, c, cin, cout, si):
    shape = shapes_of(c)[si]
    check_simt(c, make_data(c, cin, cout, shape, cuda, 1100 + si), f"{c.name} {cin}->{cout} at {shape}")


@pytest.mark.parametrize("c,cin,cout,verdict", ACCEPTED_CASES)
def test_accepted_is_right_or_refused(cuda, c, cin, cout, verdict):
    """A call outside the engine's classes meets the fp64 bar or returns FEMASR_ERR_ARG - never a wrong result."""
    shape = shapes_of(c)[1]
    what = f"{c.name} {cin}->{cout} at {shape}"
    d = make_data(c, cin, cout, shape, cuda, 1200)
    if verdict == "right":
        check_tc(c, d, what)
    else:       # refused on the host before any operand is read: staged as the plain conv, which every helper can pack
        op = tc_operand(dataclasses.replace(c, up=0, num="f8" if c.num.startswith("f8") else "one"), d)
        with pytest.raises(L.FemasrError, match="error -1"):
            tc_call(c, d, op)
    if c.name in SIMT_REFUSES:
        with pytest.raises(L.FemasrError, match="error -1"):
            simt_call(c, d)
    elif not c.kb:                         # femasr_igemm_simt has no K ranges; every other row it computes
        check_simt(c, d, what)


# ------------------------------------------------------------------------------------------------ persistent-loop invariants
def by_name(name):
    return next(c for c in CLASSES if c.name == name)


# (class, Cin, Cout): one pass BN 128; slice_kb + stride 2 + partials; F8 + in-place residual + partials at BN 64 (cpg 2);
# F8 + upsample + partials at BN 64; slice_kb at BN 128 x 2 n-tiles; 4x4 taps; split output
INVARIANT_CASES = [("vgg_f32", 128, 128), ("down_planes", 64, 128), ("res5_f8_gn", 64, 64), ("up_f8", 128, 64),
                   ("swin_conv", 256, 256), ("disc_down", 64, 128), ("vgg_split", 64, 128)]


@pytest.mark.parametrize("name,cin,cout", INVARIANT_CASES, ids=[f"{n}-{a}x{b}" for n, a, b in INVARIANT_CASES])
def test_batch_invariance_and_repeatability(cuda, name, cin, cout):
    """Image b of a large batch == the same image run alone, bit for bit, output and partial rows; two identical calls are
    bit-identical.  The batch has several times more tiles than the launch has CTAs (min(tiles, SM count)), so a tile
    computed as some CTA's fifth work item is compared with the same tile computed as a first one: accumulator, running
    sum, pipeline phase or partial-sum state leaking from one tile into the next shows here."""
    c = by_name(name)
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    H, W = (26, 37) if c.stride == 2 else (13, 19)
    th, tw = tile_grid(c, 1, H, W)
    wt, ht = tile_shape(th, tw)
    per_image = math.ceil(th / ht) * math.ceil(tw / wt) * (4 if c.up else 1) * (cout // (128 if cout % 128 == 0 else 64))
    B = math.ceil(5 * sms / per_image) + 1
    g = torch.Generator().manual_seed(1300)
    d = dict(B=B, H=H, W=W, cin=cin, cout=cout)
    d["Ho"], d["Wo"] = out_dims(c, H, W)
    x = rnd(g, B, H, W, cin, scale=2.0) + 0.5 if c.pro != "none" else rnd(g, B, H, W, cin)
    d.update(x=x.to(cuda), w=rnd(g, cout, cin, c.k, c.k, scale=0.03).to(cuda), b=rnd(g, cout).to(cuda) if c.bias else None,
             res1=rnd(g, B, d["Ho"], d["Wo"], cout).to(cuda) if c.res1 != "none" else None, res2=None)
    if c.pro == "gn":
        d["gamma"], d["beta"] = (1 + 0.2 * rnd(g, cin)).to(cuda), (0.2 * rnd(g, cin)).to(cuda)
        d["sc"], d["sh"] = G.gn_tables(d["x"], d["gamma"], d["beta"])
    hi, lo, blob = tc_operand(c, d)
    out, part, _ = tc_call(c, d, (hi, lo, blob))
    out_b, part_b, _ = tc_call(c, d, (hi, lo, blob))
    planes = lambda o: o if isinstance(o, tuple) else (o,)
    for a, b in zip(planes(out), planes(out_b)):
        assert torch.equal(a, b), "two identical calls differ"
    assert part is None or torch.equal(part, part_b), "two identical calls differ in their partials"
    ys = simt_call(c, d)[0]
    assert torch.equal(ys, simt_call(c, d)[0]), "simt: two identical calls differ"
    for i in sorted({0, 1, B // 2, B - 2, B - 1}):
        one = {k: v[i:i + 1] if k in ("x", "res1", "sc", "sh") and v is not None else v for k, v in d.items()}
        one["B"] = 1
        o1, p1, _ = tc_call(c, one, (hi[i:i + 1], lo[i:i + 1], blob))
        for a, b in zip(planes(out), planes(o1)):
            assert torch.equal(a[i:i + 1], b), f"image {i} of {B} differs from the same image alone"
        assert part is None or torch.equal(part[i:i + 1], p1), f"partial rows of image {i} of {B} differ from the image alone"
        assert torch.equal(ys[i:i + 1], simt_call(c, one)[0]), f"simt: image {i} of {B} differs from the same image alone"


@pytest.mark.parametrize("step", [3, 5])
def test_k_range_additivity(cuda, step):
    """Chained kb_begin / kb_count launches with res1 = y sum to the whole conv at the K-sliced bar: Cin = 128 has two
    k-blocks per tap, so slices of 3 and of 5 begin inside a tap, and 18 k-blocks in slices of 5 leave a last slice of 3."""
    c = Cls("k_range", ((128, 128),))
    B, H, W = shapes_of(c)[1]
    d = make_data(c, 128, 128, (B, H, W), cuda, 1400)
    hi, lo, blob = tc_operand(c, d)
    buf, y = guarded((B, H, W, 128), torch.float32, cuda)
    for k0 in range(0, 18, step):
        G.tc_igemm(hi, lo, blob, d["b"] if k0 == 0 else None, 128, 3, res1=None if k0 == 0 else y, y=y, kb_begin=k0,
                   kb_count=min(step, 18 - k0))
    assert_canaries(buf, "chained k-ranges")
    e = rel_err(y, d["want"])
    print(f"k-range chain in slices of {step}: rel err {e:.2e}")
    assert e <= 2e-6


def test_zz_largest_errors(cuda):
    """Runs last in this file: the largest relative error each numerics mode showed (DESIGN.md section 6, GEMM matrix)."""
    for num, (e, what) in sorted(WORST.items()):
        print(f"largest rel err, {num}: {e:.2e} ({what})")
