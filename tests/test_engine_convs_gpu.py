"""GPU: every conv / linear launch of the engine's networks against float64 on its own operands.

For each configuration and GEMM path the conv trace of a sizing run (femasr_net_conv_trace_json) lists the Ctx::conv
calls; femasr_net_set_conv_capture copies each call's operand (fp32 x, or the split planes a producer wrote), residuals,
output and GroupNorm partials out of a real forward.  Each launch is then recomputed on the CPU in float64 from the
captured operand and the module's own parameters, looked up by the trace's weight name: the prologue (GroupNorm(32,
1e-6) + SiLU or LayerNorm(1e-5), from the state dict's gamma / beta, not the engine's tables), nearest x2, the conv,
bias, activation and the captured residuals.  Spectral-norm weights are weight_orig / sigma with sigma from u and v in
float64.  The im2col GEMMs (in_conv, the discriminator's conv0, VGG conv1_1, the LPIPS first convs) are checked against
conv2d of the network input with the unpadded weight.  Prologue, activation, bias and numerics class come from the
layer's place in the network (as_cls), and the bar is the GEMM matrix's for that class (tests/test_gemm_matrix_gpu.py:
tc_bar, SIMT_BAR), so a wrong eps, gamma, SiLU form, K-slicing, F8 or bias in the wiring of one layer fails here, naming
the layer.  The quantiser (z . E^T on gemm_path 0) is the VQ matrix's.

Also: outputs of every run with captures registered are bitwise equal to a run without, and the real run's trace equals
the sizing run's."""
import ctypes as C
import json
import math

import pytest
import torch
import torch.nn.functional as F

from femasr_b200 import lib as L
from femasr_b200.net import NativeDisc, NativeLPIPS, NativeNet
from femasr_b200.spec import random_disc_state_dict, random_lpips_state_dict, random_state_dict
from tests import gpu_util as G
from tests.test_conv_trace import expect_precise, f8_form, k_blocks, rec_key
from tests.test_engine_plan import CONFIGS
from tests.test_gemm_matrix_gpu import SIMT_BAR, Cls, check_gn_partials, reference, rel_err, tc_bar

pytestmark = pytest.mark.gpu

# (configuration, (B, H, W) of the input): Swin map 24 x 40 for the LQ nets; the HQ net runs the semantic VGG19
CASES = [("x4_e256", (2, 48, 80)), ("x2_cb3", (2, 96, 160)), ("hq_e512_sem", (1, 192, 320)),
         ("disc_skip", (2, 24, 40)), ("disc_noskip", (2, 24, 40)), ("lpips_alex", (2, 67, 93)), ("lpips_vgg", (2, 32, 48))]
CAPTURE_BYTES = 4 << 30        # device bytes of captures registered per forward
# Launches whose operand is a ReLU / LeakyReLU output (VGG, LPIPS, the discriminator after conv0) measured up to 1.52
# times the matrix's bar for their class, an error of the GEMM itself: they have no prologue, so no statistics enter.
# The matrix draws zero-mean operands; the ratio kappa of the products' absolute sum to max |y| does not explain the
# difference (DESIGN.md section 6, per-launch matrix).  Those launches get twice the bar.
POST_ACT = 2.0
WORST = {}                     # class -> (largest relative error, layer): printed by test_zz_largest_errors


# ------------------------------------------------------------------------------------------------ the engines
class Run:
    """One engine handle, its state dict, its input and one forward entry point over a workspace."""

    def __init__(self, name, gemm_path, shape, dev):
        B, H, W = shape
        self.name, self.shape, self.dev = name, shape, dev
        g = torch.Generator().manual_seed(B * H + W)
        if name.startswith("disc"):
            self.sd = random_disc_state_dict(seed=81)
            self.eng = NativeDisc(skip_connection=name == "disc_skip", gemm_path=gemm_path)
            self.x = torch.rand(B, 3, H, W, generator=g)
        elif name.startswith("lpips"):
            net = name.split("_")[1]
            self.sd = random_lpips_state_dict(net, seed=82)
            self.eng = NativeLPIPS(net, gemm_path=gemm_path)
            self.x = torch.rand(2 * B, 3, H, W, generator=g)           # x0 then x1
        else:
            scale, cbs, sem, _tap = CONFIGS[name]
            self.sd = random_state_dict(scale, cbs[0][2], seed=80, init="perturbed", codebooks=cbs, semantic=sem)
            self.eng = NativeNet(scale, cbs[0][1], cbs[0][2], gemm_path=gemm_path, codebooks=cbs, use_semantic_loss=sem)
            self.x = torch.rand(B, 3, H, W, generator=g)
            self.sem = sem
        self.eng.load_state_dict(self.sd, dev)
        self.xd = self.x.to(dev)
        self.lib, self.h = self.eng.lib, self.eng._h
        need = C.c_size_t()
        L.check(self.size(need))
        self.need = need.value
        self.trace = json.loads(self.lib.femasr_net_conv_trace_json(self.h).decode())

    def size(self, need):
        B, H, W = self.shape
        if self.name.startswith("disc"):
            return self.lib.femasr_disc_workspace_bytes(self.h, B, H, W, C.byref(need))
        if self.name.startswith("lpips"):
            return self.lib.femasr_lpips_workspace_bytes(self.h, B, H, W, C.byref(need))
        return self.lib.femasr_net_workspace_bytes_sem(self.h, B, H, W, int(self.sem), C.byref(need))

    def forward(self):
        """The network's outputs (a dict of device tensors) from one real run."""
        B, H, W = self.shape
        ws = torch.empty(self.need, dtype=torch.uint8, device=self.dev)
        d = lambda *s, dt=torch.float32: torch.empty(s, dtype=dt, device=self.dev)
        if self.name.startswith("disc"):
            o = dict(y=d(B, 1, H, W))
            s = self.lib.femasr_disc_forward(self.h, self.xd.data_ptr(), o["y"].data_ptr(), B, H, W, ws.data_ptr(),
                                             self.need, G.S())
        elif self.name.startswith("lpips"):
            o = dict(d=d(B), r=d(5, B))
            s = self.lib.femasr_lpips_forward(self.h, self.xd[:B].data_ptr(), self.xd[B:].data_ptr(), o["d"].data_ptr(),
                                              o["r"].data_ptr(), B, H, W, 1, ws.data_ptr(), self.need, G.S())
        else:
            e = self.eng
            nidx = sum(math.prod(sh) for sh in e.index_shapes(B, H, W))
            o = dict(y=d(B, 3, H * e.scale, W * e.scale), idx=d(nidx, dt=torch.int64), loss=d())
            if self.sem:
                o["sem"] = d()
            s = self.lib.femasr_net_forward_sem(self.h, self.xd.data_ptr(), o["y"].data_ptr(), o["idx"].data_ptr(),
                                                o["loss"].data_ptr(), None, G.p(o.get("sem")), B, H, W, ws.data_ptr(),
                                                self.need, G.S())
        L.check(s)
        torch.cuda.synchronize()
        return o


# ------------------------------------------------------------------------------------------------ captures
def out_hw(r):
    if r["stride"] == 2:
        return (r["H"] + 2 - r["k"]) // 2 + 1, (r["W"] + 2 - r["k"]) // 2 + 1
    return r["H"] << r["upsample"], r["W"] << r["upsample"]


def captures_of(r):
    """{what: (dtype, NHWC shape)} this test takes from the launch of record r."""
    B, Cin, Cout = r["B"], r["Cin"], r["Cout"]
    Ho, Wo = out_hw(r)
    x, o = (B, r["H"], r["W"], Cin), (B, Ho, Wo, Cout)
    caps = {}
    if r["operand"] == "planes":
        caps.update(a_hi=(torch.float16, x), a_lo=(torch.float16, x))
    elif r["operand"] == "staged":
        caps["x"] = (torch.float32, x)
    if r["prologue"] in ("gn", "gn_fast"):                      # the engine's own tables, for a report over the bar
        caps.update(pa=(torch.float32, (B, Cin)), pb=(torch.float32, (B, Cin)))
    if r["res1"] != "none":
        caps["res1"] = (torch.float32, o)
    if r["res2"]:
        caps["res2"] = (torch.float32, o)
    if r["out"] == "split":
        caps.update(o_hi=(torch.float16, o), o_lo=(torch.float16, o))
    else:
        caps["y"] = (torch.float32, o)
    if r["gn_partial"]:
        rows = G.tc_gn_rows(B, r["H"], r["W"], Cin, Cout, upsample=r["upsample"], stride=r["stride"])
        caps["gn_partial"] = (torch.float32, (B, rows, 32, 2))
    return caps


def nbytes(caps):
    return sum(math.prod(s) * torch.empty((), dtype=dt).element_size() for dt, s in caps.values())


def chunks(records):
    """The records in groups whose captures fit CAPTURE_BYTES together."""
    group, size = [], 0
    for r in records:
        n = nbytes(captures_of(r))
        if group and size + n > CAPTURE_BYTES:
            yield group
            group, size = [], 0
        group.append(r)
        size += n
    if group:
        yield group


def captured_forward(run, group):
    """One forward with every capture of `group` registered: ({ordinal: {what: CPU tensor}}, the outputs)."""
    bufs = {r["ordinal"]: {k: torch.full(s, float("nan"), dtype=dt, device=run.dev) for k, (dt, s) in captures_of(r).items()}
            for r in group}
    for o, caps in bufs.items():
        for k, t in caps.items():
            L.check(run.lib.femasr_net_set_conv_capture(run.h, o, k.encode(), t.data_ptr(), t.numel() * t.element_size()))
    try:
        out = run.forward()
    finally:
        for o, caps in bufs.items():
            for k in caps:
                run.lib.femasr_net_set_conv_capture(run.h, o, k.encode(), None, 0)
    return {o: {k: t.cpu() for k, t in caps.items()} for o, caps in bufs.items()}, out


# ------------------------------------------------------------------------------------------------ float64 reference
def weight(sd, r):
    """The launch's OIHW weight in float64 (spectral norm: weight_orig / u . (W v); a Linear's [out, in] as 1x1) and its
    bias."""
    w = sd[r["w"]].double()
    if w.dim() == 2:
        w = w[:, :, None, None]
    if r["sn"]:
        p = r["w"][: -len(".weight_orig")]
        sigma = torch.dot(sd[p + ".weight_u"].double(), w.reshape(w.shape[0], -1) @ sd[p + ".weight_v"].double())
        return w / sigma, None
    b = sd.get(r["w"][: -len(".weight")] + ".bias")
    return w, None if b is None else b.double()


def norm_params(sd, r):
    """gamma, beta of the norm in front of the layer (ResBlock conv.2 / conv.5: conv.0 / conv.3; Swin qkv / fc1:
    norm1 / norm2)."""
    w = r["w"]
    for conv, norm in ((".conv.2.weight", ".conv.0.norm"), (".conv.5.weight", ".conv.3.norm"),
                       (".attn.qkv.weight", ".norm1"), (".mlp.fc1.weight", ".norm2")):
        if w.endswith(conv):
            p = w[: -len(conv)] + norm
            return sd[p + ".weight"], sd[p + ".bias"]
    raise AssertionError(f"{w}: no norm in front of this layer")


def first_input(run, r):
    """The network input an im2col GEMM reads, after its scaling, in float64 NCHW."""
    x = run.x.double()
    if r["w"].startswith("vgg_feat_extractor."):
        return (x - run.sd["vgg_feat_extractor.mean"].double()) / run.sd["vgg_feat_extractor.std"].double()
    if run.name.startswith("lpips"):
        return (2 * x - 1 - run.sd["scaling_layer.shift"].double()) / run.sd["scaling_layer.scale"].double()
    return x


def as_cls(run, r):
    """The launch as a matrix class (tc_bar and reference read num, k, stride, up, pro, act).  Prologue, activation, bias
    and numerics come from the layer's place in the network, not from the trace, so a launch wired like another layer
    is held to its own layer's reference and bar."""
    operand, _num, out, res1, res2, gn, _pro, _act, _bias, k, stride, up = rec_key(r)
    w, name = r["w"], run.name
    pro = ("gn" if w.endswith((".conv.2.weight", ".conv.5.weight")) else
           "ln" if w.endswith((".attn.qkv.weight", ".mlp.fc1.weight")) else "none")
    semantic = name.startswith("lpips") or w.startswith(("vgg_feat_extractor.", "conv_semantic."))
    act = (L.ACT_GELU if w.endswith(".mlp.fc1.weight") else L.ACT_RELU if semantic else
           L.ACT_LRELU if name.startswith("disc") else L.ACT_NONE)
    num = "one"
    if r["path"] == "tc" and not semantic:
        if name.startswith("disc") or expect_precise(name, ("forward",), w):
            num = "slice" if k_blocks(r) > 4 else "one"
        elif f8_form(r) and pro != "ln" and r["operand"] == "staged":
            num = "f8"
    return Cls(w, ((r["Cin"], r["Cout"]),), k=k, stride=stride, up=up, pro=pro, act=act, bias=weight(run.sd, r)[1] is not None,
               res1=res1, res2=res2, out=out, gn=gn, operand=operand, num=num)


def nchw(t):
    return None if t is None else t.permute(0, 3, 1, 2)


def want_of(run, r, cap):
    """float64 NHWC result of launch r from its captured operands."""
    c = as_cls(run, r)
    w, b = weight(run.sd, r)
    if r["operand"] == "im2col":
        k = w.shape[-1]
        y = F.conv2d(first_input(run, r), w, b, stride=4 if k == 11 else 1, padding=2 if k == 11 else 1)
        y = {L.ACT_NONE: lambda t: t, L.ACT_RELU: F.relu, L.ACT_LRELU: lambda t: F.leaky_relu(t, 0.2)}[c.act](y)
        assert r["res1"] == "none" and not r["res2"]
        return y.permute(0, 2, 3, 1)
    x = cap["a_hi"].double() + cap["a_lo"].double() if "a_hi" in cap else cap["x"]
    gamma = beta = None
    if c.pro != "none":
        gamma, beta = norm_params(run.sd, r)
    return reference(c, nchw(x), w, b, gamma, beta, nchw(cap.get("res1")), nchw(cap.get("res2"))).permute(0, 2, 3, 1)


def got_of(cap):
    return cap["o_hi"].double() + cap["o_lo"].double() if "o_hi" in cap else cap["y"]


def with_engine_tables(run, r, cap):
    """The same launch in float64 with the engine's GroupNorm scale / shift instead of fp64 statistics: tells a GEMM
    error from a statistics error when a launch goes over its bar."""
    w, b = weight(run.sd, r)
    x = (cap["a_hi"].double() + cap["a_lo"].double() if "a_hi" in cap else cap["x"].double())
    v = F.silu(x * cap["pa"].double()[:, None, None, :] + cap["pb"].double()[:, None, None, :])
    c = as_cls(run, r)
    return reference(Cls(c.name, c.ch, k=c.k, stride=c.stride, up=c.up, act=c.act), nchw(v), w, b, None, None,
                     nchw(cap.get("res1")), nchw(cap.get("res2"))).permute(0, 2, 3, 1)


def kappa(run, r, cap, want):
    """max conv(|x|, |w|) / max |y| of a launch without prologue: the absolute sum of the products an accumulation error
    scales with, over the magnitude the error is measured against (DESIGN.md section 6, per-launch matrix)."""
    if r["operand"] == "im2col" or r["prologue"] != "none":
        return float("nan")
    c = as_cls(run, r)
    x = cap["a_hi"].double() + cap["a_lo"].double() if "a_hi" in cap else cap["x"].double()
    a = reference(Cls(c.name, c.ch, k=c.k, stride=c.stride, up=c.up), nchw(x).abs(), weight(run.sd, r)[0].abs(), None,
                  None, None, None, None)
    return a.max().item() / want.abs().max().item()


def bar_of(r, c, gemm_path):
    """The GEMM matrix's bar for the launch's class; POST_ACT times it where the operand is a ReLU / LeakyReLU output."""
    if not gemm_path:
        return SIMT_BAR
    post_act = r["act"] in (L.ACT_RELU, L.ACT_LRELU) and r["operand"] != "im2col" and r["w"] != "conv_semantic.0.weight"
    return tc_bar(c) * (POST_ACT if post_act else 1.0)


def check_launch(run, r, cap, gemm_path):
    what = f"{run.name}/gp{gemm_path} #{r['ordinal']} {r['w']} {r['Cin']}->{r['Cout']}"
    for k, t in cap.items():
        assert not torch.isnan(t.float()).any(), f"{what}: capture {k} not written"
    c = as_cls(run, r)
    got, want = got_of(cap), want_of(run, r, cap)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    e = rel_err(got, want)
    cls = f"tc:{c.num}" if gemm_path else "simt"
    bar = bar_of(r, c, gemm_path)
    if e > WORST.get(cls, (0.0, ""))[0]:
        WORST[cls] = (e, f"{what}, bar {bar:.1e}, kappa {kappa(run, r, cap, want):.2f}")
    if e > bar:
        msg = f"{what} [{cls}]: rel err {e:.3e} > {bar:.1e}, kappa {kappa(run, r, cap, want):.2f}"
        if "pa" in cap:
            msg += f"; with the engine's own GroupNorm tables {rel_err(got, with_engine_tables(run, r, cap)):.3e}"
        raise AssertionError(msg)
    if r["gn_partial"]:
        check_gn_partials(cap["gn_partial"].to(run.dev), cap["y"].to(run.dev), what)
    return e


# ------------------------------------------------------------------------------------------------ the test
def same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32)) if a.dtype == torch.float32 else torch.equal(a, b)


@pytest.mark.parametrize("gemm_path", [0, 1])
@pytest.mark.parametrize("name,shape", CASES, ids=[n for n, _s in CASES])
def test_every_launch_against_float64(cuda, name, shape, gemm_path):
    run = Run(name, gemm_path, shape, cuda)
    base = run.forward()
    assert json.loads(run.lib.femasr_net_conv_trace_json(run.h).decode()) == run.trace, "real run's trace != sizing run's"
    records = [r for r in run.trace if not r["w"].startswith("quantize_group.")]
    assert len(records) >= 5
    worst = (0.0, "")
    for group in chunks(records):
        caps, out = captured_forward(run, group)
        for k in base:
            assert same_bits(out[k], base[k]), f"{name}/gp{gemm_path}: output {k} changes with captures registered"
        for r in group:
            e = check_launch(run, r, caps[r["ordinal"]], gemm_path)
            worst = max(worst, (e, f"#{r['ordinal']} {r['w']}"))
        del caps
    print(f"{name}/gp{gemm_path}: {len(records)} launches, largest rel err {worst[0]:.2e} ({worst[1]})")


def test_capture_errors(cuda):
    """A capture buffer that is too small, an ordinal the run never reaches and an operand the launch does not have
    each fail the run with FEMASR_ERR_ARG."""
    run = Run("disc_skip", 1, (1, 16, 16), cuda)
    r = run.trace[1]                                           # conv1: staged fp32 operand, no residual
    y = torch.empty(math.prod(captures_of(r)["y"][1]), device=cuda)
    for o, what, nb in ((1, b"y", y.numel() * 4 - 4), (len(run.trace), b"y", y.numel() * 4), (1, b"res1", y.numel() * 4)):
        L.check(run.lib.femasr_net_set_conv_capture(run.h, o, what, y.data_ptr(), nb))
        try:
            with pytest.raises(L.FemasrError, match="error -1"):
                run.forward()
        finally:
            run.lib.femasr_net_set_conv_capture(run.h, o, what, None, 0)
    run.forward()


def test_zz_largest_errors(cuda):
    """Runs last in this file: the largest relative error each numerics class showed, and where (DESIGN.md section 6)."""
    for cls, (e, what) in sorted(WORST.items()):
        print(f"largest rel err, {cls}: {e:.2e} ({what})")
