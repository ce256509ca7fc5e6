"""CPU: the conv trace of sizing runs (femasr_net_conv_trace_json) against the GEMM matrix's class table and the numerics
policy, for every configuration and legal shape of tests/test_engine_plan.py and every HEADS entry, on both GEMM paths.

- Matrix coverage both ways: every gemm_path 1 record is a row of test_gemm_matrix_gpu.CLASSES at one of that row's
  channel pairs, and every row and pair is launched by some configuration; every gemm_path 0 record is a class
  femasr_igemm_simt is checked on there.
- Numerics pinned per record: which layers sit in front of the last quantiser (precise_region), and in it no F8, no fast
  SiLU and K-slicing (slice_kb 4) wherever the launch has more than 4 k-blocks; behind it F8 for exactly the staged 3x3
  convs without a LayerNorm prologue whose weight has the F8 form, and the fast SiLU; the semantic branch and LPIPS in one
  pass without F8; every discriminator conv precise.
- The trace is repeatable and independent of registered taps and conv captures.
- Workspace bytes and traces ignore the environment variables that once selected other numerics."""
import ctypes
import json

import pytest

from femasr_b200 import lib
from tests.test_engine_plan import CONFIGS, DIV, HEAD_SHAPES, HEADS, SHAPES, head_plan, plan
from tests.test_gemm_matrix_gpu import ACCEPTED, CLASSES, SIMT_ONLY, SIMT_REFUSES

I3 = ctypes.c_int * 3


def trace(L, h):
    return json.loads(L.femasr_net_conv_trace_json(h).decode())


def create_gen(L, name, gemm_path):
    scale, cbs, sem, _tap = CONFIGS[name]
    pad = lambda v: I3(*(v + [0] * (3 - len(v))))
    cfg = lib.NetConfig(scale, cbs[0][1], cbs[0][2], 3, 1, 1, gemm_path, len(cbs), pad([c[0] for c in cbs]),
                        pad([c[1] for c in cbs]), pad([c[2] for c in cbs]))
    h = ctypes.c_void_p()
    assert L.femasr_net_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
    if sem:
        assert L.femasr_net_enable_semantic(h) == 0
    return h


def create_head(L, name, gemm_path):
    kind, arg = HEADS[name]
    h = ctypes.c_void_p()
    if kind == "disc":
        assert L.femasr_disc_create(ctypes.byref(lib.DiscConfig(3, 64, arg, gemm_path)), ctypes.byref(h)) == 0
    else:
        assert L.femasr_lpips_create(ctypes.byref(lib.LpipsConfig(arg, gemm_path)), ctypes.byref(h)) == 0
    return h


def gen_traces(L, name, gemm_path):
    """{(entry, B, H, W): trace} of every sizing run a generator configuration accepts: forward, forward with the
    semantic loss where it exists, decode_indices."""
    scale = CONFIGS[name][0]
    h = create_gen(L, name, gemm_path)
    out = {}
    try:
        n = ctypes.c_size_t()
        for (B, H, W) in SHAPES:
            if L.femasr_net_workspace_bytes(h, B, H, W, ctypes.byref(n)) != 0:
                continue
            out[("forward", B, H, W)] = trace(L, h)
            if L.femasr_net_workspace_bytes_sem(h, B, H, W, 1, ctypes.byref(n)) == 0:
                out[("forward_sem", B, H, W)] = trace(L, h)
            assert L.femasr_net_decode_workspace_bytes(h, B, H // DIV[scale], W // DIV[scale], ctypes.byref(n)) == 0
            out[("decode", B, H, W)] = trace(L, h)
    finally:
        L.femasr_net_destroy(h)
    return out


def head_traces(L, name, gemm_path):
    kind = HEADS[name][0]
    h = create_head(L, name, gemm_path)
    ws = L.femasr_disc_workspace_bytes if kind == "disc" else L.femasr_lpips_workspace_bytes
    out = {}
    try:
        n = ctypes.c_size_t()
        for (B, H, W) in HEAD_SHAPES[kind]:
            if ws(h, B, H, W, ctypes.byref(n)) == 0:
                out[(kind, B, H, W)] = trace(L, h)
    finally:
        L.femasr_net_destroy(h)
    return out


_ALL = {}


def all_traces(gemm_path):
    """[(configuration, run key, trace)] of every configuration, head and legal shape (computed once per path)."""
    if gemm_path not in _ALL:
        L = lib.load()
        runs = []
        for name in sorted(CONFIGS):
            runs += [(name, key, t) for key, t in gen_traces(L, name, gemm_path).items()]
        for name in sorted(HEADS):
            runs += [(name, key, t) for key, t in head_traces(L, name, gemm_path).items()]
        _ALL[gemm_path] = runs
    return _ALL[gemm_path]


# ------------------------------------------------------------------------------------------------ matrix classes
def cls_key(c):
    pro = c.pro
    return (c.operand, c.num, c.out, c.res1, c.res2, c.gn, pro, c.act, c.bias, c.k, c.stride, c.up)


def rec_key(r):
    """The record as the matrix's Cls columns: im2col rows are planes the im2col kernel wrote; the fast SiLU is what the
    F8 class stages for a GroupNorm prologue."""
    num = "f8" if r["f8"] else ("slice" if r["slice_kb"] == 4 else ("one" if r["slice_kb"] == 0 else f"slice{r['slice_kb']}"))
    pro = {"gn_fast": "gn"}.get(r["prologue"], r["prologue"])
    assert (r["prologue"] == "gn_fast") == (pro == "gn" and num == "f8"), ("fast SiLU outside the F8 class", r)
    operand = "planes" if r["operand"] == "im2col" else r["operand"]
    return (operand, num, r["out"], r["res1"], r["res2"], r["gn_partial"], pro, r["act"], r["bias"], r["k"], r["stride"],
            r["upsample"])


def simt_key(r):
    return (r["prologue"], r["act"], r["bias"], r["res1"] != "none", r["res2"], r["k"], r["stride"], r["upsample"])


def simt_classes():
    """The classes check_simt runs: every CLASSES row, the ACCEPTED rows femasr_igemm_simt computes, SIMT_ONLY."""
    rows = list(CLASSES) + [c for c, _v in ACCEPTED if c.name not in SIMT_REFUSES and not c.kb] + list(SIMT_ONLY)
    return {(c.pro, c.act, c.bias, c.res1 != "none", c.res2, c.k, c.stride, c.up) for c in rows}


def where(name, key, r):
    return f"{name} {key} #{r['ordinal']} {r['w']} {r['Cin']}->{r['Cout']}"


def test_every_tensor_core_launch_is_a_matrix_class(built_lib):
    by_key = {}
    for c in CLASSES:
        by_key.setdefault(cls_key(c), []).append(c)
    unmatched = []
    for name, key, t in all_traces(1):
        for r in t:
            assert r["path"] == "tc", where(name, key, r)
            rows = by_key.get(rec_key(r), [])
            if not any((r["Cin"], r["Cout"]) in c.ch for c in rows):
                unmatched.append(f"{where(name, key, r)}: {rec_key(r)} (rows {[c.name for c in rows]})")
    assert not unmatched, "launches no CLASSES row covers:\n" + "\n".join(sorted(set(unmatched))[:40])


def test_every_matrix_class_is_launched(built_lib):
    launched = set()
    for _name, _key, t in all_traces(1):
        launched |= {(rec_key(r), r["Cin"], r["Cout"]) for r in t}
    missing = [f"{c.name} {ci}x{co}" for c in CLASSES for (ci, co) in c.ch if (cls_key(c), ci, co) not in launched]
    assert not missing, f"CLASSES rows no configuration launches: {missing}"


def test_every_simt_launch_is_a_checked_class(built_lib):
    known = simt_classes()
    for name, key, t in all_traces(0):
        for r in t:
            assert r["path"] == "simt" and not r["f8"] and r["slice_kb"] == 0 and r["prologue"] != "gn_fast", where(name, key, r)
            assert r["out"] == "f32" and r["operand"] != "planes" and not r["gn_partial"], where(name, key, r)
            assert r["Cin"] % 16 == 0, where(name, key, r)
            assert simt_key(r) in known, f"{where(name, key, r)}: {simt_key(r)} is no class check_simt runs"


# ------------------------------------------------------------------------------------------------ numerics policy
def expect_precise(name, key, w):
    """Whether the layer with weight w sits in front of the configuration's last quantiser (Ctx::precise_region)."""
    if name.startswith("disc"):
        return True
    scale, cbs, _sem, _tap = CONFIGS[name]
    if key[0] == "decode":
        return False
    depth = {4: 1, 2: 2, 1: 3}[scale]
    last_q = max({32: 0, 64: 1, 128: 2}[c[0]] for c in cbs)
    if w.startswith("multiscale_encoder."):
        if ".in_conv." in w:
            return True
        j = int(w.split(".")[2])
        return j <= depth or last_q >= j - depth
    if w.startswith(("before_quant_group.", "quantize_group.")):     # quantize_group: z . E^T without the fused VQ
        return True
    if w.startswith("after_quant_group."):
        return {32: 0, 64: 1, 128: 2}[cbs[int(w.split(".")[1])][0]] < last_q
    assert w.startswith("decoder_group."), w
    return int(w.split(".")[1]) < last_q


def k_blocks(r):
    return (4 if r["upsample"] else r["k"] * r["k"]) * (r["Cin"] // 64)


def f8_form(r):
    """femasr_net's weight forms: the F8 packing exists for the generator's tensor-core 3x3 convs."""
    return r["k"] == 3 and r["Cin"] % 64 == 0 and r["Cout"] % 64 == 0 and not r["semantic"] and not r["sn"]


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_numerics_policy(built_lib, gemm_path):
    for name, key, t in all_traces(gemm_path):
        for r in t:
            at = where(name, key, r)
            if r["semantic"]:            # the VGG branch, conv_semantic, LPIPS: one pass, no F8, exact prologue
                assert not name.startswith("disc") and (r["w"].startswith(("vgg_feat_extractor.", "conv_semantic.")) or
                                                        name.startswith("lpips")), at
                assert r["slice_kb"] == 0 and not r["f8"] and r["prologue"] == "none", at
                continue
            assert not name.startswith("lpips"), at
            precise = expect_precise(name, key, r["w"])
            assert r["precise_region"] == precise, f"{at}: precise_region {r['precise_region']}, expected {precise}"
            assert r["sn"] == (name.startswith("disc") and r["w"] != "conv0.weight"), at
            if gemm_path == 0:
                continue
            if precise:
                assert not r["f8"] and r["prologue"] != "gn_fast", at
                assert r["slice_kb"] == (4 if k_blocks(r) > 4 else 0), f"{at}: slice_kb {r['slice_kb']}, {k_blocks(r)} k-blocks"
            else:
                want_f8 = f8_form(r) and r["prologue"] != "ln" and r["operand"] == "staged"
                assert r["f8"] == want_f8, f"{at}: f8 {r['f8']}, expected {want_f8}"
                assert r["slice_kb"] == 0, at
                assert r["prologue"] != "gn", f"{at}: exact SiLU behind the VQ"


# environment variables that once selected other numerics, each with a value that did so
FORMER_KNOBS = {"FEMASR_TC_PRECISE": "0", "FEMASR_FAST_SILU": "0", "FEMASR_VQ_FUSED": "0", "FEMASR_F8_CROSS": "0",
                "FEMASR_TC_SLICE_KB": "2", "FEMASR_SEM_SLICE_KB": "4"}


def sizing(gemm_path):
    """Every configuration's and head's plan table (tests/test_engine_plan.py: workspace bytes, FLOPs) and sizing traces."""
    L = lib.load()
    return ({name: plan(L, name, gemm_path) for name in CONFIGS}, {name: head_plan(L, name, gemm_path) for name in HEADS},
            {name: gen_traces(L, name, gemm_path) for name in CONFIGS},
            {name: head_traces(L, name, gemm_path) for name in HEADS})


@pytest.mark.parametrize("var", sorted(FORMER_KNOBS))
def test_numerics_ignore_the_environment(built_lib, monkeypatch, var):
    for v in FORMER_KNOBS:
        monkeypatch.delenv(v, raising=False)
    want = [sizing(gp) for gp in (0, 1)]
    monkeypatch.setenv(var, FORMER_KNOBS[var])
    for gp in (0, 1):
        assert sizing(gp) == want[gp], f"{var}={FORMER_KNOBS[var]} changes the gemm_path {gp} plan"


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_trace_is_repeatable_and_independent_of_taps_and_captures(built_lib, gemm_path):
    L = lib.load()
    for name in ("x4_e256", "x2_cb3", "hq_e512_sem"):
        h = create_gen(L, name, gemm_path)
        try:
            n, n2 = ctypes.c_size_t(), ctypes.c_size_t()
            sem = int(CONFIGS[name][2])
            B, H, W = 2, 96, 160
            assert L.femasr_net_workspace_bytes_sem(h, B, H, W, sem, ctypes.byref(n)) == 0
            t0 = trace(L, h)
            assert len(t0) > 20 and [r["ordinal"] for r in t0] == list(range(len(t0)))
            assert L.femasr_net_workspace_bytes_sem(h, B, H, W, sem, ctypes.byref(n2)) == 0
            assert trace(L, h) == t0 and n2.value == n.value
            stages = list(lib.TAP_STAGES) + (list(lib.SEMANTIC_TAP_STAGES) if sem else [])
            for s in stages:
                assert L.femasr_net_set_tap(h, s.encode(), ctypes.c_void_p(1 << 20), 1 << 40) == 0
            for o in range(len(t0)):
                for what in (b"x", b"y", b"res1", b"gn_partial", b"a_hi"):
                    assert L.femasr_net_set_conv_capture(h, o, what, ctypes.c_void_p(1 << 20), 1 << 40) == 0
            assert L.femasr_net_workspace_bytes_sem(h, B, H, W, sem, ctypes.byref(n2)) == 0
            # the in_conv tap adds the fp32 in_conv on gemm_path 1: a kernel of its own, not a conv of the trace
            assert trace(L, h) == t0
            assert gemm_path == 1 or n2.value == n.value
        finally:
            L.femasr_net_destroy(h)


def test_set_conv_capture_arguments(built_lib):
    L = lib.load()
    h = create_head(L, "disc_skip", 1)
    try:
        dst = ctypes.c_void_p(1 << 20)
        assert L.femasr_net_set_conv_capture(None, 0, b"x", dst, 4) == -1
        assert L.femasr_net_set_conv_capture(h, 0, None, dst, 4) == -1
        assert L.femasr_net_set_conv_capture(h, -1, b"x", dst, 4) == -1
        assert L.femasr_net_set_conv_capture(h, 0, b"w", dst, 4) == -1
        assert b"unknown operand" in L.femasr_last_error()
        for what in (b"x", b"a_hi", b"a_lo", b"pa", b"pb", b"res1", b"res2", b"y", b"o_hi", b"o_lo", b"gn_partial"):
            assert L.femasr_net_set_conv_capture(h, 3, what, dst, 4) == 0
            assert L.femasr_net_set_conv_capture(h, 3, what, None, 0) == 0
    finally:
        L.femasr_net_destroy(h)
