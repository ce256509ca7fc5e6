"""GPU: engines that share one device across streams and host threads.  Every engine keeps its weights in its own handle,
so its result depends on its own inputs and weights only, whatever runs beside it.

Each pair of engines gets different weights (other seeds, and the out_conv / conv9 heads negated or scaled against each
other), so a head that read the other engine's weights would miss its fp64 bar by orders of magnitude.  Every case
enqueues one fixed schedule and synchronises once; results are compared bitwise with each engine's solo result on the
default stream.  The engine-pair cases record device events around each stream's work from one common start event and
assert that the intervals overlap, so they cannot pass by running one stream after the other.

- ABI level: femasr_out_conv3x3_n (Cout 3 and 1, SIMT and mma) on two streams with two weight sets, 8 calls each.
- Engine pairs on both GEMM paths: two x4 generators; a generator and the discriminator (out_conv beside conv9); a
  generator and LPIPS alex, with PSNR / SSIM and a degradation blur on a third stream.
- A generator's captured forward_graph replayed on one stream while the discriminator runs eagerly on another.
- Two host threads, each with its own engine, stream and workspace; error messages stay per thread.
- Per-shape profile labels (FEMASR_PROFILE_DETAIL=1) from two threads at once, in a subprocess."""
import json
import os
import subprocess
import sys
import threading

import pytest
import torch
import torch.nn.functional as F

from femasr_b200 import lib as L
from femasr_b200.degrade import _Gpu, fspecial_gaussian
from femasr_b200.metrics import PSNR, SSIM
from tests import gpu_util as G
from tests.test_buffers_gpu import (check_head, disc_entry, gen_dec2_entry, lpips_entry, make_disc, make_gen, make_lpips,
                                    same_bits)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, H, W = 8, 128, 128            # an x4 forward of tens of milliseconds per stream


def rand(shape, seed, scale=1.0):
    return torch.rand(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def alloc(specs, dev):
    return {k: torch.empty(shape, dtype=dt, device=dev) for k, (dt, shape) in specs.items()}


def ptrs(outs):
    return {k: t.data_ptr() for k, t in outs.items()}


def solo(entry, dev):
    """The entry's result alone on the default stream (the second of two calls in a row)."""
    need, specs, launch = entry
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    for _ in range(2):
        outs = alloc(specs, dev)
        L.check(launch(ptrs(outs), ws.data_ptr(), need))
    torch.cuda.synchronize()
    return outs


def engine_call(entry, dev, calls):
    """Zero-argument closures, one per call, that launch `entry` into their own preallocated outputs and one shared
    workspace on the current stream.  Allocated on the current stream (the one the calls will run on)."""
    need, specs, launch = entry
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    outs = [alloc(specs, dev) for _ in range(calls)]

    def make(o):
        def call():
            L.check(launch(ptrs(o), ws.data_ptr(), need))
            return o
        return call
    return [make(o) for o in outs]


def run_streams(work, dev):
    """work: {name: [closure per call]}, each name on its own stream, the calls enqueued round-robin across the streams
    after one common start event.  Returns ({name: [result per call]}, {name: (begin ms, end ms)} from the start)."""
    streams = {k: torch.cuda.Stream(dev) for k in work}
    torch.cuda.synchronize()
    start = torch.cuda.Event(enable_timing=True)
    start.record()
    ev = {k: (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for k in work}
    for k, s in streams.items():
        s.wait_event(start)
        ev[k][0].record(s)
    res = {k: [] for k in work}
    for i in range(max(len(v) for v in work.values())):
        for k, calls in work.items():
            if i < len(calls):
                with torch.cuda.stream(streams[k]):
                    res[k].append(calls[i]())
    for k, s in streams.items():
        ev[k][1].record(s)
    torch.cuda.synchronize()
    return res, {k: (start.elapsed_time(b), start.elapsed_time(e)) for k, (b, e) in ev.items()}


def assert_overlap(spans, a, b, tag):
    (a0, a1), (b0, b1) = spans[a], spans[b]
    ov = min(a1, b1) - max(a0, b0)
    print(f"{tag}: {a} {a0:.2f}-{a1:.2f} ms, {b} {b0:.2f}-{b1:.2f} ms, overlap {ov:.2f} ms")
    assert ov > 0, f"{tag}: the streams' work did not overlap ({a} {a0:.2f}-{a1:.2f} ms, {b} {b0:.2f}-{b1:.2f} ms)"


# ------------------------------------------------------------------------------------------------ ABI level
@pytest.mark.parametrize("mma", [0, 1])
@pytest.mark.parametrize("co", [3, 1])
def test_out_conv_two_streams(cuda, co, mma):
    """8 calls per stream, alternating between two streams with their own weights, at 4x256x256 and a ragged 3x61x97:
    every output bitwise equal to the same call alone and within test_in_conv_out_conv's bars of fp64 conv2d."""
    shapes = ((4, 256, 256), (3, 61, 97))
    xs = [torch.randn(b, 64, h, w, generator=torch.Generator().manual_seed(40 + i)) * (1.5 if mma else 1.0)
          for i, (b, h, w) in enumerate(shapes)]
    wsets = []
    for s, sign in ((0, 1.0), (1, -4.0)):
        g = torch.Generator().manual_seed(50 + 10 * co + s)
        w, b = torch.randn(co, 64, 3, 3, generator=g) * 0.05 * sign, torch.randn(co, generator=g) * sign
        wsets.append((w, b, G.pack_weight(w.to(cuda)), b.to(cuda)))
    xg = [G.nhwc(x).to(cuda) for x in xs]
    lib = L.load()

    def launch(s, i, y):
        (b, h, w), (_w, _b, wp, bg) = shapes[i], wsets[s]
        L.check(lib.femasr_out_conv3x3_n(xg[i].data_ptr(), wp.data_ptr(), bg.data_ptr(), y.data_ptr(), b, h, w, 64, co,
                                         mma, G.S()))
        return y

    want, alone = {}, {}
    for s in range(2):
        for i, (b, h, w) in enumerate(shapes):
            wt, bt = wsets[s][:2]
            ref = F.conv2d(xg[i].permute(0, 3, 1, 2).double(), wt.to(cuda).double(), bt.to(cuda).double(), padding=1)
            want[s, i] = ref.cpu()
            alone[s, i] = launch(s, i, torch.empty(b, co, h, w, device=cuda))
            torch.cuda.synchronize()
    work = {}
    for s in range(2):
        work[s] = []
        for k in range(8):
            b, h, w = shapes[k % 2]
            y = torch.full((b, co, h, w), float("nan"), device=cuda)
            work[s].append(lambda s=s, i=k % 2, y=y: launch(s, i, y))
    res, _spans = run_streams(work, cuda)
    for s in range(2):
        for k, y in enumerate(res[s]):
            tag = f"out_conv Cout {co} mma={mma} stream {s} call {k}"
            same_bits(y, alone[s, k % 2], tag + " vs alone")
            ref = want[s, k % 2]
            err = (y.cpu().double() - ref).abs().max().item()
            bar = 5e-6 * ref.abs().max().item() if mma else 2e-5 * max(1.0, ref.abs().max().item())
            assert err <= bar, f"{tag}: max-abs {err:.3e} vs fp64 > {bar:.1e}"


# ------------------------------------------------------------------------------------------------ engine pairs
def x_in(seed):
    return rand((B, 3, H, W), seed)


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_two_generators(cuda, gemm_path):
    ga = make_gen("x4_e256", gemm_path, cuda)
    gb = make_gen("x4_e256", gemm_path, cuda, seed=93, head=-1.0)
    ea, eb = gen_dec2_entry(ga, x_in(1).to(cuda)), gen_dec2_entry(gb, x_in(2).to(cuda))
    want = {"a": solo(ea, cuda), "b": solo(eb, cuda)}
    work = {}
    for k, e in (("a", ea), ("b", eb)):
        work[k] = engine_call(e, cuda, 2)
    res, spans = run_streams(work, cuda)
    assert_overlap(spans, "a", "b", f"gp{gemm_path} two generators")
    for k, net in (("a", ga), ("b", gb)):
        for i, got in enumerate(res[k]):
            for o in got:
                same_bits(got[o], want[k][o], f"gp{gemm_path} generator {k} call {i} {o}")
            check_head(net, got["y"], got["tap:dec2"], f"gp{gemm_path} generator {k} call {i}")
    for e in (ga, gb):
        e.close()


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_generator_and_discriminator(cuda, gemm_path):
    """out_conv (Cout 3) on one stream, the discriminator's conv9 (Cout 1) on the other."""
    gen = make_gen("x4_e256", gemm_path, cuda)
    d = make_disc(1, gemm_path, cuda, seed=94, head=-8.0)
    ge = gen_dec2_entry(gen, x_in(3).to(cuda))
    de = disc_entry(d, (rand((B, 3, 2 * H, 2 * W), 4) * 2 - 1).to(cuda))
    want = {"gen": solo(ge, cuda), "disc": solo(de, cuda)}
    res, spans = run_streams({"gen": engine_call(ge, cuda, 2), "disc": engine_call(de, cuda, 2)}, cuda)
    assert_overlap(spans, "gen", "disc", f"gp{gemm_path} generator + discriminator")
    for k in ("gen", "disc"):
        for i, got in enumerate(res[k]):
            for o in got:
                same_bits(got[o], want[k][o], f"gp{gemm_path} {k} call {i} {o}")
            if k == "gen":
                check_head(gen, got["y"], got["tap:dec2"], f"gp{gemm_path} generator call {i}")
    gen.close()
    d.close()


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_generator_lpips_and_controls(cuda, gemm_path):
    """A generator beside LPIPS alex, with PSNR, SSIM and a degradation blur on a third stream: none of them holds state
    the others could see."""
    gen = make_gen("x4_e256", gemm_path, cuda, seed=95, head=2.0)
    m = make_lpips("alex", gemm_path, cuda, seed=96)
    ge = gen_dec2_entry(gen, x_in(5).to(cuda))
    a, b = rand((B, 3, 4 * H, 4 * W), 6).to(cuda), rand((B, 3, 4 * H, 4 * W), 7).to(cuda)
    me = lpips_entry(m, a, b, 1)
    img = rand((4 * H, 4 * W, 3), 8).to(cuda)
    blur = fspecial_gaussian(7, 1.6)

    def controls():
        return {"psnr": PSNR()(a, b), "ssim": SSIM()(a, b), "blur": _Gpu(cuda).conv(img, blur, 1, True)}
    want = {"gen": solo(ge, cuda), "lpips": solo(me, cuda), "ctl": controls()}
    torch.cuda.synchronize()
    res, spans = run_streams({"gen": engine_call(ge, cuda, 2), "lpips": engine_call(me, cuda, 2),
                              "ctl": [controls, controls]}, cuda)
    assert_overlap(spans, "gen", "lpips", f"gp{gemm_path} generator + LPIPS")
    assert_overlap(spans, "gen", "ctl", f"gp{gemm_path} generator + metrics / degradation")
    for k in ("gen", "lpips", "ctl"):
        for i, got in enumerate(res[k]):
            for o in got:
                same_bits(got[o], want[k][o], f"gp{gemm_path} {k} call {i} {o}")
    for i, got in enumerate(res["gen"]):
        check_head(gen, got["y"], got["tap:dec2"], f"gp{gemm_path} generator call {i}")
    gen.close()
    m.close()


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_graph_replay_beside_discriminator(cuda, gemm_path):
    """A generator's captured forward_graph replayed on one stream while the discriminator runs eagerly on another."""
    net = make_gen("x4_e256", gemm_path, cuda)
    net.use_graph = True
    d = make_disc(1, gemm_path, cuda, seed=97, head=-8.0)
    x = x_in(9).to(cuda)
    dx = (rand((B, 3, 2 * H, 2 * W), 10) * 2 - 1).to(cuda)
    want = [t.clone() for t in net.forward(x)]
    dwant = d.forward(dx).clone()
    net.forward_graph(x)
    net.forward_graph(x)                           # second sighting: captured
    assert net.last_from_graph
    torch.cuda.synchronize()
    res, spans = run_streams({"graph": [lambda: net.forward_graph(x)], "disc": [lambda: d.forward(dx), lambda: d.forward(dx)]},
                             cuda)
    assert net.last_from_graph
    (a0, a1), (b0, b1) = spans["graph"], spans["disc"]
    print(f"gp{gemm_path} graph replay + discriminator: overlap {min(a1, b1) - max(a0, b0):.2f} ms")
    for got, w_, k in zip(res["graph"][0], want, ("y", "loss", "idx")):
        same_bits(got, w_, f"gp{gemm_path} replay {k}")
    for i, got in enumerate(res["disc"]):
        same_bits(got, dwant, f"gp{gemm_path} discriminator call {i}")
    net.release_graphs()
    net.close()
    d.close()


# ------------------------------------------------------------------------------------------------ host threads
REFUSED = {0: b"must be even", 1: b"set_poison"}


def threaded(engines, dev):
    """engines: two (handle, entry); each thread owns its engine, stream and workspace and runs 3 forwards after a
    common barrier.  Between them thread 0 makes a refused forward (odd H) while thread 1 runs, then thread 1 a refused
    set_poison while thread 0 runs.  Returns each thread's results; raises the first failure of either thread."""
    barrier = threading.Barrier(2)
    res, errors = [None, None], []
    dummy = torch.zeros(64, device=dev)           # the refused call's operands: never read
    lib = L.load()

    def body(t):
        try:
            h, entry = engines[t]
            with torch.cuda.stream(torch.cuda.Stream(dev)):
                calls = engine_call(entry, dev, 3)
                barrier.wait()
                out = [calls[0]()]
                barrier.wait()
                if t == 0:
                    d = dummy.data_ptr()
                    assert lib.femasr_net_forward(h, d, d, None, None, 1, 127, 128, d, dummy.numel() * 4, G.S()) == -1
                    assert REFUSED[0] in lib.femasr_last_error()
                else:
                    out.append(calls[1]())
                barrier.wait()
                if t == 1:
                    assert lib.femasr_net_set_poison(h, 256) == -1
                    assert REFUSED[1] in lib.femasr_last_error()
                else:
                    out.append(calls[1]())
                barrier.wait()
                out.append(calls[2]())
                torch.cuda.current_stream().synchronize()
            msg = lib.femasr_last_error()
            assert REFUSED[t] in msg and REFUSED[1 - t] not in msg, f"thread {t} last_error: {msg!r}"
            res[t] = out
        except BaseException as e:                # noqa: BLE001  (re-raised on the main thread)
            errors.append(e)
            barrier.abort()

    threads = [threading.Thread(target=body, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    if errors:
        raise errors[0]
    return res


@pytest.mark.parametrize("other", ["disc", "gen"])
def test_two_host_threads(cuda, other):
    """A gemm_path 1 generator in one thread, a gemm_path 0 discriminator or generator in the other."""
    ga = make_gen("x4_e256", 1, cuda)
    ea = gen_dec2_entry(ga, x_in(11).to(cuda))
    if other == "disc":
        ob = make_disc(1, 0, cuda, seed=98, head=-8.0)
        eb = disc_entry(ob, (rand((B, 3, 2 * H, 2 * W), 12) * 2 - 1).to(cuda))
    else:
        ob = make_gen("x4_e256", 0, cuda, seed=99, head=-1.0)
        eb = gen_dec2_entry(ob, x_in(12).to(cuda))
    want = [solo(ea, cuda), solo(eb, cuda)]
    res = threaded([(ga._h, ea), (ob._h, eb)], cuda)
    for t, net in enumerate((ga, ob)):
        assert len(res[t]) == 3
        for i, got in enumerate(res[t]):
            for o in got:
                same_bits(got[o], want[t][o], f"thread {t} ({other}) forward {i} {o}")
            if "tap:dec2" in got:
                check_head(net, got["y"], got["tap:dec2"], f"thread {t} forward {i}")
    ga.close()
    ob.close()


PROFILE_SCRIPT = r"""
import json, sys, threading
import torch
sys.path.insert(0, sys.argv[1])
from tests.test_buffers_gpu import make_gen
dev = torch.device("cuda", 0)
nets = [make_gen("x4_e256", 1, dev), make_gen("x4_e256", 1, dev, seed=93, head=-1.0)]
x = torch.rand(2, 3, 64, 64, generator=torch.Generator().manual_seed(13)).to(dev)
barrier, out, errors = threading.Barrier(2), [None, None], []
def body(t):
    try:
        with torch.cuda.stream(torch.cuda.Stream(dev)):
            nets[t].set_profile(True)
            barrier.wait()
            for _ in range(3):
                nets[t].forward(x)
            torch.cuda.current_stream().synchronize()
            out[t] = nets[t].profile()
            nets[t].set_profile(False)
    except BaseException as e:
        errors.append(repr(e))
        barrier.abort()
threads = [threading.Thread(target=body, args=(t,)) for t in range(2)]
for th in threads: th.start()
for th in threads: th.join()
print(json.dumps({"errors": errors, "profiles": out}))
"""


def test_profile_labels_from_two_threads(cuda):
    """FEMASR_PROFILE_DETAIL=1 (read once per process, so in a subprocess) with profiling on for two generators driven
    from two threads at once: both profiles parse and carry the per-shape tc_igemm labels."""
    env = dict(os.environ, FEMASR_PROFILE_DETAIL="1", FEMASR_CUDA_GRAPH="0")
    r = subprocess.run([sys.executable, "-c", PROFILE_SCRIPT, ROOT], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, f"subprocess failed ({r.returncode}):\n{r.stderr[-3000:]}"
    doc = json.loads(r.stdout.strip().splitlines()[-1])
    assert not doc["errors"], doc["errors"]
    for t, prof in enumerate(doc["profiles"]):
        labels = [k for k in prof if k.startswith("tc_igemm:k")]
        assert labels, f"thread {t}: no per-shape tc_igemm labels in {sorted(prof)[:8]}"
        assert all(v["launches"] % 3 == 0 for k, v in prof.items() if k in labels), f"thread {t}: {prof}"
