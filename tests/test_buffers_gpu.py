"""GPU: the engine's memory contract.  An engine result depends on its inputs and weights only, and nothing is written
outside the buffers a call was given.

- Poison matrix: every configuration of tests/test_engine_plan.py on both GEMM paths, at the smallest legal input and at a
  B = 2 non-square input whose Swin map is 24 x 40 (ragged against the GEMMs' 128-pixel tiles), plus the discriminator
  and both LPIPS nets.  Every entry point runs with femasr_net_set_poison off and at 0x00, 0x41 (finite in fp32, fp16
  and e4m3) and 0xFF (NaN in all three, -1 in int64): every workspace block a run hands out starts as that byte, so a
  kernel that reads an element it did not write in this call (a K-padding column, a partial row, a masked tile lane
  multiplied by zero) changes the result.  The results must be bitwise equal across the four runs.
- Guard bands: the poisoned runs get the workspace as exactly the reported bytes at offsets 0, 16 and 255 into a buffer
  with 1 MiB of 0xA5 on each side, and every output (and tap) inside its own guards, prefilled with a NaN pattern.
  Afterwards the guards are intact and no output element still holds the prefill.
- Sequences on one stream: shapes and entry points alternating on one handle and workspace; generator, discriminator and
  LPIPS interleaved (they share the out_conv kernels' library-global weights); a captured graph replayed around them.
- The kernels outside the arena (test(), test_tile(), sr_uint8() and out_conv's writes into the caller's y) against
  exact references, inside guard bands."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from basicsr.utils import img2tensor, tensor2img
from femasr_b200 import lib as L
from femasr_b200.net import NativeDisc, NativeLPIPS, NativeNet
from femasr_b200.spec import random_disc_state_dict, random_lpips_state_dict, random_state_dict
from tests import gpu_util as G
from tests.test_engine_plan import CONFIGS

pytestmark = pytest.mark.gpu

GUARD = 1 << 20
GUARD_BYTE = 0xA5
NAN_FILL = 0x7FA5A5A5                      # an fp32 NaN bit pattern no kernel produces
POISONS = (0x00, 0x41, 0xFF)
WS_OFFSETS = (0, 16, 255)                  # where the poisoned runs' workspace starts: both sides of the 256-byte round-up
DIV = {4: 2, 2: 4, 1: 8}                   # input size / latent size
SMALL = {4: (1, 16, 16), 2: (1, 32, 32), 1: (1, 8, 8)}
RAGGED = {4: (2, 48, 80), 2: (2, 96, 160), 1: (2, 192, 320)}   # Swin map (or HQ latent x 8) 24 x 40


class Guarded:
    """`nbytes` of device memory at `offset` bytes past GUARD bytes of 0xA5, with GUARD more after it."""

    def __init__(self, nbytes, dev, offset=0):
        self.lo, self.n = GUARD + offset, nbytes
        self.raw = torch.full((2 * GUARD + offset + nbytes,), GUARD_BYTE, dtype=torch.uint8, device=dev)

    def ptr(self):
        return self.raw.data_ptr() + self.lo

    def view(self, dtype, shape):
        return self.raw[self.lo:self.lo + self.n].view(dtype).view(shape)

    def check(self, what):
        bad = int((self.raw[:self.lo] != GUARD_BYTE).sum()) + int((self.raw[self.lo + self.n:] != GUARD_BYTE).sum())
        assert bad == 0, f"{what}: {bad} guard bytes changed"


def guarded_out(dtype, shape, dev):
    """A guarded output prefilled with NAN_FILL (fp32) or 0xA5 bytes (int64)."""
    g = Guarded(math.prod(shape) * torch.empty((), dtype=dtype).element_size(), dev)
    if dtype == torch.float32:
        g.view(torch.int32, shape).fill_(NAN_FILL)
    return g


def bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def prefilled(t):
    fill = NAN_FILL if t.dtype == torch.float32 else int(np.array([GUARD_BYTE] * 8, np.uint8).view(np.int64)[0])
    return int((bits(t) == fill).sum())


def same_bits(got, want, what):
    if not torch.equal(bits(got), bits(want)):
        diff = int((bits(got) != bits(want)).sum())
        raise AssertionError(f"{what}: {diff} of {want.numel()} elements differ bitwise")


def poison_matrix(what, handle, need, specs, launch, dev):
    """Runs launch(ptrs, ws_ptr, ws_bytes) with poison off on plain buffers, then at each POISONS byte on guarded ones
    (workspace of exactly `need` bytes at WS_OFFSETS); every result bitwise equal to the first.  specs: {name: (dtype,
    shape)}.  Returns the first run's outputs."""
    lib = L.load()
    L.check(lib.femasr_net_set_poison(handle, -1))
    plain = {k: torch.empty(shape, dtype=dt, device=dev) for k, (dt, shape) in specs.items()}
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    L.check(launch({k: t.data_ptr() for k, t in plain.items()}, ws.data_ptr(), need))
    torch.cuda.synchronize()
    for k, t in plain.items():
        if t.dtype == torch.float32:
            assert bool(torch.isfinite(t).all()), f"{what}: {k} not finite with poison off"
    for byte, off in zip(POISONS, WS_OFFSETS):
        gws = Guarded(need, dev, off)
        outs = {k: guarded_out(dt, shape, dev) for k, (dt, shape) in specs.items()}
        L.check(lib.femasr_net_set_poison(handle, byte))
        try:
            L.check(launch({k: g.ptr() for k, g in outs.items()}, gws.ptr(), need))
        finally:
            L.check(lib.femasr_net_set_poison(handle, -1))
        torch.cuda.synchronize()
        tag = f"{what} poison 0x{byte:02X} ws+{off}"
        gws.check(tag + " workspace")
        for k, g in outs.items():
            g.check(f"{tag} {k}")
            got = g.view(plain[k].dtype, specs[k][1])
            assert prefilled(got) == 0, f"{tag} {k}: {prefilled(got)} elements never written"
            same_bits(got, plain[k], f"{tag} {k}")
    return plain


# ------------------------------------------------------------------------------------------------ generator
_SD = {}


def make_gen(name, gemm_path, dev):
    scale, cbs, sem, _tap = CONFIGS[name]
    key = (scale, str(cbs), sem)
    if key not in _SD:
        if len(_SD) > 1:
            _SD.clear()
        _SD[key] = random_state_dict(scale, cbs[0][2], seed=90, init="perturbed", codebooks=cbs, semantic=sem)
    net = NativeNet(scale, cbs[0][1], cbs[0][2], gemm_path=gemm_path, codebooks=cbs, use_semantic_loss=sem)
    net.sd = _SD[key]
    net.load_state_dict(net.sd, dev)
    net.use_graph = False
    return net


def gen_need(net, B, H, W, sem):
    need = C.c_size_t()
    L.check(net.lib.femasr_net_workspace_bytes_sem(net._h, B, H, W, int(sem), C.byref(need)))
    return need.value


def sem_legal(net, B, H, W):
    need = C.c_size_t()
    return net.use_semantic_loss and net.lib.femasr_net_workspace_bytes_sem(net._h, B, H, W, 1, C.byref(need)) == 0


def gen_taps(net, B, H, W, sem):
    """The taps a forward of this net writes, with their shapes."""
    shapes = net.tap_shapes(B, H, W)
    skip = set() if sem else {"vgg", "semantic"}
    if net.scale == 1:
        skip |= {"up1", "up2"}
    return {k: v for k, v in shapes.items() if k not in skip}


def gen_forward(net, x, B, H, W, sem, gt=None, taps=()):
    """(specs, launch) of forward_sem with indices and loss (and the semantic loss, gt_indices, taps when given)."""
    s = net.scale
    nidx = sum(math.prod(sh) for sh in net.index_shapes(B, H, W))
    specs = {"y": (torch.float32, (B, 3, H * s, W * s)), "idx": (torch.int64, (nidx,)), "loss": (torch.float32, ())}
    if sem:
        specs["sem"] = (torch.float32, ())
    tshape = gen_taps(net, B, H, W, sem) if taps else {}
    specs.update({"tap:" + k: (torch.float32, v) for k, v in tshape.items()})

    def launch(p, ws, n):
        for k in tshape:
            L.check(net.lib.femasr_net_set_tap(net._h, k.encode(), p["tap:" + k], math.prod(tshape[k])))
        try:
            return net.lib.femasr_net_forward_sem(net._h, x.data_ptr(), p["y"], p["idx"], p["loss"], G.p(gt),
                                                  p.get("sem"), B, H, W, ws, n, G.S())
        finally:
            for k in tshape:
                net.lib.femasr_net_set_tap(net._h, k.encode(), None, 0)
    return specs, launch


@pytest.mark.parametrize("gemm_path", [0, 1])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_generator_poison_and_guards(cuda, name, gemm_path):
    net = make_gen(name, gemm_path, cuda)
    tag0 = f"{name}/gp{gemm_path}"
    for shape in (SMALL[net.scale], RAGGED[net.scale]):
        B, H, W = shape
        tag = f"{tag0} {B}x{H}x{W}"
        x = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(B * H + W)).to(cuda)
        sem = sem_legal(net, B, H, W)
        assert sem == (name == "hq_e512_sem")
        need = gen_need(net, B, H, W, sem)
        specs, launch = gen_forward(net, x, B, H, W, sem)
        base = poison_matrix(tag + " forward", net._h, need, specs, launch, cuda)
        idx = base["idx"]
        if net.scale != 1:   # the LQ stage's gt_indices loss
            specs, launch = gen_forward(net, x, B, H, W, sem, gt=idx)
            poison_matrix(tag + " forward_gt", net._h, need, specs, launch, cuda)
        # every tap registered: another arena plan (in_conv's tap adds the fp32 in_conv on gemm_path 1), same results
        specs, launch = gen_forward(net, x, B, H, W, sem, taps=True)
        for k in specs:
            if k.startswith("tap:"):
                L.check(net.lib.femasr_net_set_tap(net._h, k[4:].encode(), C.c_void_p(1 << 20), 1 << 40))
        try:
            tneed = gen_need(net, B, H, W, sem)
        finally:
            for k in specs:
                if k.startswith("tap:"):
                    net.lib.femasr_net_set_tap(net._h, k[4:].encode(), None, 0)
        tapped = poison_matrix(tag + " taps", net._h, tneed, specs, launch, cuda)
        for k in base:
            same_bits(tapped[k], base[k], f"{tag} taps vs untapped {k}")
        # decode_indices on codebook 0's indices
        h, w = H // DIV[net.scale], W // DIV[net.scale]
        idx0 = idx[:B * h * w].contiguous()
        dneed = C.c_size_t()
        L.check(net.lib.femasr_net_decode_workspace_bytes(net._h, B, h, w, C.byref(dneed)))
        poison_matrix(tag + " decode", net._h, dneed.value, {"y": (torch.float32, (B, 3, 8 * h, 8 * w))},
                            lambda p, ws, n: net.lib.femasr_net_decode_indices(net._h, idx0.data_ptr(), p["y"], B, h, w,
                                                                               ws, n, G.S()), cuda)
    net.close()


# ------------------------------------------------------------------------------------------------ discriminator, LPIPS
def make_disc(skip, gemm_path, dev, seed=91):
    d = NativeDisc(skip_connection=bool(skip), gemm_path=gemm_path)
    d.load_state_dict(random_disc_state_dict(seed), dev)
    return d


def disc_entry(d, x):
    B, _, H, W = x.shape
    need = C.c_size_t()
    L.check(d.lib.femasr_disc_workspace_bytes(d._h, B, H, W, C.byref(need)))
    return need.value, {"y": (torch.float32, (B, 1, H, W))}, \
        lambda p, ws, n: d.lib.femasr_disc_forward(d._h, x.data_ptr(), p["y"], B, H, W, ws, n, G.S())


def make_lpips(net, gemm_path, dev, seed=92):
    m = NativeLPIPS(net, gemm_path=gemm_path)
    m.load_state_dict(random_lpips_state_dict(net, seed), dev)
    return m


def lpips_entry(m, x0, x1, normalize):
    B, _, H, W = x0.shape
    need = C.c_size_t()
    L.check(m.lib.femasr_lpips_workspace_bytes(m._h, B, H, W, C.byref(need)))
    return need.value, {"d": (torch.float32, (B,)), "r": (torch.float32, (5, B))}, \
        lambda p, ws, n: m.lib.femasr_lpips_forward(m._h, x0.data_ptr(), x1.data_ptr(), p["d"], p["r"], B, H, W,
                                                     normalize, ws, n, G.S())


@pytest.mark.parametrize("gemm_path", [0, 1])
@pytest.mark.parametrize("skip", [1, 0])
def test_disc_poison_and_guards(cuda, skip, gemm_path):
    d = make_disc(skip, gemm_path, cuda)
    for (B, H, W) in ((1, 8, 8), (2, 48, 80)):
        x = (torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(H + W)) * 2 - 1).to(cuda)
        need, specs, launch = disc_entry(d, x)
        poison_matrix(f"disc skip {skip}/gp{gemm_path} {B}x{H}x{W}", d._h, need, specs, launch, cuda)
    d.close()


@pytest.mark.parametrize("gemm_path", [0, 1])
@pytest.mark.parametrize("net", ["alex", "vgg"])
def test_lpips_poison_and_guards(cuda, net, gemm_path):
    m = make_lpips(net, gemm_path, cuda)
    shapes = ((1, 31, 31), (3, 67, 93)) if net == "alex" else ((1, 16, 16), (3, 48, 80))
    for (B, H, W) in shapes:
        g = torch.Generator().manual_seed(B + H + W)
        x0, x1 = torch.rand(B, 3, H, W, generator=g).to(cuda), torch.rand(B, 3, H, W, generator=g).to(cuda)
        for normalize in (0, 1):
            need, specs, launch = lpips_entry(m, x0, x1, normalize)
            poison_matrix(f"lpips {net}/gp{gemm_path} {B}x{H}x{W} normalize {normalize}", m._h, need, specs, launch, cuda)
    m.close()


# ------------------------------------------------------------------------------------------------ sequences on one stream
def run_entry(need, specs, launch, dev, ws=None):
    outs = {k: torch.empty(shape, dtype=dt, device=dev) for k, (dt, shape) in specs.items()}
    if ws is None:
        ws = torch.empty(need, dtype=torch.uint8, device=dev)
    assert ws.numel() >= need
    L.check(launch({k: t.data_ptr() for k, t in outs.items()}, ws.data_ptr(), ws.numel()))
    return outs


def check_head(net, y, dec2, tag):
    """y against out_conv in fp64 on the dec2 tap: a reference that does not go through the library-global out_conv
    weights (bars of tests/test_ops_gpu.py::test_in_conv_out_conv)."""
    sd = net.sd
    want = F.conv2d(G.nchw(dec2).double().cpu(), sd["out_conv.weight"].double(), sd["out_conv.bias"].double(), padding=1)
    err = (y.double().cpu() - want).abs().max().item()
    bar = 5e-6 * want.abs().max().item() if net.cfg.gemm_path == 1 else 2e-5 * max(1.0, want.abs().max().item())
    assert err <= bar, f"{tag}: out_conv vs fp64 max-abs {err:.3e} > {bar:.1e}"


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_sequences_one_handle(cuda, gemm_path):
    """Shape A -> B -> A and forward -> decode_indices -> forward on one handle and one workspace equal each call's solo
    result (a fresh handle and workspace)."""
    name = "x4_cb2"
    net, solo = make_gen(name, gemm_path, cuda), make_gen(name, gemm_path, cuda)
    shapes = [SMALL[4], RAGGED[4]]
    xs = {s: torch.rand(s[0], 3, s[1], s[2], generator=torch.Generator().manual_seed(sum(s))).to(cuda) for s in shapes}
    entries, want = {}, {}
    for s in shapes:
        B, H, W = s
        entries[s] = (gen_need(net, B, H, W, False),) + gen_forward(net, xs[s], B, H, W, False)
        sneed = gen_need(solo, B, H, W, False)
        want[s] = run_entry(sneed, *gen_forward(solo, xs[s], B, H, W, False), cuda)
    B, H, W = shapes[0]
    h, w = H // 2, W // 2
    idx0 = want[shapes[0]]["idx"][:B * h * w].contiguous()
    dneed = C.c_size_t()
    L.check(net.lib.femasr_net_decode_workspace_bytes(net._h, B, h, w, C.byref(dneed)))
    dec_specs = {"y": (torch.float32, (B, 3, 8 * h, 8 * w))}
    dec = lambda hd: (lambda p, ws, n: hd.lib.femasr_net_decode_indices(hd._h, idx0.data_ptr(), p["y"], B, h, w, ws, n,
                                                                        G.S()))
    want_dec = run_entry(dneed.value, dec_specs, dec(solo), cuda)
    ws = torch.empty(max([e[0] for e in entries.values()] + [dneed.value]), dtype=torch.uint8, device=cuda)
    ws.fill_(0xFF)
    order = [shapes[0], shapes[1], shapes[0], "decode", shapes[0], "decode", shapes[1]]
    for step, s in enumerate(order):
        if s == "decode":
            got = run_entry(dneed.value, dec_specs, dec(net), cuda, ws)
            same_bits(got["y"], want_dec["y"], f"gp{gemm_path} step {step} decode_indices")
            continue
        got = run_entry(*entries[s], cuda, ws)
        for k in got:
            same_bits(got[k], want[s][k], f"gp{gemm_path} step {step} {s} {k}")
    net.close()
    solo.close()


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_engines_interleaved(cuda, gemm_path):
    """Generator -> discriminator -> generator -> LPIPS -> generator on one stream: each result equals that engine's
    solo result, and the generator's y equals out_conv of its dec2 tap in fp64.  The generator's out_conv (Cout 3) and
    the discriminator's conv9 (Cout 1) share the SIMT kernel's __constant__ weights (gemm_path 0) and the mma kernel's
    global B fragments (gemm_path 1), both refreshed in stream order on every call."""
    gen = make_gen("x4_e256", gemm_path, cuda)
    d = make_disc(1, gemm_path, cuda)
    m = make_lpips("vgg", gemm_path, cuda)
    B, H, W = RAGGED[4]
    x = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(5)).to(cuda)
    gspecs, glaunch = gen_forward(gen, x, B, H, W, False)
    gspecs["tap:dec2"] = (torch.float32, gen.tap_shapes(B, H, W)["dec2"])
    tshape = gspecs["tap:dec2"][1]

    def glaunch_tap(p, ws, n):
        L.check(gen.lib.femasr_net_set_tap(gen._h, b"dec2", p["tap:dec2"], math.prod(tshape)))
        try:
            return glaunch(p, ws, n)
        finally:
            gen.lib.femasr_net_set_tap(gen._h, b"dec2", None, 0)
    gentry = (gen_need(gen, B, H, W, False), gspecs, glaunch_tap)
    dentry = disc_entry(d, (x * 2 - 1).contiguous())
    x1 = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(6)).to(cuda)
    mentry = lpips_entry(m, x, x1, 1)
    solo = {}
    for k, e in (("gen", gentry), ("disc", dentry), ("lpips", mentry)):
        run_entry(*e, cuda)
        solo[k] = run_entry(*e, cuda)                    # the second of two calls in a row
    check_head(gen, solo["gen"]["y"], solo["gen"]["tap:dec2"], f"gp{gemm_path} solo generator")
    for step, k in enumerate(("gen", "disc", "gen", "lpips", "gen", "disc", "disc", "gen")):
        got = run_entry(*{"gen": gentry, "disc": dentry, "lpips": mentry}[k], cuda)
        for o in got:
            same_bits(got[o], solo[k][o], f"gp{gemm_path} step {step} {k} {o}")
        if k == "gen":
            check_head(gen, got["y"], got["tap:dec2"], f"gp{gemm_path} step {step} generator")
    for e in (gen, d, m):
        e.close()


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_graph_replay_around_other_engines(cuda, gemm_path):
    """forward_graph captured with poison on (second sighting of the shape), the discriminator run eagerly in between,
    and the graph's pinned workspace filled with 0xFF between replays: every replay equals the eager forward."""
    net = make_gen("x4_e256", gemm_path, cuda)
    net.use_graph = True
    d = make_disc(1, gemm_path, cuda)
    B, H, W = RAGGED[4]
    x = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(7)).to(cuda)
    y, loss, idx = net.forward(x)
    want = (y.clone(), loss.clone(), idx.clone())
    dx = (x * 2 - 1).contiguous()
    dwant = d.forward(dx).clone()

    def same(outs, what):
        for a, b, k in zip(outs, want, ("y", "loss", "idx")):
            same_bits(a, b, f"gp{gemm_path} {what} {k}")
    L.check(net.lib.femasr_net_set_poison(net._h, 0x41))
    try:
        same(net.forward_graph(x), "first sighting (eager)")
        assert not net.last_from_graph
        same(net.forward_graph(x), "capture + first replay")
        assert net.last_from_graph
    finally:
        L.check(net.lib.femasr_net_set_poison(net._h, -1))
    ent = net._graphs[tuple(x.shape)]
    for step in range(3):
        same_bits(d.forward(dx), dwant, f"gp{gemm_path} disc between replays {step}")
        ent["ws"].fill_(0xFF)
        same(net.forward_graph(x), f"replay {step}")
        assert net.last_from_graph
    net.release_graphs()
    net.close()
    d.close()


# ------------------------------------------------------------------------------------------------ kernels outside the arena
def fetch(g, dtype, shape, what):
    torch.cuda.synchronize()
    g.check(what)
    return g.view(dtype, shape)


def flip_pad_ref(x, hp, wp):
    h, w = x.shape[2:]
    x = torch.cat([x, x.flip(2)], 2)[:, :, :hp]
    return torch.cat([x, x.flip(3)], 3)[:, :, :, :wp]


def test_flip_pad(cuda):
    lib = L.load()
    B, Cc = 2, 3
    for h, w in ((1, 1), (1, 5), (2, 3), (5, 1), (7, 12)):
        x = torch.randn(B, Cc, h, w, generator=torch.Generator().manual_seed(h * 31 + w)).to(cuda)
        for hp in range(h, 2 * h + 1):
            for wp in sorted({w, w + (w + 1) // 2, 2 * w}):
                g = guarded_out(torch.float32, (B, Cc, hp, wp), cuda)
                L.check(lib.femasr_flip_pad(x.data_ptr(), g.ptr(), B, Cc, h, w, hp, wp, G.S()))
                got = fetch(g, torch.float32, (B, Cc, hp, wp), f"flip_pad {h}x{w} -> {hp}x{wp}")
                same_bits(got, flip_pad_ref(x, hp, wp), f"flip_pad {h}x{w} -> {hp}x{wp}")
        assert lib.femasr_flip_pad(x.data_ptr(), x.data_ptr(), B, Cc, h, w, 2 * h + 1, w, G.S()) == -1


def test_copy_window(cuda):
    """Ragged windows touching each edge of the source and of the destination; the rest of the destination is the
    caller's and must keep its contents."""
    lib = L.load()
    B, Cc, sh, sw, dh, dw = 2, 3, 13, 17, 11, 19
    src = torch.randn(B, Cc, sh, sw, generator=torch.Generator().manual_seed(1)).to(cuda)
    old = torch.randn(B, Cc, dh, dw, generator=torch.Generator().manual_seed(2)).to(cuda)
    for (sy, sx, dy, dx, ch, cw) in ((0, 0, 0, 0, 11, 17), (2, 0, 0, 2, 11, 17), (12, 16, 10, 18, 1, 1),
                                     (0, 16, 10, 0, 1, 1), (0, 5, 3, 0, 8, 1), (5, 0, 0, 1, 1, 17),
                                     (1, 3, 4, 2, 7, 13), (2, 1, 0, 6, 11, 13)):
        g = Guarded(old.numel() * 4, cuda)
        g.view(torch.float32, old.shape).copy_(old)
        L.check(lib.femasr_copy_window(src.data_ptr(), g.ptr(), B, Cc, sh, sw, dh, dw, sy, sx, dy, dx, ch, cw, G.S()))
        want = old.clone()
        want[:, :, dy:dy + ch, dx:dx + cw] = src[:, :, sy:sy + ch, sx:sx + cw]
        tag = f"copy_window {(sy, sx, dy, dx, ch, cw)}"
        same_bits(fetch(g, torch.float32, old.shape, tag), want, tag)


def test_u8_to_input(cuda):
    """Every byte value in every channel, through the maximal reflection: bit for bit img2tensor(img) / 255. then
    test()'s flip pad."""
    lib = L.load()
    rng = np.random.default_rng(3)
    for (B, h, w, hp, wp) in ((2, 16, 16, 32, 32), (3, 5, 7, 10, 14), (1, 1, 1, 2, 2), (2, 9, 4, 9, 8)):
        imgs = rng.integers(0, 256, (B, h, w, 3), dtype=np.uint8)
        if h * w == 256:
            for b in range(B):
                for c in range(3):
                    imgs[b, :, :, c] = rng.permutation(256).astype(np.uint8).reshape(h, w)
        want = torch.stack([img2tensor(im) / 255. for im in imgs])
        want = flip_pad_ref(want, hp, wp)
        g = guarded_out(torch.float32, (B, 3, hp, wp), cuda)
        img_g = torch.from_numpy(imgs).to(cuda)
        L.check(lib.femasr_u8_to_input(img_g.data_ptr(), g.ptr(), B, h, w, hp, wp, G.S()))
        tag = f"u8_to_input {B}x{h}x{w} -> {hp}x{wp}"
        same_bits(fetch(g, torch.float32, (B, 3, hp, wp), tag).cpu(), want, tag)


def test_output_to_u8(cuda):
    """Every k/255 and its neighbouring floats, every rounding midpoint (k + 1/2)/255 and its neighbours, negatives,
    values above 1, +-inf: bit for bit tensor2img's fp32 clamp -> x255 -> round half to even.  NaN gives 0."""
    lib = L.load()
    k = np.arange(256, dtype=np.float64)
    base = np.concatenate([k / 255, (k + 0.5) / 255]).astype(np.float32)
    vals = np.concatenate([base, np.nextafter(base, np.float32(np.inf)), np.nextafter(base, np.float32(-np.inf)),
                           np.array([-1.0, -0.0, -1e-30, -1e30, 1.0 + 2 ** -23, 1.5, 2.0, 1e30, np.inf, -np.inf, np.nan],
                                    np.float32)])
    B, SH, SW, ch, cw = 2, 41, 37, 40, 35          # the crop leaves one row and two columns out
    n = B * 3 * ch * cw
    assert n >= vals.size
    flat = np.resize(vals, n)
    np.random.default_rng(4).shuffle(flat)
    y = torch.full((B, 3, SH, SW), float("nan"))
    y[:, :, :ch, :cw] = torch.from_numpy(flat.reshape(B, 3, ch, cw))
    g = Guarded(B * ch * cw * 3, cuda)
    yg = y.to(cuda)
    L.check(lib.femasr_output_to_u8(yg.data_ptr(), g.ptr(), B, SH, SW, ch, cw, G.S()))
    got = fetch(g, torch.uint8, (B, ch, cw, 3), "output_to_u8").cpu().numpy()
    for b in range(B):
        crop = y[b:b + 1, :, :ch, :cw]
        want = tensor2img(torch.nan_to_num(crop, nan=0.0, posinf=np.inf, neginf=-np.inf))
        assert np.array_equal(got[b], want), f"output_to_u8 image {b}: {(got[b] != want).sum()} bytes differ"
        assert (got[b][np.isnan(crop[0].permute(1, 2, 0).numpy()[:, :, ::-1])] == 0).all()


OUT_SHAPES = {0: ((3, 31), (4, 32), (5, 33), (1, 1), (9, 65)), 1: ((7, 29), (8, 30), (9, 31), (1, 1), (17, 61))}


@pytest.mark.parametrize("mma", [0, 1])
def test_out_conv_guarded(cuda, mma):
    """femasr_out_conv3x3_n writes the caller's NCHW y: Cout 3 and Cout 1 alternating (they share the library-global
    weights), at sizes one below, at and one above the 4x32 (SIMT) and 8x30 (mma) tiles, B = 3, inside guard bands."""
    lib = L.load()
    B = 3
    for i, (H, W) in enumerate(OUT_SHAPES[mma]):
        for co in (3, 1):
            g = torch.Generator().manual_seed(100 * i + co)
            x = torch.randn(B, 64, H, W, generator=g) * (1.5 if mma else 1.0)     # the scales of test_in_conv_out_conv
            w, b = torch.randn(co, 64, 3, 3, generator=g) * 0.05, torch.randn(co, generator=g)
            want = F.conv2d(x.double(), w.double(), b.double(), padding=1)
            out = guarded_out(torch.float32, (B, co, H, W), cuda)
            xg, wp, bg = G.nhwc(x).to(cuda), G.pack_weight(w.to(cuda)), b.to(cuda)
            L.check(lib.femasr_out_conv3x3_n(xg.data_ptr(), wp.data_ptr(), bg.data_ptr(), out.ptr(), B, H, W, 64, co, mma,
                                             G.S()))
            tag = f"out_conv mma={mma} Cout {co} {H}x{W}"
            got = fetch(out, torch.float32, (B, co, H, W), tag)
            assert prefilled(got) == 0, f"{tag}: {prefilled(got)} outputs never written"
            err = (got.cpu().double() - want).abs().max().item()
            bar = 5e-6 * want.abs().max().item() if mma else 2e-5
            assert err <= bar, f"{tag}: max-abs {err:.3e} > {bar:.1e}"


@pytest.mark.parametrize("W", [6, 7, 8, 9])
def test_in_conv_cout64(cuda, W):
    """femasr_in_conv4x4 at Cout 64 (the HQ stage's in_conv) with W - 1 = 1, 2, 3, 0 (mod 4), against fp64."""
    lib = L.load()
    B, H, cout = 2, 5, 64
    g = torch.Generator().manual_seed(W)
    x, w, b = torch.rand(B, 3, H, W, generator=g), torch.randn(cout, 3, 4, 4, generator=g) * 0.15, torch.randn(cout, generator=g)
    want = F.conv2d(x.double(), w.double(), b.double(), padding=1)
    out = guarded_out(torch.float32, (B, H - 1, W - 1, cout), cuda)
    xg, wp, bg = x.to(cuda), G.pack_weight(w.to(cuda)), b.to(cuda)
    L.check(lib.femasr_in_conv4x4(xg.data_ptr(), wp.data_ptr(), bg.data_ptr(), out.ptr(), B, 3, H, W, cout, G.S()))
    got = fetch(out, torch.float32, (B, H - 1, W - 1, cout), f"in_conv W={W}")
    assert prefilled(got) == 0
    err = (G.nchw(got).cpu().double() - want).abs().max().item()
    assert err <= 2e-6 * 48 ** 0.5 * 4, f"in_conv Cout 64 W={W}: max-abs {err:.3e}"
