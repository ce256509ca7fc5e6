"""CPU: UNetDiscriminatorSN (the training configs' network_d) - the module's state_dict against the reference's stored
inventory, build_network, the constructor rejections, the oracle against the reference's goldens (tests/golden/disc/),
and the engine's sizing run (workspace, geometry rejection, FLOP count) without a GPU."""
import ctypes as C
import glob
import gzip
import json
import os

import numpy as np
import pytest
import torch

from femasr_b200.spec import disc_spec, random_disc_state_dict
from tests import disc_oracle as DO

DISC_DIR = os.path.join(os.path.dirname(__file__), "golden", "disc")
DISC_GOLDEN = sorted(glob.glob(os.path.join(DISC_DIR, "*.npz")))
DISC_IDS = [os.path.basename(p)[:-4] for p in DISC_GOLDEN]


def load_disc_case(path):
    g = np.load(path)
    return g, random_disc_state_dict(int(g["seed"]), power_iterations=int(g["power_iterations"]))


def disc_flops_closed_form(B, H, W, F=64):
    """2 * MAC of every conv; conv0 at K = 27."""
    f = H * W * F * 27                                                   # conv0
    f += sum((H >> i) * (W >> i) * (F << i) * (F << (i - 1)) * 16 for i in (1, 2, 3))   # conv1 .. conv3
    f += sum((H >> lv) * (W >> lv) * (F << lv) * (F << (lv + 1)) * 9 for lv in (2, 1, 0))   # conv4 .. conv6
    f += 2 * H * W * F * F * 9 + H * W * F * 9                           # conv7, conv8, conv9
    return 2.0 * B * f


def test_state_dict_matches_reference_inventory():
    from basicsr.archs.discriminator_arch import UNetDiscriminatorSN
    with gzip.open(os.path.join(DISC_DIR, "reference_state_dict_disc.json.gz"), "rt") as f:
        inv = json.load(f)
    sd = UNetDiscriminatorSN(3).state_dict()
    assert len(inv) == len(sd) == 28
    assert {k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in sd.items()} == inv
    assert [n for n, *_ in disc_spec()] == list(sd)
    assert set(random_disc_state_dict(0)) == set(inv)
    net = UNetDiscriminatorSN(3)
    assert {k for k, _ in net.named_buffers()} == {k for k in inv if k.endswith(("weight_u", "weight_v"))}
    for k, _ in net.named_buffers():
        assert abs(sd[k].norm().item() - 1.0) < 1e-5                     # normalize(randn), like spectral_norm


def test_build_network_and_strict_load():
    from basicsr.archs import build_network
    net = build_network({"type": "UNetDiscriminatorSN", "num_in_ch": 3})
    assert type(net).__name__ == "UNetDiscriminatorSN" and net.skip_connection
    missing = net.load_state_dict(random_disc_state_dict(1), strict=True)
    assert not missing.missing_keys and not missing.unexpected_keys
    net = build_network({"type": "UNetDiscriminatorSN", "num_in_ch": 3, "num_feat": 64, "skip_connection": False})
    assert not net.skip_connection


def test_constructor_rejections():
    from basicsr.archs.discriminator_arch import UNetDiscriminatorSN
    with pytest.raises(NotImplementedError, match="num_in_ch"):
        UNetDiscriminatorSN(1)
    with pytest.raises(NotImplementedError, match="num_feat"):
        UNetDiscriminatorSN(3, num_feat=32)


@pytest.mark.parametrize("path", DISC_GOLDEN, ids=DISC_IDS)
def test_oracle_matches_reference_goldens(path):
    g, sd = load_disc_case(path)
    taps = {}
    with torch.no_grad():
        out = DO.forward(sd, torch.from_numpy(g["input"]), bool(g["skip"]), taps)
    want = g["out"]
    assert np.abs(out.numpy() - want).max() <= 1e-6 * np.abs(want).max()
    big = want.shape[2] * want.shape[3] > 64 * 64
    for i in range(10):
        t = taps[f"conv{i}"]
        s = (t[:, ::16, ::8, ::8] if big else t[:, ::8, ::2, ::2]).numpy()
        w = g[f"tap_conv{i}"]
        assert np.abs(s - w).max() <= 1e-6 * np.abs(w).max(), f"conv{i}"


def test_iterated_weights_keep_activations_in_range():
    """30 power iterations: sigma == |W v| to fp32 rounding, and the SR-output workload stays O(1) everywhere."""
    sd = random_disc_state_dict(5)
    for i in range(1, 9):
        w = sd[f"conv{i}.weight_orig"]
        wv = torch.mv(w.reshape(w.shape[0], -1).double(), sd[f"conv{i}.weight_v"].double())
        assert abs(DO.sigma(sd, f"conv{i}").item() - wv.norm().item()) <= 1e-5 * wv.norm().item()
    taps = {}
    with torch.no_grad():
        DO.forward(sd, torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(0)), True, taps)
    assert max(t.abs().max().item() for t in taps.values()) < 10


def _disc_handle(gemm_path, skip=1):
    from femasr_b200 import lib as L
    lib = L.load()
    h = C.c_void_p()
    L.check(lib.femasr_disc_create(C.byref(L.DiscConfig(3, 64, skip, gemm_path)), C.byref(h)))
    return lib, h


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_workspace_and_geometry(built_lib, gemm_path):
    lib, h = _disc_handle(gemm_path)
    try:
        need = C.c_size_t()
        sizes = {}
        for B, H, W in ((1, 8, 8), (2, 24, 40), (8, 256, 256)):
            assert lib.femasr_disc_workspace_bytes(h, B, H, W, C.byref(need)) == 0
            assert need.value > 0
            sizes[(B, H, W)] = need.value
        # at least the live activations of the widest point (x0 and x1 beside conv6's input)
        assert sizes[(8, 256, 256)] >= 8 * 256 * 256 * 64 * 4 * 2
        for H, W in ((12, 16), (16, 20), (0, 8), (250, 256)):
            need.value = 12345
            assert lib.femasr_disc_workspace_bytes(h, 1, H, W, C.byref(need)) == -1
            assert need.value == 12345
            assert lib.femasr_disc_flops(h, 1, H, W) == 0.0
        assert lib.femasr_net_params_complete(h) == -3                   # nothing uploaded
    finally:
        lib.femasr_net_destroy(h)


@pytest.mark.parametrize("gemm_path", [0, 1])
def test_flops_equal_closed_form(built_lib, gemm_path):
    lib, h = _disc_handle(gemm_path, skip=gemm_path)
    try:
        assert abs(lib.femasr_disc_flops(h, 1, 256, 256) / 1e9 - 51.84) < 0.005
        for B, H, W in ((1, 256, 256), (2, 24, 40), (8, 256, 256), (3, 8, 64)):
            assert lib.femasr_disc_flops(h, B, H, W) == disc_flops_closed_form(B, H, W)
    finally:
        lib.femasr_net_destroy(h)


def test_generator_and_discriminator_entry_points_refuse_each_other(built_lib):
    from femasr_b200 import lib as L
    lib, d = _disc_handle(0)
    g = C.c_void_p()
    L.check(lib.femasr_net_create(C.byref(L.NetConfig(4, 1024, 256, 3, 1, 1, 0)), C.byref(g)))
    try:
        need = C.c_size_t()
        x = C.c_void_p(256)
        assert lib.femasr_net_workspace_bytes(d, 1, 32, 32, C.byref(need)) == -1
        assert lib.femasr_net_workspace_bytes_sem(d, 1, 32, 32, 0, C.byref(need)) == -1
        assert lib.femasr_net_forward(d, x, x, None, None, 1, 32, 32, x, 1 << 30, None) == -1
        assert lib.femasr_net_decode_workspace_bytes(d, 1, 4, 4, C.byref(need)) == -1
        assert lib.femasr_net_set_tap(d, b"down", None, 0) == -1
        assert lib.femasr_net_enable_semantic(d) == -1
        assert lib.femasr_net_flops(d, 1, 32, 32) == 0.0
        assert lib.femasr_disc_workspace_bytes(g, 1, 32, 32, C.byref(need)) == -1
        assert lib.femasr_disc_forward(g, x, x, 1, 32, 32, x, 1 << 30, None) == -1
        assert lib.femasr_disc_flops(g, 1, 32, 32) == 0.0
        assert lib.femasr_net_set_param(d, b"conv1.weight", x, 1, 1, None) == -1      # SN layers have weight_orig
        bad = L.DiscConfig(3, 32, 1, 0)
        h = C.c_void_p()
        assert lib.femasr_disc_create(C.byref(bad), C.byref(h)) == -1
    finally:
        lib.femasr_net_destroy(d)
        lib.femasr_net_destroy(g)
