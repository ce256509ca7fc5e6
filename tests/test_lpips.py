"""CPU: LPIPS v0.1 (femasr_b200.lpips) - the state_dict inventory against an lpips-layout tree built from torchvision, the
constructor rejections, the oracle against the goldens (tests/golden/lpips/), and the engine's sizing run (workspace,
geometry refusals, FLOP count) without a GPU."""
import ctypes as C
import glob
import os
import warnings

import numpy as np
import pytest
import torch

from femasr_b200.spec import LPIPS_CHANNELS, LPIPS_CONVS, lpips_spec, random_lpips_state_dict
from tests import lpips_oracle as LO

LPIPS_DIR = os.path.join(os.path.dirname(__file__), "golden", "lpips")
LPIPS_GOLDEN = sorted(glob.glob(os.path.join(LPIPS_DIR, "*.npz")))
LPIPS_IDS = [os.path.basename(p)[:-4] for p in LPIPS_GOLDEN]
NETS = {"alex": 0, "vgg": 1}


def load_lpips_case(path):
    """(record, net, state_dict, in0, in1, normalize) of a golden file."""
    g = np.load(path)
    net, normalize = str(g["net"]), bool(g["normalize"])
    conv = (lambda u: torch.from_numpy(u).float() / 255.0) if normalize else (lambda u: torch.from_numpy(u).float() / 127.5 - 1.0)
    return g, net, random_lpips_state_dict(net, int(g["seed"])), conv(g["x0_u8"]), conv(g["x1_u8"]), normalize


def lpips_flops_closed_form(net, B, H, W):
    """2 * MAC of the backbone convs for both images of B pairs; alex conv1 at K = 363, vgg conv1_1 at K = 27."""
    macs, h, w = 0, H, W
    for _s, i, ci, co, k in LPIPS_CONVS[net]:
        if net == "alex":
            if i == 0:
                h, w = (h + 4 - 11) // 4 + 1, (w + 4 - 11) // 4 + 1
            elif i in (3, 6):
                h, w = (h - 3) // 2 + 1, (w - 3) // 2 + 1
        elif i in (5, 10, 17, 24):
            h, w = h // 2, w // 2
        macs += h * w * co * ci * k * k
    return 2.0 * 2 * B * macs


def test_state_dict_matches_lpips_layout_from_torchvision():
    torchvision = pytest.importorskip("torchvision")
    from femasr_b200.lpips import LPIPS
    for net, make in (("alex", torchvision.models.alexnet), ("vgg", torchvision.models.vgg16)):
        feats = make().features
        tree = {"scaling_layer.shift": (1, 3, 1, 1), "scaling_layer.scale": (1, 3, 1, 1)}
        for s, i, *_ in LPIPS_CONVS[net]:          # lpips.pretrained_networks: slice{s} holds features[i] under index i
            for p in ("weight", "bias"):
                tree[f"net.slice{s}.{i}.{p}"] = tuple(getattr(feats[i], p).shape)
        for k, c in enumerate(LPIPS_CHANNELS[net]):
            tree[f"lin{k}.model.1.weight"] = (1, c, 1, 1)
        with pytest.warns(UserWarning, match="untrained"):
            m = LPIPS(net)
        sd = m.state_dict()
        assert {k: tuple(v.shape) for k, v in sd.items()} == tree
        assert [n for n, *_ in lpips_spec(net)] == list(sd)
        assert set(random_lpips_state_dict(net, 0)) == set(tree)
        assert {k for k, _ in m.named_buffers()} == {"scaling_layer.shift", "scaling_layer.scale"}
        assert all((sd[f"lin{k}.model.1.weight"] >= 0).all() for k in range(5))
        torch.testing.assert_close(sd["scaling_layer.shift"].view(3), torch.tensor([-0.030, -0.088, -0.188]))
        torch.testing.assert_close(sd["scaling_layer.scale"].view(3), torch.tensor([0.458, 0.448, 0.450]))
        m.load_state_dict(random_lpips_state_dict(net, 1), strict=True)


def test_weight_files_load_and_report_keys(tmp_path):
    torchvision = pytest.importorskip("torchvision")
    from femasr_b200.lpips import LPIPS
    tv = torchvision.models.alexnet().state_dict()
    lins = {f"lin{k}.model.1.weight": torch.rand(1, c, 1, 1) for k, c in enumerate(LPIPS_CHANNELS["alex"])}
    torch.save(tv, tmp_path / "alex.pth")
    torch.save(lins, tmp_path / "lin.pth")
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        m = LPIPS("alex", backbone_path=str(tmp_path / "alex.pth"), lin_path=str(tmp_path / "lin.pth"))
    assert torch.equal(m.state_dict()["net.slice2.3.weight"], tv["features.3.weight"])
    assert torch.equal(m.state_dict()["lin4.model.1.weight"], lins["lin4.model.1.weight"])
    bad = dict(lins)
    bad.pop("lin2.model.1.weight")
    bad["lin9.model.1.weight"] = torch.rand(1, 3, 1, 1)
    torch.save(bad, tmp_path / "bad.pth")
    with pytest.raises(KeyError, match=r"lin2\.model\.1\.weight.*lin9\.model\.1\.weight"):
        LPIPS("alex", backbone_path=str(tmp_path / "alex.pth"), lin_path=str(tmp_path / "bad.pth"))
    tv.pop("features.8.bias")
    torch.save(tv, tmp_path / "tv_bad.pth")
    with pytest.raises(KeyError, match=r"features\.8\.bias"):
        LPIPS("alex", backbone_path=str(tmp_path / "tv_bad.pth"), lin_path=str(tmp_path / "lin.pth"))
    with pytest.warns(UserWarning):
        m = LPIPS("vgg")
    r = m.load_state_dict({k: v for k, v in random_lpips_state_dict("vgg", 2).items() if k != "lin3.model.1.weight"},
                          strict=False)
    assert r.missing_keys == ["lin3.model.1.weight"]


def test_constructor_rejections():
    from femasr_b200.lpips import LPIPS
    with pytest.raises(NotImplementedError, match="squeeze"):
        LPIPS("squeeze")
    with pytest.raises(NotImplementedError, match="lpips=False"):
        LPIPS("alex", lpips=False)
    with pytest.raises(NotImplementedError, match="spatial=True"):
        LPIPS("alex", spatial=True)
    with pytest.raises(NotImplementedError, match="version='0.0'"):
        LPIPS("vgg", version="0.0")


@pytest.mark.parametrize("path", LPIPS_GOLDEN, ids=LPIPS_IDS)
def test_oracle_matches_goldens(path):
    g, net, sd, in0, in1, normalize = load_lpips_case(path)
    with torch.no_grad():
        d, res = LO.forward(net, sd, in0, in1, retPerLayer=True, normalize=normalize)
    assert np.abs(d.view(-1).numpy() - g["d"]).max() <= 1e-6 * np.abs(g["d"]).max()
    r = torch.stack([t.view(-1) for t in res]).numpy()
    assert np.abs(r - g["r"]).max() <= 1e-6 * np.abs(g["r"]).max()
    assert 0.02 < g["d"].min() and g["d"].max() < 1.0                     # the range of a trained LPIPS


def _handle(net, gemm_path):
    from femasr_b200 import lib as L
    lib = L.load()
    h = C.c_void_p()
    L.check(lib.femasr_lpips_create(C.byref(L.LpipsConfig(NETS[net], gemm_path)), C.byref(h)))
    return lib, h


@pytest.mark.parametrize("gemm_path", [0, 1])
@pytest.mark.parametrize("net", ["alex", "vgg"])
def test_workspace_and_geometry(built_lib, net, gemm_path):
    lib, h = _handle(net, gemm_path)
    try:
        need = C.c_size_t()
        ok = ((1, 32, 48), (8, 256, 256), (1, 1344, 2032)) if net == "vgg" else ((1, 31, 31), (1, 67, 93), (8, 256, 256))
        for B, H, W in ok:
            assert lib.femasr_lpips_workspace_bytes(h, B, H, W, C.byref(need)) == 0
            assert need.value > 0
        # at least the widest live tensor: the first tap of both images of every pair
        lib.femasr_lpips_workspace_bytes(h, 8, 256, 256, C.byref(need))
        first = 256 * 256 if net == "vgg" else 63 * 63
        assert need.value >= 16 * first * 64 * 4
        bad = ((0, 32, 32), (1, 24, 64), (1, 32, 40)) if net == "vgg" else ((0, 64, 64), (1, 64, 16), (1, 30, 64))
        for B, H, W in bad:
            need.value = 12345
            assert lib.femasr_lpips_workspace_bytes(h, B, H, W, C.byref(need)) == -1
            assert need.value == 12345
            assert lib.femasr_lpips_flops(h, B, H, W) == 0.0
        assert (b"16" if net == "vgg" else b"31") in lib.femasr_last_error()
        assert lib.femasr_net_params_complete(h) == -3                   # nothing uploaded
    finally:
        lib.femasr_net_destroy(h)


@pytest.mark.parametrize("gemm_path", [0, 1])
@pytest.mark.parametrize("net", ["alex", "vgg"])
def test_flops_equal_closed_form(built_lib, net, gemm_path):
    lib, h = _handle(net, gemm_path)
    try:
        # per image, counted from torchvision's modules; femasr_lpips_flops counts both images of a pair
        table = {"alex": {(256, 256): 1.737004416e9, (1344, 2032): 78.571443072e9},
                 "vgg": {(256, 256): 40.089157632e9, (1344, 2032): 1670.590365696e9}}[net]
        for (H, W), per_image in table.items():
            assert lib.femasr_lpips_flops(h, 1, H, W) == 2 * per_image
        sizes = ((8, 256, 256), (2, 32, 48)) if net == "vgg" else ((8, 256, 256), (1, 67, 93), (3, 31, 40))
        for B, H, W in sizes:
            assert lib.femasr_lpips_flops(h, B, H, W) == lpips_flops_closed_form(net, B, H, W)
    finally:
        lib.femasr_net_destroy(h)


def test_entry_points_refuse_other_handles(built_lib):
    from femasr_b200 import lib as L
    lib, lp = _handle("alex", 0)
    g, d = C.c_void_p(), C.c_void_p()
    L.check(lib.femasr_net_create(C.byref(L.NetConfig(4, 1024, 256, 3, 1, 1, 0)), C.byref(g)))
    L.check(lib.femasr_disc_create(C.byref(L.DiscConfig(3, 64, 1, 0)), C.byref(d)))
    try:
        need = C.c_size_t()
        x = C.c_void_p(256)
        assert lib.femasr_net_workspace_bytes(lp, 1, 32, 32, C.byref(need)) == -1
        assert lib.femasr_net_workspace_bytes_sem(lp, 1, 32, 32, 0, C.byref(need)) == -1
        assert lib.femasr_net_forward(lp, x, x, None, None, 1, 32, 32, x, 1 << 30, None) == -1
        assert lib.femasr_net_decode_workspace_bytes(lp, 1, 4, 4, C.byref(need)) == -1
        assert lib.femasr_net_set_tap(lp, b"down", None, 0) == -1
        assert lib.femasr_net_enable_semantic(lp) == -1
        assert lib.femasr_net_flops(lp, 1, 32, 32) == 0.0
        assert lib.femasr_disc_workspace_bytes(lp, 1, 32, 32, C.byref(need)) == -1
        assert lib.femasr_disc_forward(lp, x, x, 1, 32, 32, x, 1 << 30, None) == -1
        assert lib.femasr_disc_flops(lp, 1, 32, 32) == 0.0
        for other in (g, d):
            assert lib.femasr_lpips_workspace_bytes(other, 1, 64, 64, C.byref(need)) == -1
            assert lib.femasr_lpips_forward(other, x, x, x, None, 1, 64, 64, 0, x, 1 << 30, None) == -1
            assert lib.femasr_lpips_flops(other, 1, 64, 64) == 0.0
        assert lib.femasr_net_set_param(lp, b"lin5.model.1.weight", x, 1, 1, None) == -1
        h = C.c_void_p()
        assert lib.femasr_lpips_create(C.byref(L.LpipsConfig(2, 0)), C.byref(h)) == -1      # squeeze
        assert lib.femasr_lpips_create(C.byref(L.LpipsConfig(0, 2)), C.byref(h)) == -1
    finally:
        for h in (lp, g, d):
            lib.femasr_net_destroy(h)
