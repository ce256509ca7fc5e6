"""CPU: the HQ stage's semantic loss (use_semantic_loss=True, femasr_arch.py:301-309, 318-320, 344-347, 372).
The oracle (tests/semantic_oracle.py) against the reference's outputs in tests/golden/semantic/ (written by
tests/golden/make_golden_semantic.py from the unmodified reference), the parameter inventory against the reference's, the
C engine's spec after femasr_net_enable_semantic, and the VGG weight sources of the drop-in module."""
import ctypes
import glob
import gzip
import json
import os
import warnings

import numpy as np
import pytest
import torch

from femasr_b200.spec import VGG_CONVS, VGG_TORCHVISION_INDEX, param_spec, random_state_dict
from tests import semantic_oracle as SO
from tests.golden_util import indices_of

HERE = os.path.dirname(os.path.abspath(__file__))
SEM_DIR = os.path.join(HERE, "golden", "semantic")
SEM_GOLDEN = sorted(glob.glob(os.path.join(SEM_DIR, "*.npz")))
SEM_IDS = [os.path.basename(p)[:-4] for p in SEM_GOLDEN]
INVENTORY = os.path.join(SEM_DIR, "reference_state_dicts_sem.json.gz")
INV_CONFIGS = {"x1_1cb_e512_sem": (1, [[32, 1024, 512]]), "x4_1cb_e512_sem": (4, [[32, 1024, 512]])}


def sample(t):
    return t[:, ::17, ::3, ::3].contiguous().numpy()


def load_sem_case(path):
    g = np.load(path)
    scale, e_dim = int(g["scale"]), int(g["e_dim"])
    cbs = [[int(v) for v in row] for row in g["codebooks"]]
    sd = random_state_dict(scale, e_dim, seed=int(g["seed"]), init=str(g["init"]), codebooks=cbs, semantic=True)
    return g, sd, cbs


def make_module(scale, cbs, **kw):
    from basicsr.archs.femasr_arch import FeMaSRNet
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        return FeMaSRNet(codebook_params=cbs, LQ_stage=scale != 1, scale_factor=scale, use_semantic_loss=True, **kw)


def test_semantic_goldens_present():
    assert SEM_IDS == ["hq_e512_sem_fwd", "hq_e512_sem_fwd_default", "x4_e512_sem_test"]


@pytest.mark.parametrize("path", SEM_GOLDEN, ids=SEM_IDS)
def test_oracle_matches_semantic_golden(path):
    from tests.test_oracle import digest
    g, sd, cbs = load_sem_case(path)
    assert digest(sd) == str(g["digest"]), "seeded weight generator drifted from the one used for the goldens"
    scale = int(g["scale"])
    x = torch.from_numpy(g["input"])
    with torch.no_grad():
        if str(g["entry"]) == "forward":
            taps = {}
            out, loss, sem, idx = SO.encode_and_decode(sd, x, scale, taps, semantic=True)
            assert np.array_equal(idx[0].numpy(), indices_of(g)[0]), "codebook indices must be bit-exact"
            np.testing.assert_allclose(loss.numpy(), g["loss"], rtol=1e-6)
            np.testing.assert_allclose(sem.numpy(), g["sem"], rtol=1e-6)
            assert float(sem) > 0
            for ours, theirs in (("vgg", "vgg"), ("semantic", "semantic"), ("z", "z"), ("after_quant", "after_quant"),
                                 ("dec0", "dec0"), ("dec1", "dec1"), ("dec2", "dec2")):
                np.testing.assert_allclose(sample(taps[ours]), g["tap_" + theirs], rtol=0, atol=1e-5)
        else:
            from oracle import femasr_oracle as O
            out = O.test(sd, x, scale)        # test() switches the flag off for its call (femasr_arch.py:451-452, 467)
    np.testing.assert_allclose(out.numpy(), g["out"], rtol=0, atol=1e-5)


def test_oracle_semantic_raises_where_the_reference_does():
    sd = random_state_dict(4, 512, seed=5, semantic=True)
    with pytest.raises(RuntimeError):      # LQ x4: z_quant at H/2, relu4_4 at H/8
        SO.encode_and_decode(sd, torch.rand(1, 3, 32, 32), 4, semantic=True)


@pytest.mark.parametrize("cid", sorted(INV_CONFIGS))
def test_spec_and_module_match_reference_inventory(cid):
    with gzip.open(INVENTORY, "rt") as f:
        ref = json.load(f)[cid]
    scale, cbs = INV_CONFIGS[cid]
    want = {k: (tuple(shape), getattr(torch, dtype)) for k, (shape, dtype) in ref.items()}
    spec = {n: tuple(s) for n, s, _k, _f in param_spec(scale, cbs[0][2], cbs[0][1], codebooks=cbs, semantic=True)}
    assert spec == {k: s for k, (s, _d) in want.items()}
    sd = random_state_dict(scale, cbs[0][2], seed=3, codebooks=cbs, semantic=True)
    assert {k: tuple(v.shape) for k, v in sd.items()} == spec
    mine = make_module(scale, cbs)
    # strict both ways: the reference-shaped dict loads here, and what this module holds is exactly the reference's keys
    res = mine.load_state_dict({k: torch.zeros(s, dtype=d) for k, (s, d) in want.items()}, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert {k: (tuple(v.shape), v.dtype) for k, v in mine.state_dict().items()} == want
    if scale == 1:
        assert len(want) == 145


def test_semantic_entries_only_when_asked():
    base = param_spec(1, 512, 1024)
    sem = param_spec(1, 512, 1024, semantic=True)
    assert sem[:len(base)] == base and len(sem) - len(base) == 28
    a = random_state_dict(1, 512, seed=7, init="perturbed")
    b = random_state_dict(1, 512, seed=7, init="perturbed", semantic=True)
    assert list(b)[:len(a)] == list(a)
    for k, v in a.items():
        assert torch.equal(v, b[k]), k
    for n, ci, co in VGG_CONVS:
        w = random_state_dict(1, 512, seed=7, semantic=True)[f"vgg_feat_extractor.vgg_net.{n}.weight"]
        assert tuple(w.shape) == (co, ci, 3, 3)
        assert abs(w.std().item() / (2.0 / (9 * co)) ** 0.5 - 1) < 0.15
    d = random_state_dict(1, 512, seed=7, semantic=True)
    assert all(not d[f"vgg_feat_extractor.vgg_net.{n}.bias"].any() for n, _ci, _co in VGG_CONVS)
    assert b["vgg_feat_extractor.vgg_net.conv1_1.bias"].abs().max() > 0
    assert torch.equal(b["vgg_feat_extractor.mean"].flatten(), torch.tensor([0.485, 0.456, 0.406]))
    assert torch.equal(b["vgg_feat_extractor.std"].flatten(), torch.tensor([0.229, 0.224, 0.225]))


@pytest.mark.parametrize("scale,cbs", [(1, [[32, 1024, 512]]), (4, [[32, 1024, 256]])])
def test_engine_accepts_semantic_names_after_enable(built_lib, scale, cbs):
    """The C engine knows the 28 names only after femasr_net_enable_semantic, and then requires them.  Host buffers,
    no kernel launches (wrong-size uploads are rejected for their SIZE, unknown names for their NAME)."""
    from femasr_b200 import lib
    L = lib.load()
    I3 = ctypes.c_int * 3
    cfg = lib.NetConfig(scale, cbs[0][1], cbs[0][2], 3, 1, 1, 0, 1, I3(32, 0, 0), I3(cbs[0][1], 0, 0), I3(cbs[0][2], 0, 0))
    extra = [(n, s) for n, s, _k, _f in param_spec(scale, cbs[0][2], cbs[0][1], codebooks=cbs, semantic=True)][
        len(param_spec(scale, cbs[0][2], cbs[0][1], codebooks=cbs)):]
    assert len(extra) == 28
    buf = torch.zeros(4)
    for enable in (False, True):
        h = ctypes.c_void_p()
        assert L.femasr_net_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
        try:
            if enable:
                assert L.femasr_net_enable_semantic(h) == 0
            for n, s in extra:
                numel = int(np.prod(s))
                assert L.femasr_net_set_param(h, n.encode(), buf.data_ptr(), numel + 1, 0, None) == -1
                msg = L.femasr_last_error()
                assert (b"wrong size" in msg) if enable else (b"unknown parameter" in msg), (n, msg)
            need, need0 = ctypes.c_size_t(), ctypes.c_size_t()
            H, W = (64, 96) if scale == 1 else (32, 32)
            assert L.femasr_net_workspace_bytes(h, 2, H, W, ctypes.byref(need0)) == 0
            assert L.femasr_net_workspace_bytes_sem(h, 2, H, W, 0, ctypes.byref(need)) == 0
            assert need.value == need0.value
            st = L.femasr_net_workspace_bytes_sem(h, 2, H, W, 1, ctypes.byref(need))
            if not enable:
                assert st == -3
            elif scale == 1:
                assert st == 0 and need.value > need0.value
            else:                                   # LQ x4 e256: conv_semantic channels, then sizes
                assert st == -1
                msg = L.femasr_last_error()
                assert b"[B,256,16,16]" in msg and b"[B,512,4,4]" in msg, msg
        finally:
            L.femasr_net_destroy(h)


def _write_torchvision_vgg(path, seed=0):
    """A torchvision-layout vgg19 state_dict ('features.{i}.weight', ...), without needing torchvision."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for (_n, ci, co), i in zip(VGG_CONVS, VGG_TORCHVISION_INDEX):
        sd[f"features.{i}.weight"] = torch.randn(co, ci, 3, 3, generator=g)
        sd[f"features.{i}.bias"] = torch.randn(co, generator=g)
    for i, (ci, co) in enumerate(((512, 512),) * 4):        # conv5_x (beyond relu4_4, unused)
        sd[f"features.{28 + 2 * i}.weight"] = torch.randn(co, ci, 3, 3, generator=g)
    sd["classifier.0.weight"] = torch.randn(8, 8, generator=g)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    torch.save(sd, path)
    return sd


def _block_downloads(monkeypatch):
    import torch.hub

    def refuse(*_a, **_k):
        raise AssertionError("network access attempted")
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)


def test_vgg_weights_from_torchvision_file(tmp_path, monkeypatch):
    from basicsr.archs.femasr_arch import FeMaSRNet
    _block_downloads(monkeypatch)
    monkeypatch.chdir(tmp_path)
    tv = _write_torchvision_vgg(os.path.join("experiments", "pretrained_models", "vgg19-dcbb9e9d.pth"))
    with warnings.catch_warnings():
        warnings.simplefilter("error", UserWarning)          # the file is there: no warning
        net = FeMaSRNet(codebook_params=[[32, 1024, 512]], LQ_stage=False, use_semantic_loss=True)
    sd = net.state_dict()
    for (n, _ci, _co), i in zip(VGG_CONVS, VGG_TORCHVISION_INDEX):
        assert torch.equal(sd[f"vgg_feat_extractor.vgg_net.{n}.weight"], tv[f"features.{i}.weight"]), n
        assert torch.equal(sd[f"vgg_feat_extractor.vgg_net.{n}.bias"], tv[f"features.{i}.bias"]), n


def test_vgg_missing_file_warns_and_never_downloads(tmp_path, monkeypatch):
    from basicsr.archs.femasr_arch import FeMaSRNet
    _block_downloads(monkeypatch)
    monkeypatch.chdir(tmp_path)
    with pytest.warns(UserWarning, match="ImageNet VGG19 weights are expected from a checkpoint"):
        net = FeMaSRNet(codebook_params=[[32, 1024, 512]], LQ_stage=False, use_semantic_loss=True)
    w = net.state_dict()["vgg_feat_extractor.vgg_net.conv4_4.weight"]
    assert abs(w.std().item() / (2.0 / (9 * 512)) ** 0.5 - 1) < 0.05
    with warnings.catch_warnings():
        warnings.simplefilter("error", UserWarning)
        FeMaSRNet(codebook_params=[[32, 1024, 512]], LQ_stage=False)      # no flag: no VGG, no warning


def test_hq_pretrain_config_constructs():
    """network_g of options/train_FeMaSR_HQ_pretrain_stage.yml builds and loads a semantic state_dict strictly."""
    net = make_module(1, [[32, 1024, 512]], gt_resolution=256, norm_type="gn", act_type="silu")
    assert net.use_semantic_loss
    res = net.load_state_dict(random_state_dict(1, 512, seed=1, semantic=True), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
