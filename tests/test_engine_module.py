"""CPU: every engine-backed module (FeMaSRNet, UNetDiscriminatorSN, LPIPS) uploads its tensors to the native handle
exactly when one of them changes, and copies / pickles drop the handle.  A fake engine with the real handle's names
records every upload."""
import copy
import pickle
import warnings

import pytest
import torch
from torch import nn

from basicsr.archs.discriminator_arch import UNetDiscriminatorSN
from basicsr.archs.femasr_arch import FeMaSRNet
from femasr_b200 import default_gemm_path
from femasr_b200.lpips import LPIPS

DEV = torch.device("cpu")      # the fake engine never touches a device


class FakeEngine:
    def __init__(self, names, gemm_path):
        self.names, self.gemm_path = names, gemm_path
        self.uploads = []

    def load_state_dict(self, sd, device):
        self.uploads.append(dict(sd))


BUILD = {
    "femasr": lambda: FeMaSRNet(codebook_params=[[32, 1024, 256]], LQ_stage=True, scale_factor=4),
    "disc": lambda: UNetDiscriminatorSN(3),
    "lpips": lambda: LPIPS("alex"),
}


@pytest.fixture(params=sorted(BUILD))
def net(request, monkeypatch, built_lib):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)       # LPIPS without weight files
        m = BUILD[request.param]()
    cls = type(m)
    real = cls._make_engine
    monkeypatch.setattr(cls, "_make_engine", lambda self, gp: FakeEngine(real(self, gp).names, gp))
    return m


def assert_uploaded_current(net, upload):
    """The upload holds exactly the engine's names, each the module's current tensor object."""
    cur = net.state_dict(keep_vars=True)
    assert list(upload) == net._engine.names
    stale = [n for n, t in upload.items() if t is not cur[n]]
    assert not stale, f"stale tensors uploaded: {stale[:3]}"


def last_param(net):
    params = dict(net.named_parameters())
    return next(n for n in reversed(net._engine.names) if n in params)


def test_first_call_uploads_every_name_then_nothing(net):
    eng = net._native(DEV)
    assert eng.gemm_path == default_gemm_path()
    assert len(eng.uploads) == 1
    assert_uploaded_current(net, eng.uploads[0])
    assert net._native(DEV) is eng and len(eng.uploads) == 1


def _add(net, name):
    with torch.no_grad():
        net.get_parameter(name).add_(1.0)


def _load(net, name, assign=False):
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    sd[name] += 1.0
    net.load_state_dict(sd, assign=assign)


def _replace(net, name):
    path, _, leaf = name.rpartition(".")
    setattr(net.get_submodule(path), leaf, nn.Parameter(net.get_parameter(name).detach() + 1.0, requires_grad=False))


CHANGES = {
    "add_": _add,
    "load_state_dict": _load,
    "load_state_dict_assign": lambda net, name: _load(net, name, assign=True),
    "to_float64": lambda net, name: net.to(torch.float64),
    "replace_parameter": _replace,
}


@pytest.mark.parametrize("change", sorted(CHANGES))
def test_each_change_uploads_once(net, change):
    eng = net._native(DEV)
    name = last_param(net)
    before = net.get_parameter(name).detach().clone()
    CHANGES[change](net, name)
    net._native(DEV)
    net._native(DEV)
    assert len(eng.uploads) == 2
    assert_uploaded_current(net, eng.uploads[1])
    if change != "to_float64":
        assert torch.equal(eng.uploads[1][name], before + 1.0)


def test_data_write_needs_refresh_weights(net):
    eng = net._native(DEV)
    name = last_param(net)
    net.get_parameter(name).data.add_(1.0)        # .data writes do not bump _version (BasicSR's model_ema)
    net._native(DEV)
    assert len(eng.uploads) == 1
    net.refresh_weights()
    net._native(DEV)
    net._native(DEV)
    assert len(eng.uploads) == 2
    assert_uploaded_current(net, eng.uploads[1])


@pytest.mark.parametrize("how", ["deepcopy", "pickle"])
def test_copies_drop_the_handle(net, how):
    eng = net._native(DEV)
    clone = copy.deepcopy(net) if how == "deepcopy" else pickle.loads(pickle.dumps(net))
    assert clone._engine is None and clone._engine_sig is None
    assert net._engine is eng and net._engine_sig is not None
    fresh = clone._native(DEV)
    assert fresh is not eng and len(fresh.uploads) == 1
    assert_uploaded_current(clone, fresh.uploads[0])
