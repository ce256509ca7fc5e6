"""Generate tests/golden/semantic/ (the use_semantic_loss=True fixtures) by running the UNMODIFIED reference, imported
from /root/reference through oracle/ref_shim.py, offline.  Build container only (needs the reference and torchvision):

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_semantic.py

The reference's VGGFeatureExtractor reads experiments/pretrained_models/vgg19-dcbb9e9d.pth relative to the working
directory and otherwise downloads ImageNet weights (vgg_arch.py:104-110).  So the reference is constructed inside a
temporary directory holding that file (a seeded torchvision vgg19(weights=None) state_dict), with torch.hub's download
functions replaced by ones that raise; the seeded weights of femasr_b200.spec.random_state_dict(..., semantic=True) are
then loaded with strict=True.  The files of tests/golden/*.npz are not touched.
"""
from __future__ import annotations

import contextlib
import gzip
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from femasr_b200.spec import random_state_dict  # noqa: E402
from make_golden import sample, sd_digest  # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "semantic")

# name, scale, e_dim, init, seed, entry, input shape
CASES = [
    ("hq_e512_sem_fwd", 1, 512, "perturbed", 30, "forward", (2, 3, 64, 96)),
    ("hq_e512_sem_fwd_default", 1, 512, "default", 31, "forward", (1, 3, 128, 128)),
    ("x4_e512_sem_test", 4, 512, "perturbed", 32, "test", (1, 3, 40, 24)),
]
# reference_state_dicts_sem.json.gz: the reference's inventory with the flag (id -> scale, codebook_params)
INVENTORY = {"x1_1cb_e512_sem": (1, [[32, 1024, 512]]), "x4_1cb_e512_sem": (4, [[32, 1024, 512]])}


def _refuse_download(*_a, **_k):
    raise RuntimeError("network access attempted while generating the semantic goldens")


@contextlib.contextmanager
def offline_vgg_cwd():
    """cwd = a temporary directory with the seeded VGG19 file; every download entry point raises."""
    import torch.hub
    import torchvision
    import torchvision.models._api as tv_api
    saved = (torch.hub.load_state_dict_from_url, torch.hub.download_url_to_file, tv_api.load_state_dict_from_url)
    torch.hub.load_state_dict_from_url = torch.hub.download_url_to_file = _refuse_download
    tv_api.load_state_dict_from_url = _refuse_download
    old = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "experiments", "pretrained_models"))
        torch.manual_seed(0)
        torch.save(torchvision.models.vgg19(weights=None).state_dict(),
                   os.path.join(tmp, "experiments", "pretrained_models", "vgg19-dcbb9e9d.pth"))
        os.chdir(tmp)
        try:
            yield
        finally:
            os.chdir(old)
            torch.hub.load_state_dict_from_url, torch.hub.download_url_to_file, tv_api.load_state_dict_from_url = saved


def main():
    ref = import_reference()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    os.makedirs(OUT, exist_ok=True)
    with offline_vgg_cwd():
        for name, scale, e_dim, init, seed, entry, shape in CASES:
            cbs = [[32, 1024, e_dim]]
            sd = random_state_dict(scale, e_dim, seed=seed, init=init, codebooks=cbs, semantic=True)
            net = ref.FeMaSRNet(codebook_params=cbs, LQ_stage=scale != 1, scale_factor=scale, use_semantic_loss=True).eval()
            net.load_state_dict(sd, strict=True)
            g = torch.Generator().manual_seed(1000 + seed)
            x = torch.rand(shape, generator=g)
            rec = dict(scale=scale, e_dim=e_dim, init=init, seed=seed, entry=entry, digest=sd_digest(sd),
                       codebooks=np.array(cbs, dtype=np.int64))
            taps, hooks = {}, []

            def hook(key):
                def fn(_m, _i, o):
                    taps[key] = o.detach().clone()
                return fn
            hooks.append(net.vgg_feat_extractor.vgg_net.relu4_4.register_forward_hook(hook("vgg")))
            hooks.append(net.conv_semantic.register_forward_hook(hook("semantic")))
            hooks.append(net.before_quant_group[0].register_forward_hook(hook("z")))
            hooks.append(net.after_quant_group[0].register_forward_hook(hook("after_quant")))
            for i in range(3):
                hooks.append(net.decoder_group[i].register_forward_hook(hook(f"dec{i}")))
            with torch.no_grad():
                if entry == "forward":
                    out, loss, sem, idx = net(x)
                    rec.update(loss=loss.numpy(), sem=sem.numpy(), indices=idx[0].numpy())
                else:
                    out = net.test(x)
                    assert not any(k in taps for k in ("vgg", "semantic")), "test() must not run the VGG branch"
            for h in hooks:
                h.remove()
            rec.update(input=x.numpy(), out=out.numpy())
            if entry == "forward":
                rec.update({f"tap_{k}": sample(v) for k, v in taps.items()})
            path = os.path.join(OUT, name + ".npz")
            np.savez_compressed(path, **rec)
            print(f"{name}: out {tuple(out.shape)} sem {float(rec.get('sem', 0.0)):.6g} -> {os.path.getsize(path) / 1e3:.0f} kB")
        inv = {}
        for cid, (scale, cbs) in INVENTORY.items():
            net = ref.FeMaSRNet(codebook_params=cbs, LQ_stage=scale != 1, scale_factor=scale, use_semantic_loss=True)
            inv[cid] = {k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in net.state_dict().items()}
    text = json.dumps(inv, sort_keys=True, separators=(",", ":")) + "\n"
    with gzip.GzipFile(os.path.join(OUT, "reference_state_dicts_sem.json.gz"), "wb", compresslevel=9, mtime=0) as f:
        f.write(text.encode())


if __name__ == "__main__":
    main()
