"""Generate tests/golden/disc/ (the UNetDiscriminatorSN fixtures) by running the UNMODIFIED reference, imported from
/root/reference through oracle/ref_shim.py, offline.  Build container only (needs the reference):

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_disc.py

Weights are femasr_b200.spec.random_disc_state_dict(seed, power_iterations), loaded with strict=True into the reference's
network in eval mode.  Each case stores the input, the output, and a strided sample of every conv's output before its
activation (forward hooks on conv0 ... conv9).  The other golden files are not touched.
"""
from __future__ import annotations

import gzip
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from femasr_b200.spec import random_disc_state_dict  # noqa: E402
from make_golden import sd_digest  # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "disc")

# name, skip_connection, seed, power iterations of u / v, input shape
CASES = [
    ("skip_b1_8x8", True, 70, 30, (1, 3, 8, 8)),
    ("skip_b2_24x40", True, 71, 30, (2, 3, 24, 40)),
    ("noskip_b2_32x16", False, 72, 30, (2, 3, 32, 16)),
    ("skip_b1_256x256", True, 73, 30, (1, 3, 256, 256)),
    ("fresh_skip_b1_16x16", True, 74, 0, (1, 3, 16, 16)),       # u, v never iterated: sigma is tiny, outputs are huge
]


def sample(t: torch.Tensor, big: bool) -> np.ndarray:
    """Strided sample of an NCHW conv output (keeps the fixtures small)."""
    return (t[:, ::16, ::8, ::8] if big else t[:, ::8, ::2, ::2]).contiguous().numpy()


def main():
    ref = import_reference()
    mod = ref._ref_modules["basicsr.archs.discriminator_arch"]
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    os.makedirs(OUT, exist_ok=True)
    for name, skip, seed, iters, shape in CASES:
        sd = random_disc_state_dict(seed, power_iterations=iters)
        net = mod.UNetDiscriminatorSN(3, num_feat=64, skip_connection=skip).eval()
        net.load_state_dict(sd, strict=True)
        x = torch.rand(shape, generator=torch.Generator().manual_seed(1000 + seed))
        taps, hooks = {}, []
        for i in range(10):
            def fn(_m, _i, o, key=f"conv{i}"):
                taps[key] = o.detach().clone()      # before the in-place leaky_relu
            hooks.append(getattr(net, f"conv{i}").register_forward_hook(fn))
        with torch.no_grad():
            out = net(x)
        for h in hooks:
            h.remove()
        big = shape[2] * shape[3] > 64 * 64
        rec = dict(skip=int(skip), seed=seed, power_iterations=iters, digest=sd_digest(sd), input=x.numpy(),
                   out=out.numpy(), **{f"tap_{k}": sample(v, big) for k, v in taps.items()})
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **rec)
        print(f"{name}: out {tuple(out.shape)} max|out| {out.abs().max().item():.4g} -> {os.path.getsize(path) / 1e3:.0f} kB")
    inv = {k: [list(v.shape), str(v.dtype).replace("torch.", "")]
           for k, v in mod.UNetDiscriminatorSN(3).state_dict().items()}
    text = json.dumps(inv, sort_keys=True, separators=(",", ":")) + "\n"
    with gzip.GzipFile(os.path.join(OUT, "reference_state_dict_disc.json.gz"), "wb", compresslevel=9, mtime=0) as f:
        f.write(text.encode())


if __name__ == "__main__":
    main()
