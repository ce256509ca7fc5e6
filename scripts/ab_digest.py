#!/usr/bin/env python
"""Digest of the public-surface outputs, the launch count and the per-kernel (launches, flops) profile of a set of generator,
discriminator and LPIPS cases on both GEMM paths, with the library selected by FEMASR_LIB: two library builds that claim to
be arithmetic-identical (an epilogue / scheduling / host-graph refactor) must print the same JSON.
    FEMASR_LIB=... python scripts/ab_digest.py > a.json
Runs eagerly (FEMASR_CUDA_GRAPH=0) so that every launch is counted and profiled."""
import hashlib
import json
import os
import sys
import warnings

os.environ.setdefault("FEMASR_CUDA_GRAPH", "0")

import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from basicsr.archs.discriminator_arch import UNetDiscriminatorSN  # noqa: E402
from basicsr.archs.femasr_arch import FeMaSRNet  # noqa: E402
from femasr_b200.lib import TAP_STAGES  # noqa: E402
from femasr_b200.lpips import LPIPS  # noqa: E402
from femasr_b200.spec import random_disc_state_dict, random_lpips_state_dict, random_state_dict  # noqa: E402


def dig(t):
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()[:16]


def rand(shape, seed):
    return torch.rand(*shape, generator=torch.Generator().manual_seed(seed))


def make(dev, gp, scale, cb, sem=False):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)          # no VGG file: the weights come from the state dict
        net = FeMaSRNet(codebook_params=cb, LQ_stage=scale != 1, scale_factor=scale, use_semantic_loss=sem, gemm_path=gp)
    sd = random_state_dict(scale, cb[0][2], seed=3, init="default", n_e=cb[0][1], codebooks=cb, semantic=sem)
    net.load_state_dict(sd, strict=False)
    return net.to(dev).eval()


def case(out, key, net, dev, fn):
    """out[key] = output digests / values, the last forward's launch count and {kernel: [launches, flops]}."""
    eng = net._native(dev)
    eng.set_profile(True)
    vals = fn()
    prof = eng.profile()
    eng.set_profile(False)
    vals = [dig(v) if torch.is_tensor(v) and v.numel() > 1 else float(v) for v in vals]
    out[key] = {"out": vals, "launches": eng.last_launch_count(),
                "profile": {k: [v["launches"], v["flops"]] for k, v in sorted(prof.items())}}


def fwd(net, x, gt=None):
    y, loss, sem, idx = net(x, gt_indices=gt)
    return [y, loss, sem, *idx]


def lpips_fwd(net, x0, x1, normalize):
    d, r = net(x0, x1, retPerLayer=True, normalize=normalize)
    return [d, *r]


def taps_fwd(eng, x):
    y, loss, idx, taps = eng.forward(x, taps=list(TAP_STAGES))
    return [y, loss, idx, *(taps[k] for k in sorted(taps))]


def main():
    dev = torch.device("cuda", 0)
    out = {}
    for gp in (0, 1):
        for scale, cb, shapes in ((4, [[32, 1024, 256]], [(4, 128, 128), (1, 96, 160)]), (2, [[32, 1024, 512]], [(2, 64, 96)])):
            net = make(dev, gp, scale, cb)
            for (b, h, w) in shapes:
                x = rand((b, 3, h, w), 5).to(dev)
                case(out, f"gp{gp}/x{scale}_fwd_{b}x{h}x{w}", net, dev, lambda: fwd(net, x))
            x = rand((1, 3, 75, 52), 6).to(dev)      # ragged: edge tiles everywhere
            case(out, f"gp{gp}/x{scale}_test_75x52", net, dev, lambda: [net.test(x)])
            if scale == 4:
                x = rand((1, 3, 200, 136), 7).to(dev)
                case(out, f"gp{gp}/x4_tile_200x136", net, dev, lambda: [net.test_tile(x, tile_size=96, tile_pad=8)])
                x = rand((2, 3, 64, 96), 8).to(dev)
                idx = net(x)[3][0]
                case(out, f"gp{gp}/x4_decode_indices", net, dev, lambda: [net.decode_indices(idx)])
                eng = net._native(dev)
                x = rand((1, 3, 64, 64), 9).to(dev)
                case(out, f"gp{gp}/x4_fwd_all_taps", net, dev, lambda: taps_fwd(eng, x))
        x = rand((2, 3, 64, 96), 10).to(dev)
        net = make(dev, gp, 1, [[32, 1024, 512]])
        case(out, f"gp{gp}/hq_e512_fwd", net, dev, lambda: fwd(net, x))
        net = make(dev, gp, 1, [[32, 1024, 512]], sem=True)
        net.use_semantic_loss = True
        case(out, f"gp{gp}/hq_e512_semantic", net, dev, lambda: fwd(net, x))
        for scale, cb, shape in ((4, [[32, 1024, 256], [64, 512, 128]], (2, 3, 64, 64)),
                                 (2, [[32, 1024, 512], [64, 512, 256], [128, 256, 128]], (1, 3, 64, 96))):
            net = make(dev, gp, scale, cb)
            x = rand(shape, 11).to(dev)
            g = torch.Generator().manual_seed(12)
            gt = [torch.randint(0, n_e, i.shape, generator=g).to(dev) for i, (_s, n_e, _e) in zip(net(x)[3], cb)]
            case(out, f"gp{gp}/x{scale}_cb{len(cb)}_fwd", net, dev, lambda: fwd(net, x))
            case(out, f"gp{gp}/x{scale}_cb{len(cb)}_fwd_gt", net, dev, lambda: fwd(net, x, gt))
        x = rand((2, 3, 64, 96), 13).to(dev)
        for skip in (0, 1):
            net = UNetDiscriminatorSN(3, skip_connection=skip, gemm_path=gp)
            net.load_state_dict(random_disc_state_dict(14), strict=True)
            net = net.to(dev).eval()
            case(out, f"gp{gp}/disc_skip{skip}", net, dev, lambda: [net(x)])
        for name, shape in (("alex", (2, 3, 67, 93)), ("vgg", (2, 3, 64, 96))):
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", UserWarning)      # no weight files: seeded untrained tensors below
                net = LPIPS(name, gemm_path=gp)
            net.load_state_dict(random_lpips_state_dict(name, seed=15), strict=True)
            net = net.to(dev)
            x0, x1 = rand(shape, 16).to(dev), rand(shape, 17).to(dev)
            for normalize in (False, True):
                a, b = (x0, x1) if normalize else (2 * x0 - 1, 2 * x1 - 1)    # [0, 1] with normalize, else [-1, 1]
                case(out, f"gp{gp}/lpips_{name}_normalize{int(normalize)}", net, dev, lambda: lpips_fwd(net, a, b, normalize))
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
