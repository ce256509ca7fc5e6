"""CPU oracle of the HQ stage's semantic loss (TEST INFRASTRUCTURE ONLY): the VGG19 relu4_4 extractor and
semantic_loss = mse(ReLU(conv_semantic(z_quant)), vgg_feat), restated in ATen functional ops on top of
oracle/femasr_oracle.py's encode_and_decode.  Pinned against the unmodified reference by tests/golden/semantic/*.npz
(tests/golden/make_golden_semantic.py) in tests/test_semantic.py.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from femasr_b200.spec import VGG_CONVS
from oracle import femasr_oracle as O

POOL_BEFORE = ("conv2_1", "conv3_1", "conv4_1")      # vgg_arch.py:27-32: pool1..pool3 in front of these


def vgg_relu4_4(sd, x: torch.Tensor) -> torch.Tensor:
    """VGGFeatureExtractor(['relu4_4']).forward (vgg_arch.py:141-163, use_input_norm=True, range_norm=False):
    (x - mean) / std, then VGG19 features conv1_1 ... relu4_4 (3x3 pad 1 convs + ReLU, MaxPool2d(2, 2))."""
    h = (x - sd["vgg_feat_extractor.mean"]) / sd["vgg_feat_extractor.std"]
    for name, _ci, _co in VGG_CONVS:
        if name in POOL_BEFORE:
            h = F.max_pool2d(h, kernel_size=2, stride=2)
        p = f"vgg_feat_extractor.vgg_net.{name}"
        h = F.relu(F.conv2d(h, sd[p + ".weight"], sd[p + ".bias"], stride=1, padding=1))
    return h


def semantic_term(sd, z_quant: torch.Tensor, vgg_feat: torch.Tensor, taps: dict | None = None) -> torch.Tensor:
    """femasr_arch.py:344-347: F.mse_loss(conv_semantic(z_quant), vgg_feat), conv_semantic = Conv2d(512, 512, 1) + ReLU."""
    s = F.relu(F.conv2d(z_quant, sd["conv_semantic.0.weight"], sd["conv_semantic.0.bias"]))
    if s.shape != vgg_feat.shape:       # the reference raises from conv_semantic (channels) or mse_loss (sizes)
        raise RuntimeError(f"semantic loss: conv_semantic(z_quant) is {tuple(s.shape)}, relu4_4 is {tuple(vgg_feat.shape)}")
    if taps is not None:
        taps["semantic"] = s
    return F.mse_loss(s, vgg_feat)


def encode_and_decode(sd, x: torch.Tensor, scale: int, taps: dict | None = None, cb_scales=(32,), semantic: bool = False,
                      **kw):
    """femasr_oracle.encode_and_decode plus, with ``semantic``, the semantic loss of femasr_arch.py:318-320, 344-347, 372
    in place of codebook_loss * 0.  z_quant is the quantiser's output, taken before the use_quantize override (:349-350),
    re-derived from the tapped z by the same deterministic vector_quantize."""
    t = {} if taps is None else taps
    out, loss, sem, idx = O.encode_and_decode(sd, x, scale, t, cb_scales=cb_scales, **kw)
    if not semantic:
        return out, loss, sem, idx
    vgg = vgg_relu4_4(sd, x)
    t["vgg"] = vgg
    if len(cb_scales) != 1:             # a second codebook sits at 64 or 128: its z_quant never matches relu4_4's size
        raise RuntimeError("semantic loss: only a single codebook at 32 meets relu4_4")
    z_quant = O.vector_quantize(sd["quantize_group.0.embedding.weight"], t["z"], None, scale != 1)[0]
    return out, loss, semantic_term(sd, z_quant, vgg, t), idx
