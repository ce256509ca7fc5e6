"""Parameter inventory of the in-scope FeMaSRNet graph and seeded random weights for it.

The names/shapes are the reference's ``state_dict`` contract (SURVEY.md section 8b; built by
femasr_arch.py:216-309, fema_utils.py:65-99, network_swinir.py:65-145,164-214,419-482) so that a
checkpoint written by the reference loads here and vice versa.  ``tests/test_boundary.py`` checks
this list against the reference's own ``state_dict()`` when /root/reference is present.
"""
from __future__ import annotations

import hashlib
import math
from typing import Dict, List, Tuple

import torch

CHANNELS = {8: 256, 16: 256, 32: 256, 64: 256, 128: 128, 256: 64, 512: 32}   # femasr_arch.py:244-252
GT_RES = 256
CB_SCALE = 32
WINDOW = 8
HEADS = 8
SWIN_DIM = 256
SWIN_DEPTH = 6
N_RSTB = 4
MLP_RATIO = 4
SWIN_INIT_RES = 32        # SwinLayers default input_resolution=(32,32), femasr_arch.py:115


def encode_depth(scale: int) -> int:
    """femasr_arch.py:256."""
    return int(math.log2(GT_RES // scale // CB_SCALE))


def _res_block(p: str, c: int) -> List[Tuple[str, tuple, str, int]]:
    return [
        (f"{p}.conv.0.norm.weight", (c,), "norm_w", 0), (f"{p}.conv.0.norm.bias", (c,), "norm_b", 0),
        (f"{p}.conv.2.weight", (c, c, 3, 3), "w", c * 9), (f"{p}.conv.2.bias", (c,), "b", c * 9),
        (f"{p}.conv.3.norm.weight", (c,), "norm_w", 0), (f"{p}.conv.3.norm.bias", (c,), "norm_b", 0),
        (f"{p}.conv.5.weight", (c, c, 3, 3), "w", c * 9), (f"{p}.conv.5.bias", (c,), "b", c * 9),
    ]


def _conv(p: str, ci: int, co: int, k: int) -> List[Tuple[str, tuple, str, int]]:
    return [(f"{p}.weight", (co, ci, k, k), "w", ci * k * k), (f"{p}.bias", (co,), "b", ci * k * k)]


def _linear(p: str, ci: int, co: int) -> List[Tuple[str, tuple, str, int]]:
    return [(f"{p}.weight", (co, ci), "w", ci), (f"{p}.bias", (co,), "b", ci)]


def normalize_codebooks(codebooks, n_e: int = 1024, e_dim: int = 256):
    """[(scale, n_e, e_dim), ...] as ints (the reference's ``codebook_params`` rows, femasr_arch.py:231-235).
    The first codebook must sit at scale 32 (it fixes the encoder/decoder depth, :255-256); further ones at
    strictly increasing decoder resolutions 64 / 128 (:329-331)."""
    if codebooks is None:
        return [(CB_SCALE, int(n_e), int(e_dim))]
    cbs = [(int(s), int(n), int(e)) for s, n, e in codebooks]
    if not cbs or cbs[0][0] != CB_SCALE:
        raise NotImplementedError("the first codebook must be at scale 32")
    scales = [s for s, _, _ in cbs]
    if any(s not in (32, 64, 128) for s in scales) or scales != sorted(set(scales)):
        raise NotImplementedError(f"codebook scales must be an increasing subset of 32, 64, 128, got {scales}")
    return cbs


# VGG19 `features` up to relu4_4 (vgg_arch.py:27-32, 55-139): conv name, Cin, Cout; every conv is 3x3 pad 1
VGG_CONVS = [("conv1_1", 3, 64), ("conv1_2", 64, 64), ("conv2_1", 64, 128), ("conv2_2", 128, 128),
             ("conv3_1", 128, 256), ("conv3_2", 256, 256), ("conv3_3", 256, 256), ("conv3_4", 256, 256),
             ("conv4_1", 256, 512), ("conv4_2", 512, 512), ("conv4_3", 512, 512), ("conv4_4", 512, 512)]
# index of each conv in torchvision's vgg19().features (the layout of vgg19-dcbb9e9d.pth)
VGG_TORCHVISION_INDEX = [0, 2, 5, 7, 10, 12, 14, 16, 19, 21, 23, 25]
VGG_MEAN = (0.485, 0.456, 0.406)       # vgg_arch.py:133-136
VGG_STD = (0.229, 0.224, 0.225)


def semantic_spec() -> List[Tuple[str, tuple, str, int]]:
    """The 28 tensors use_semantic_loss=True adds (femasr_arch.py:301-309): conv_semantic = Sequential(Conv2d(512, 512, 1),
    ReLU) and VGGFeatureExtractor(['relu4_4']) with its mean / std buffers."""
    spec = _conv("conv_semantic.0", 512, 512, 1)
    spec += [("vgg_feat_extractor.mean", (1, 3, 1, 1), "vgg_mean", 0), ("vgg_feat_extractor.std", (1, 3, 1, 1), "vgg_std", 0)]
    for name, ci, co in VGG_CONVS:
        p = f"vgg_feat_extractor.vgg_net.{name}"
        spec += [(f"{p}.weight", (co, ci, 3, 3), "vgg_w", co * 9), (f"{p}.bias", (co,), "vgg_b", co * 9)]
    return spec


def param_spec(scale: int, e_dim: int, n_e: int = 1024, in_channel: int = 3, codebooks=None, semantic: bool = False):
    """Ordered [(name, shape, kind, fan_in)].  scale 4 | 2: LQ_stage=True;
    scale 1: the HQ autoencoder (LQ_stage=False, femasr_arch.py:241: scale_factor forced to 1; no Swin, no up branches).
    ``codebooks`` = [(scale, n_e, e_dim), ...] for the multi-scale variant (femasr_arch.py:280-299); default: one
    codebook (32, n_e, e_dim).  ``semantic``: append the use_semantic_loss tensors (semantic_spec()).

    kind: w | b (kaiming-uniform bound 1/sqrt(fan_in)), norm_w | norm_b, rpb (trunc-normal .02),
    rpi | mask (buffers), codebook (U(+-1/n_e)), vgg_w | vgg_b (torchvision's VGG init: N(0, 2 / (9 Cout)) | 0;
    fan_in carries 9 Cout), vgg_mean | vgg_std (the extractor's constant buffers).
    """
    d = encode_depth(scale)
    res = GT_RES // scale
    spec: List[Tuple[str, tuple, str, int]] = []
    enc = "multiscale_encoder"
    spec += _conv(f"{enc}.in_conv", in_channel, CHANNELS[res], 4)
    for i in range(d):
        ci, co = CHANNELS[res], CHANNELS[res // 2]
        spec += _conv(f"{enc}.blocks.{i}.0", ci, co, 3)
        spec += _res_block(f"{enc}.blocks.{i}.1", co) + _res_block(f"{enc}.blocks.{i}.2", co)
        res //= 2
    C = SWIN_DIM
    hq = scale == 1
    for r in range(0 if hq else N_RSTB):
        for b in range(SWIN_DEPTH):
            p = f"{enc}.blocks.{d}.swin_blks.{r}.residual_group.blocks.{b}"
            if b % 2 == 1:
                nw = (SWIN_INIT_RES // WINDOW) ** 2
                spec.append((f"{p}.attn_mask", (nw, WINDOW ** 2, WINDOW ** 2), "mask", 0))
            spec += [(f"{p}.norm1.weight", (C,), "norm_w", 0), (f"{p}.norm1.bias", (C,), "norm_b", 0),
                     (f"{p}.attn.relative_position_bias_table", ((2 * WINDOW - 1) ** 2, HEADS), "rpb", 0),
                     (f"{p}.attn.relative_position_index", (WINDOW ** 2, WINDOW ** 2), "rpi", 0)]
            spec += _linear(f"{p}.attn.qkv", C, 3 * C) + _linear(f"{p}.attn.proj", C, C)
            spec += [(f"{p}.norm2.weight", (C,), "norm_w", 0), (f"{p}.norm2.bias", (C,), "norm_b", 0)]
            spec += _linear(f"{p}.mlp.fc1", C, MLP_RATIO * C) + _linear(f"{p}.mlp.fc2", MLP_RATIO * C, C)
        spec += _conv(f"{enc}.blocks.{d}.swin_blks.{r}.conv", C, C, 3)
    for j in (() if hq else (d + 1, d + 2)):
        ci, co = CHANNELS[res], CHANNELS[res * 2]
        spec += _conv(f"{enc}.blocks.{j}.1", ci, co, 3)
        spec += _res_block(f"{enc}.blocks.{j}.2", co) + _res_block(f"{enc}.blocks.{j}.3", co)
        res *= 2
    for i in range(3):
        r = GT_RES // 8 * 2 ** i
        ci, co = CHANNELS[r], CHANNELS[r * 2]
        spec += _conv(f"decoder_group.{i}.block.1", ci, co, 3)
        spec += _res_block(f"decoder_group.{i}.block.2", co) + _res_block(f"decoder_group.{i}.block.3", co)
    spec += _conv("out_conv", CHANNELS[GT_RES], 3, 3)
    cbs = normalize_codebooks(codebooks, n_e, e_dim)
    for k, (cs, ne, ed) in enumerate(cbs):                 # femasr_arch.py:280-299
        ch = CHANNELS[cs]
        spec.append((f"quantize_group.{k}.embedding.weight", (ne, ed), "codebook", ne))
        spec += _conv(f"before_quant_group.{k}", ch if k == 0 else 2 * ch, ed, 1)
        spec += _conv(f"after_quant_group.{k}.conv", ed if k == 0 else cbs[k - 1][2] + ed, ch, 3)
    if semantic:
        spec += semantic_spec()
    return spec


def relative_position_index(ws: int = WINDOW) -> torch.Tensor:
    """The fixed [ws^2, ws^2] int64 buffer of network_swinir.py:91-101."""
    ar = torch.arange(ws)
    cy, cx = torch.meshgrid(ar, ar, indexing="ij")
    cy, cx = cy.flatten(), cx.flatten()
    dy = cy[:, None] - cy[None, :] + ws - 1
    dx = cx[:, None] - cx[None, :] + ws - 1
    return dy * (2 * ws - 1) + dx


def shift_attn_mask(H: int, W: int, ws: int = WINDOW, shift: int = WINDOW // 2) -> torch.Tensor:
    """0 / -100 shifted-window mask [nW, ws^2, ws^2] (what network_swinir.py:216-237 builds),
    computed from region ids: rows/cols in [0,H-ws) -> 0, [H-ws,H-shift) -> 1, [H-shift,H) -> 2."""
    def region(n):
        r = torch.zeros(n, dtype=torch.int64)
        r[n - ws:n - shift] = 1
        r[n - shift:] = 2
        return r
    ids = region(H)[:, None] * 3 + region(W)[None, :]
    ids = ids.view(H // ws, ws, W // ws, ws).permute(0, 2, 1, 3).reshape(-1, ws * ws)
    diff = ids[:, None, :] != ids[:, :, None]
    return torch.where(diff, torch.tensor(-100.0), torch.tensor(0.0))


def _gen(seed: int, name: str) -> torch.Generator:
    h = hashlib.sha256(f"{seed}:{name}".encode()).digest()
    g = torch.Generator()
    g.manual_seed(int.from_bytes(h[:7], "little"))
    return g


def random_state_dict(scale: int, e_dim: int, seed: int = 0, init: str = "default",
                      n_e: int = 1024, codebooks=None, semantic: bool = False) -> Dict[str, torch.Tensor]:
    """Seeded random weights with the reference's default-init distributions.

    Each tensor is drawn from its own generator keyed by (seed, name), so the dict is reproducible
    anywhere without the reference.  ``init='default'``: exactly the reference's distributions
    (conv/linear U(+-1/sqrt(fan_in)); GN/LN weight 1 bias 0; rel-pos table trunc-normal(.02),
    network_swinir.py:111; codebook U(+-1/n_e), femasr_arch.py:33).  ``init='perturbed'``: norm affine
    parameters and the codebook get non-trivial values so tests exercise them.  ``semantic``: also the use_semantic_loss
    tensors; VGG weights N(0, 2 / (9 Cout)) like torchvision's VGG init, VGG biases 0 (default) or small random values
    (perturbed), conv_semantic kaiming-uniform.
    """
    sd: Dict[str, torch.Tensor] = {}
    for name, shape, kind, fan_in in param_spec(scale, e_dim, n_e, codebooks=codebooks, semantic=semantic):
        g = _gen(seed, name)
        if kind in ("w", "b"):
            bound = 1.0 / math.sqrt(fan_in)
            t = (torch.rand(shape, generator=g) * 2 - 1) * bound
        elif kind == "norm_w":
            t = torch.ones(shape)
            if init == "perturbed":
                t = t + 0.2 * torch.randn(shape, generator=g)
        elif kind == "norm_b":
            t = torch.zeros(shape)
            if init == "perturbed":
                t = 0.2 * torch.randn(shape, generator=g)
        elif kind == "rpb":
            std = 0.02 if init == "default" else 0.5
            t = (torch.randn(shape, generator=g) * std).clamp_(-2 * std, 2 * std)
        elif kind == "rpi":
            t = relative_position_index()
        elif kind == "mask":
            t = shift_attn_mask(SWIN_INIT_RES, SWIN_INIT_RES)
        elif kind == "codebook":
            if init == "default":
                t = (torch.rand(shape, generator=g) * 2 - 1) / fan_in      # fan_in carries this codebook's n_e
            else:
                t = torch.randn(shape, generator=g) * 0.5
        elif kind in ("vgg_w", "vgg_b", "vgg_mean", "vgg_std"):
            t = vgg_init(shape, kind, fan_in, g, init)
        else:
            raise ValueError(kind)
        sd[name] = t.contiguous()
    return sd


def disc_spec(num_in_ch: int = 3, num_feat: int = 64) -> List[Tuple[str, tuple, str, int]]:
    """UNetDiscriminatorSN's 28 state_dict tensors (discriminator_arch.py): conv0 / conv9 weight + bias, and for the
    spectral_norm convs conv1 ... conv8 weight_orig [Cout,Cin,k,k], weight_u [Cout], weight_v [Cin*k*k].
    kind: w | b (kaiming-uniform, fan_in), sn_w (weight_orig), sn_u | sn_v (fan_in carries their length)."""
    F = num_feat
    convs = [("conv1", F, 2 * F, 4), ("conv2", 2 * F, 4 * F, 4), ("conv3", 4 * F, 8 * F, 4), ("conv4", 8 * F, 4 * F, 3),
             ("conv5", 4 * F, 2 * F, 3), ("conv6", 2 * F, F, 3), ("conv7", F, F, 3), ("conv8", F, F, 3)]
    spec = _conv("conv0", num_in_ch, F, 3)
    for name, ci, co, k in convs:
        spec += [(f"{name}.weight_orig", (co, ci, k, k), "sn_w", ci * k * k), (f"{name}.weight_u", (co,), "sn_u", co),
                 (f"{name}.weight_v", (ci * k * k,), "sn_v", ci * k * k)]
    return spec + _conv("conv9", F, 1, 3)


def power_iterate(w: torch.Tensor, u: torch.Tensor, v: torch.Tensor, n: int):
    """n steps of torch.nn.utils.spectral_norm's power iteration on W = w.reshape(Cout, -1) (v = normalize(W^T u),
    u = normalize(W v)), in fp64."""
    wm = w.double().reshape(w.shape[0], -1)
    u, v = u.double(), v.double()
    for _ in range(n):
        v = torch.nn.functional.normalize(wm.t() @ u, dim=0, eps=1e-12)
        u = torch.nn.functional.normalize(wm @ v, dim=0, eps=1e-12)
    return u.float(), v.float()


def random_disc_state_dict(seed: int = 0, power_iterations: int = 30) -> Dict[str, torch.Tensor]:
    """Seeded UNetDiscriminatorSN weights: conv weights and biases U(+-1/sqrt(fan_in)) like nn.Conv2d's default init, u
    and v drawn like torch's spectral_norm (normalize(randn)) and then power-iterated ``power_iterations`` times in fp64,
    which is what a trained checkpoint carries (the training-mode forward iterates once per step).  power_iterations=0
    gives the never-iterated u, v of a freshly constructed network."""
    sd: Dict[str, torch.Tensor] = {}
    for name, shape, kind, fan_in in disc_spec():
        g = _gen(seed, name)
        if kind in ("w", "b", "sn_w"):
            t = (torch.rand(shape, generator=g) * 2 - 1) / math.sqrt(fan_in)
        elif kind in ("sn_u", "sn_v"):
            t = torch.nn.functional.normalize(torch.randn(shape, generator=g), dim=0, eps=1e-12)
        else:
            raise ValueError(kind)
        sd[name] = t.contiguous()
    for name, _shape, kind, _f in disc_spec():
        if kind == "sn_w" and power_iterations:
            p = name[: -len(".weight_orig")]
            sd[f"{p}.weight_u"], sd[f"{p}.weight_v"] = power_iterate(sd[name], sd[f"{p}.weight_u"], sd[f"{p}.weight_v"],
                                                                      power_iterations)
    return sd


def vgg_init(shape, kind: str, fan_out: int, g: torch.Generator = None, init: str = "default") -> torch.Tensor:
    """VGG extractor tensors: torchvision's VGG init (kaiming-normal fan_out / relu: N(0, 2 / fan_out), bias 0; biases
    N(0, 0.01^2) for ``init='perturbed'``) and the ImageNet mean / std buffers."""
    if kind == "vgg_w":
        return torch.randn(shape, generator=g) * math.sqrt(2.0 / fan_out)
    if kind == "vgg_b":
        return torch.randn(shape, generator=g) * 0.01 if init == "perturbed" else torch.zeros(shape)
    if kind == "vgg_mean":
        return torch.tensor(VGG_MEAN).view(shape)
    if kind == "vgg_std":
        return torch.tensor(VGG_STD).view(shape)
    raise ValueError(kind)
