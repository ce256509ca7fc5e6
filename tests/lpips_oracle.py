"""Functional ATen restatement of LPIPS v0.1 (the lpips package's LPIPS.forward with lpips=True, spatial=False, eval
mode), from the definition: ScalingLayer, torchvision's alexnet / vgg16 features up to the five ReLU taps,
normalize_tensor, the lin layers' 1x1 no-bias conv and spatial_average."""
import torch
import torch.nn.functional as F

# torchvision features index of every conv, its padding / stride, whether a max-pool precedes it, and whether its ReLU
# output is an LPIPS tap
ALEX = [(0, 2, 4, False, True), (3, 2, 1, True, True), (6, 1, 1, True, True), (8, 1, 1, False, True),
        (10, 1, 1, False, True)]
VGG = [(0, 1, 1, False, False), (2, 1, 1, False, True), (5, 1, 1, True, False), (7, 1, 1, False, True),
       (10, 1, 1, True, False), (12, 1, 1, False, False), (14, 1, 1, False, True), (17, 1, 1, True, False),
       (19, 1, 1, False, False), (21, 1, 1, False, True), (24, 1, 1, True, False), (26, 1, 1, False, False),
       (28, 1, 1, False, True)]
SLICE = {"alex": {0: 1, 3: 2, 6: 3, 8: 4, 10: 5},
         "vgg": {0: 1, 2: 1, 5: 2, 7: 2, 10: 3, 12: 3, 14: 3, 17: 4, 19: 4, 21: 4, 24: 5, 26: 5, 28: 5}}


def features(net, sd, x):
    """The five ReLU taps of x (already scaled)."""
    taps = []
    for i, pad, stride, pool, tap in (ALEX if net == "alex" else VGG):
        if pool:
            x = F.max_pool2d(x, 3, 2) if net == "alex" else F.max_pool2d(x, 2, 2)
        p = f"net.slice{SLICE[net][i]}.{i}"
        x = F.relu(F.conv2d(x, sd[p + ".weight"], sd[p + ".bias"], stride=stride, padding=pad))
        if tap:
            taps.append(x)
    return taps


def head(f0, f1, w):
    """r = spatial_average(lin((normalize_tensor(f0) - normalize_tensor(f1))^2)) [B,1,1,1]."""
    n0 = f0 / (torch.sqrt(torch.sum(f0 ** 2, dim=1, keepdim=True)) + 1e-10)
    n1 = f1 / (torch.sqrt(torch.sum(f1 ** 2, dim=1, keepdim=True)) + 1e-10)
    return F.conv2d((n0 - n1) ** 2, w).mean([2, 3], keepdim=True)


def forward(net, sd, in0, in1, retPerLayer=False, normalize=False):
    if normalize:
        in0, in1 = 2 * in0 - 1, 2 * in1 - 1
    shift, scale = sd["scaling_layer.shift"], sd["scaling_layer.scale"]
    f0 = features(net, sd, (in0 - shift) / scale)
    f1 = features(net, sd, (in1 - shift) / scale)
    res = [head(a, b, sd[f"lin{k}.model.1.weight"]) for k, (a, b) in enumerate(zip(f0, f1))]
    val = res[0]
    for r in res[1:]:
        val = val + r
    return (val, res) if retPerLayer else val
