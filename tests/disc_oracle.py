"""Functional ATen restatement of UNetDiscriminatorSN.forward in eval mode (discriminator_arch.py): the spectral-norm
weights are formed explicitly, W = weight_orig / sigma with sigma = u . (W_mat v), no power iteration."""
import torch
import torch.nn.functional as F


def sigma(sd, name):
    w = sd[f"{name}.weight_orig"]
    return torch.dot(sd[f"{name}.weight_u"], torch.mv(w.reshape(w.shape[0], -1), sd[f"{name}.weight_v"]))


def forward(sd, x, skip_connection=True, taps=None):
    """x [B,3,H,W] -> [B,1,H,W].  ``taps`` (dict) receives every conv's output before its activation, keyed conv0 ...
    conv9 (what a forward hook on the reference's conv modules sees)."""
    taps = {} if taps is None else taps

    def conv(i, t, stride=1):
        name = f"conv{i}"
        if f"{name}.weight_orig" in sd:
            y = F.conv2d(t, sd[f"{name}.weight_orig"] / sigma(sd, name), stride=stride, padding=1)
        else:
            y = F.conv2d(t, sd[f"{name}.weight"], sd[f"{name}.bias"], padding=1)
        taps[name] = y
        return y

    lrelu = lambda t: F.leaky_relu(t, negative_slope=0.2)
    up = lambda t: F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=False)
    x0 = lrelu(conv(0, x))
    x1 = lrelu(conv(1, x0, 2))
    x2 = lrelu(conv(2, x1, 2))
    x3 = lrelu(conv(3, x2, 2))
    x4 = lrelu(conv(4, up(x3)))
    if skip_connection:
        x4 = x4 + x2
    x5 = lrelu(conv(5, up(x4)))
    if skip_connection:
        x5 = x5 + x1
    x6 = lrelu(conv(6, up(x5)))
    if skip_connection:
        x6 = x6 + x0
    out = lrelu(conv(7, x6))
    out = lrelu(conv(8, out))
    return conv(9, out)
