"""CPU restatement of femasr_psnr / femasr_ssim (include/femasr_b200.h): the Y channel in fp32 in the kernels' operation
order (numpy float32, one rounding per operation, so it matches the device bit for bit), PSNR with the difference in fp32
and the mean of squares in fp64, SSIM as one fp64 conv2d with the 2-D outer-product Gaussian window (not a separable
one).  Inputs [B,3,H,W] fp32 in [0, 1]; returns [B] fp32."""
import numpy as np
import torch
import torch.nn.functional as F


def y_channel(x: torch.Tensor, color_space: str) -> np.ndarray:
    """[B,3,H,W] fp32 -> [B,1,H,W] numpy float32."""
    r, g, b = (x[:, c:c + 1].numpy().astype(np.float32) for c in range(3))
    f = np.float32
    if color_space == "yiq":
        return (f(0.299) * r + f(0.587) * g) + f(0.114) * b
    t = (f(65.481) * r + f(128.553) * g) + f(24.966) * b
    return (t + f(16.0)) / f(255.0)


def gaussian_1d() -> torch.Tensor:
    w = torch.tensor([np.exp(-float((i - 5) ** 2) / (2.0 * 1.5 * 1.5)) for i in range(11)], dtype=torch.float64)
    s = 0.0
    for v in w.tolist():
        s += v
    return w / s


def _crop(t, c):
    return t[..., c:t.shape[-2] - c, c:t.shape[-1] - c] if c else t


def psnr(x, y, test_y_channel=False, crop_border=0, color_space="yiq"):
    if test_y_channel:
        a, b = torch.from_numpy(y_channel(x, color_space)), torch.from_numpy(y_channel(y, color_space))
    else:
        a, b = x.float(), y.float()
    d = _crop(a - b, crop_border).double()
    mse = d.pow(2).flatten(1).mean(1)
    return (10.0 * torch.log10(1.0 / (mse + 1e-8))).float()


def ssim_maps(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """a, b [B,C,H,W] fp64 at data range 255 -> the SSIM map [B,C,H-10,W-10] (fp64 conv2d, 'valid')."""
    g = gaussian_1d()
    win = torch.outer(g, g).view(1, 1, 11, 11)
    B, C, H, W = a.shape

    def filt(t):
        return F.conv2d(t.reshape(B * C, 1, H, W), win).view(B, C, H - 10, W - 10)

    C1, C2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2
    mx, my = filt(a), filt(b)
    vx, vy, cxy = filt(a * a) - mx * mx, filt(b * b) - my * my, filt(a * b) - mx * my
    cs = torch.relu((2 * cxy + C2) / (vx + vy + C2))
    return (2 * mx * my + C1) / (mx * mx + my * my + C1) * cs


def ssim(x, y, test_y_channel=True, crop_border=0, color_space="yiq"):
    if test_y_channel:
        a = torch.from_numpy(np.rint(y_channel(x, color_space) * np.float32(255.0)))
        b = torch.from_numpy(np.rint(y_channel(y, color_space) * np.float32(255.0)))
    else:
        a, b = x.float() * 255.0, y.float() * 255.0
    m = ssim_maps(_crop(a, crop_border).double(), _crop(b, crop_border).double())
    return m.flatten(1).mean(1).float()
