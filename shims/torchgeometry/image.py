"""tgm.image.GaussianBlur((kh,kw),(sy,sx)) — depth-wise separable Gaussian, zero padding k//2, taps normalised to sum 1."""
import torch
import torch.nn as nn
import torch.nn.functional as F


def _taps(k, sigma, device):
    x = torch.arange(k, dtype=torch.float32, device=device) - k // 2
    g = torch.exp(-(x * x) / (2.0 * sigma * sigma))
    return g / g.sum()


class GaussianBlur(nn.Module):
    def __init__(self, kernel_size, sigma):
        super().__init__()
        self.kernel_size = tuple(kernel_size)
        self.sigma = tuple(float(s) for s in sigma)

    def forward(self, x):
        kh, kw = self.kernel_size
        sy, sx = self.sigma
        if x.is_cuda and kh == kw and sy == sx and x.dtype == torch.float32:
            import hrv_loader
            hrv_loader.load()
            from hrviton_b200 import ops
            return ops.gaussian_blur(x, kh, sy)  # hrv_gaussian_blur (sm_90a kernel)
        c = x.shape[1]
        gx, gy = _taps(kw, sx, x.device).to(x.dtype), _taps(kh, sy, x.device).to(x.dtype)
        x = F.conv2d(x, gx.view(1, 1, 1, kw).expand(c, 1, 1, kw), padding=(0, kw // 2), groups=c)
        return F.conv2d(x, gy.view(1, 1, kh, 1).expand(c, 1, kh, 1), padding=(kh // 2, 0), groups=c)
