"""fp64 restatement of gaussian-splatting's image metrics (utils/image_utils.py psnr, utils/loss_utils.py ssim) over the
float32 images metrics.py reads (to_tensor: k / 255), the oracle of the device kernel (pixie_image_metrics).

    window(g)          (11, 11) 2D window: the outer product of the float32 1D window g, exact in fp64
    ssim(a, b, g)      mean SSIM map, zero padding 5 per channel, C1 = 0.01^2 and C2 = 0.03^2 as float32 constants
    psnr(a, b)         20 log10(1 / sqrt(mean((a - b)^2))) over 3 H W values; inf for identical images

a, b: (3, H, W) float32 arrays. The reference rounds each 2D window entry to float32 and runs float32 convolutions; the
tests bound how far its results lie from these.
"""
from __future__ import annotations

import numpy as np

C1 = float(np.float32(0.01 ** 2))
C2 = float(np.float32(0.03 ** 2))


def window(g) -> np.ndarray:
    g = np.asarray(g, np.float32).astype(np.float64)
    return np.outer(g, g)


def _filter(x: np.ndarray, w2: np.ndarray) -> np.ndarray:
    """Zero-padded 'same' correlation of each channel of x (C, H, W) with the (k, k) window."""
    k = w2.shape[0]
    r = k // 2
    C, H, W = x.shape
    p = np.zeros((C, H + 2 * r, W + 2 * r))
    p[:, r:r + H, r:r + W] = x
    out = np.zeros((C, H, W))
    for i in range(k):
        for j in range(k):
            out += w2[i, j] * p[:, i:i + H, j:j + W]
    return out


def ssim(a, b, g) -> float:
    x = np.asarray(a, np.float32).astype(np.float64)
    y = np.asarray(b, np.float32).astype(np.float64)
    w2 = window(g)
    mu1, mu2 = _filter(x, w2), _filter(y, w2)
    s11 = _filter(x * x, w2) - mu1 * mu1
    s22 = _filter(y * y, w2) - mu2 * mu2
    s12 = _filter(x * y, w2) - mu1 * mu2
    m = ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s11 + s22 + C2))
    return float(m.mean())


def psnr(a, b) -> float:
    d = np.asarray(a, np.float32).astype(np.float64) - np.asarray(b, np.float32).astype(np.float64)
    mse = float(np.mean(d * d))
    with np.errstate(divide="ignore"):
        return float(20 * np.log10(1.0 / np.sqrt(mse)))
