"""Float64 restatement of the reference's evaluation metrics (test infrastructure, never imported by the product):
the record {l1, psnr, psnr_all, ssim} of gab200_image_metrics for one view.

  l1       = mean |x - y|                                               (utils/loss_utils.py:17-18)
  psnr     = mean over the channels of 20 log10(1 / sqrt(MSE_c))       (utils/image_utils.py:18-20 on [3,H,W], .mean())
  psnr_all = 20 log10(1 / sqrt(MSE over all values))                   (the same function on [1,3,H,W], metrics.py)
  ssim     = mean SSIM map, 11x11 Gaussian window (sigma 1.5), zero padding, C1 = 0.01^2, C2 = 0.03^2
             (utils/loss_utils.py:23-63), through F.conv2d in float64 with the reference's float32 2-D window
             (oracle/loss.py window_2d)

x is the float render clamped to [0, 1] (train.py:277) or the display image's bytes / 255 (metrics.py), y the
ground-truth bytes / 255.  tests/test_oracle_metrics.py checks this against tests/golden/metrics_vectors.npz, which
make_golden_metrics.py produced with the reference's own functions."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import loss as ol


def inputs(render, gt_u8):
    """(x, y) as float64 (3,H,W) arrays: a float (3,H,W) render is clamped to [0, 1] (NaN stays NaN, as
    torch.clamp); a uint8 (H,W,3) display image is read as value/255."""
    r = np.asarray(render)
    if r.dtype == np.uint8:
        x = r.transpose(2, 0, 1).astype(np.float64) / 255
    else:
        x = r.astype(np.float64)
        x = np.where(np.isnan(x), x, np.clip(x, 0.0, 1.0))
    return x, np.asarray(gt_u8).astype(np.float64) / 255


def ssim_map(x, y):
    w2 = torch.from_numpy(ol.window_2d())[None, None].expand(3, 1, 11, 11).contiguous()
    X, Y = torch.from_numpy(np.ascontiguousarray(x))[None], torch.from_numpy(np.ascontiguousarray(y))[None]
    conv = lambda a: F.conv2d(a, w2, padding=5, groups=3)  # noqa: E731
    mu1, mu2 = conv(X), conv(Y)
    mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1, s2, s12 = conv(X * X) - mu1_sq, conv(Y * Y) - mu2_sq, conv(X * Y) - mu12
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    return (((2 * mu12 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s1 + s2 + C2)))[0].numpy()


def _psnr(mse):
    with np.errstate(divide="ignore"):
        return -10.0 * np.log10(mse)   # 20 log10(1 / sqrt(mse)); mse 0 -> +inf


def metrics(render, gt_u8):
    """np.float64 array [l1, psnr, psnr_all, ssim]."""
    x, y = inputs(render, gt_u8)
    d = x - y
    mse_c = (d * d).reshape(3, -1).mean(axis=1)
    return np.array([np.abs(d).mean(), _psnr(mse_c).mean(), _psnr((d * d).mean()), ssim_map(x, y).mean()])
