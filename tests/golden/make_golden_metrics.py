"""Generates tests/golden/metrics_vectors.npz by IMPORTING the real reference evaluation functions (utils/loss_utils.py
`l1_loss`, `ssim` and utils/image_utils.py `psnr`, under /root/reference, read-only) and running them on the CPU in
float32 and float64, in the two forms the reference evaluates a view:

  train   training_report (train.py:277-288): the float render clamped to [0, 1], the ground truth value/255, [3,H,W]
          tensors -- psnr() makes one PSNR per channel and .mean() averages them.
  metrics render.py + metrics.py (render.py:41, metrics.py:24-34,71-74): the render quantised with
          mul(255).add_(0.5).clamp_(0, 255) to the PNG's bytes, read back as value/255, [1,3,H,W] tensors -- psnr()
          makes one PSNR over all values.

Each record is {l1, psnr (per-channel mean), psnr_all (one MSE over all values), ssim} of that form's inputs.
image_utils imports matplotlib.cm (for error_map, which is not used here); matplotlib is not installed, so that one
module is stubbed.  The fixture travels to the GPU box; /root/reference does not.

    python tests/golden/make_golden_metrics.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, "/root/reference")
_mpl = sys.modules.setdefault("matplotlib", types.ModuleType("matplotlib"))
_mpl.cm = sys.modules.setdefault("matplotlib.cm", types.ModuleType("matplotlib.cm"))
from utils.image_utils import psnr  # noqa: E402  (REAL reference code)
from utils.loss_utils import l1_loss, ssim  # noqa: E402

CASES = {   # name: (seed, H, W); every W % 4 != 0 (the display image's rows are then not word-aligned)
    "a": (0, 45, 70),
    "b": (1, 33, 65),
    "c": (2, 37, 1),
}


def quantise(img):
    """render.py:41 -- the bytes a PNG of the float render holds, as (3,H,W) uint8."""
    return img.mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8)


def view_pair(seed, H, W):
    """A render-like float image that strays outside [0, 1] (so train.py's clamp matters) and a uint8 ground truth
    near it."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing="ij")
    img = torch.zeros(3, H, W)
    for _ in range(6):
        cx, cy, r = torch.rand(3, generator=g)
        col = torch.rand(3, generator=g)
        img += col[:, None, None] * torch.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / (0.02 + 0.1 * r) ** 2)
    gt = (img.clamp(0, 1) + 0.08 * torch.randn(3, H, W, generator=g)).clamp(0, 1)
    gt_u8 = (gt * 255).round().to(torch.uint8)
    render = img * 1.25 - 0.1 + 0.05 * torch.randn(3, H, W, generator=g)   # below 0 and above 1 in places
    return render.contiguous(), gt_u8.contiguous()


def record(x, y):
    """{l1, psnr, psnr_all, ssim} of x against y, both (3,H,W), with the reference's functions."""
    return [float(l1_loss(x, y)), float(psnr(x, y).mean()), float(psnr(x[None], y[None]).mean()),
            float(ssim(x, y))]


def main():
    # render.py's quantisation gives every code back from code / 255: a uint8 ground truth is exact for both forms
    codes = torch.arange(256, dtype=torch.uint8)
    assert torch.equal(quantise(codes.float() / 255), codes)

    out = {}
    pairs = {name: view_pair(seed, H, W) for name, (seed, H, W) in CASES.items()}
    r, g = pairs["a"]
    pairs["same"] = ((g.float() / 255).contiguous(), g)   # identical images: PSNR +inf, SSIM 1
    for name, (render, gt_u8) in pairs.items():
        q = quantise(render.clone())
        out[f"{name}_render"] = render.numpy()
        out[f"{name}_gt_u8"] = gt_u8.numpy()
        out[f"{name}_display_u8"] = q.permute(1, 2, 0).contiguous().numpy()
        for tag, dt in (("f32", torch.float32), ("f64", torch.float64)):
            y = gt_u8.to(dt) / 255
            # "same": the float32 render is gt/255 rounded to float32, which is y itself only in float32 -- in float64
            # the identical pair is y against y
            x = y if name == "same" else torch.clamp(render.to(dt), 0.0, 1.0)
            out[f"{name}_train_{tag}"] = np.array(record(x, y), dtype=np.float64)
            out[f"{name}_metrics_{tag}"] = np.array(record(q.to(dt) / 255, y), dtype=np.float64)
    assert np.isinf(out["same_train_f64"][1]) and np.isinf(out["same_train_f64"][2])
    path = os.path.join(HERE, "metrics_vectors.npz")
    np.savez_compressed(path, **out)
    print(path, len(out), "arrays", os.path.getsize(path), "bytes")
    for k in sorted(out):
        if k.endswith(("_f32", "_f64")):
            print(k, out[k])


if __name__ == "__main__":
    main()
