"""Generates tests/golden/lpips_vectors.npz by IMPORTING the real lpipsPyTorch (/root/reference/lpipsPyTorch,
read-only) and running its LPIPS module on the CPU in float64, with seeded weights and no network:

  - torchvision's alexnet() / vgg16() are built with weights=None (networks.py asks for the pretrained ones);
  - their `features` load the seeded state dict of tests/lpips_oracle.py seeded_weights(net, seed);
  - lpipsPyTorch's get_state_dict is patched to return the seeded lin weights instead of downloading them.

Each case is a batch of two (render, ground truth) pairs of one size.  The fixture stores the images and, per case,
the per-image scores (one call per pair) and the batch call's result (the SUM over the batch, as LPIPS.forward
returns it).  The weights are not stored: they are regenerated from the seed.  Inputs are what training_report
scores: the float render clamped to [0, 1] against the ground-truth bytes / 255.  The fixture travels to the GPU box;
/root/reference does not.

    python tests/golden/make_golden_lpips.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, "/root/reference")
import torchvision.models as tvm  # noqa: E402

import lpipsPyTorch.modules.lpips as ref_lpips  # noqa: E402  (REAL reference code)
import lpipsPyTorch.modules.networks as ref_networks  # noqa: E402
from tests import lpips_oracle as ol  # noqa: E402

SEED, CASES = ol.SEED, ol.CASES


class _Models:
    """torchvision.models as lpipsPyTorch's networks.py sees it: every constructor builds an untrained network."""
    alexnet = staticmethod(lambda *a, **k: tvm.alexnet(weights=None))
    vgg16 = staticmethod(lambda *a, **k: tvm.vgg16(weights=None))
    VGG16_Weights = tvm.VGG16_Weights


def view_pair(seed, H, W):
    """A smooth render-like float image that strays outside [0, 1] and a uint8 ground truth near it."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(1, 3, H // 6 + 2, W // 6 + 2, generator=g)
    img = torch.nn.functional.interpolate(low, size=(H, W), mode="bicubic", align_corners=False)[0] * 1.3 - 0.15
    gt = (img.clamp(0, 1) + 0.08 * torch.randn(3, H, W, generator=g)).clamp(0, 1)
    return img.contiguous(), (gt * 255).round().to(torch.uint8).contiguous()


def reference(net, feats, lin):
    ref_networks.models = _Models
    ref_lpips.get_state_dict = lambda net_type, version: dict(lin)
    m = ref_lpips.LPIPS(net, "0.1")
    m.net.layers.load_state_dict({k[len("features."):]: v for k, v in feats.items()}, strict=False)
    return m.double().eval()


def main():
    out = {}
    for name, (net, H, W, seed, dead, same) in CASES.items():
        feats, lin = ol.seeded_weights(net, SEED[net], dead_conv=dead)
        model = reference(net, feats, lin)
        renders, gts = zip(*(view_pair(100 * seed + i, H, W) for i in range(2)))
        x = torch.stack([torch.clamp(r.double(), 0, 1) for r in renders])
        y = torch.stack([g.double() / 255 for g in gts])
        if same:
            x = y.clone()
        with torch.no_grad():
            per = [float(model(x[i:i + 1], y[i:i + 1]).reshape(())) for i in range(2)]
            batch = model(x, y)
        assert tuple(batch.shape) == (1, 1, 1, 1)
        out[f"{name}_render"] = torch.stack(renders).numpy()
        out[f"{name}_gt_u8"] = torch.stack(gts).numpy()
        out[f"{name}_per_image"] = np.array(per, dtype=np.float64)
        out[f"{name}_batch_sum"] = np.array(float(batch.reshape(())), dtype=np.float64)
        print(name, net, H, W, per, float(batch.reshape(())))
        if same:
            assert per == [0.0, 0.0]
    path = os.path.join(HERE, "lpips_vectors.npz")
    np.savez_compressed(path, **out)
    print(path, len(out), "arrays", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
