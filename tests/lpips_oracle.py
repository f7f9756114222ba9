"""Torch restatement of lpipsPyTorch's LPIPS v0.1 (test infrastructure, never imported by the product), in any dtype on
any device, and the seeded weight recipe the LPIPS tests and tests/golden/make_golden_lpips.py share.

  x, y      the render clamped to [0, 1] (or the display bytes / 255) and the ground-truth bytes / 255
  z-score   (x - mean) / std with lpipsPyTorch's float32 buffers (modules/networks.py BaseNet), on the [0, 1] values
  features  torchvision alexnet() / vgg16() `features` up to the last target ReLU (F.conv2d + relu, max_pool2d)
  head      per target layer: f / (sqrt(sum_c f^2) + 1e-10) (modules/utils.py normalize_activation), the squared
            difference, the lin layer (a bias-free 1x1 conv), the spatial mean; the per-image score sums the layers

In float64 this is the oracle the GPU tests hold gab200_lpips to; tests/test_oracle_lpips.py checks it against the
fixture the real lpipsPyTorch produced.  In float32 on a GPU, F.conv2d runs torch's default (TF32 cuDNN) convolution:
the reference's own arithmetic on an H100."""
import numpy as np
import torch
import torch.nn.functional as F

from gaussianavatars_b200.lpips import NETS

MEAN = torch.tensor([-.030, -.088, -.188], dtype=torch.float32)
STD = torch.tensor([.458, .448, .450], dtype=torch.float32)

# the cases of tests/golden/lpips_vectors.npz (make_golden_lpips.py) and the weight seed of each network
SEED = {"alex": 11, "vgg": 12}
CASES = {   # name: (net, H, W, image seed, dead conv or None, identical pair)
    "alex_min": ("alex", 31, 31, 1, None, False),
    "vgg_min": ("vgg", 16, 16, 2, None, False),
    "alex_odd": ("alex", 97, 131, 3, None, False),
    "vgg_odd": ("vgg", 97, 131, 4, None, False),
    "alex_dead": ("alex", 64, 75, 5, 4, False),     # relu5 is zero at every pixel
    "vgg_dead": ("vgg", 40, 37, 6, 12, False),      # relu5_3 is zero at every pixel
    "alex_same": ("alex", 45, 50, 7, None, True),
    "vgg_same": ("vgg", 33, 20, 8, None, True),
}


def seeded_weights(net, seed=0, dead_conv=None):
    """(features, lin): a torchvision-style `features.N.*` state dict and an lpipsPyTorch-style `{i}.1.weight` lin
    dict, float32, from torch.Generator(seed).  Convolutions are He-scaled so activations keep their magnitude through
    13 layers; biases are small; lin weights are non-negative as the trained ones are.  dead_conv=l: the l-th
    convolution's biases are -1e4, so its ReLU output is exactly zero at every pixel (the 1e-10 path of the head)."""
    g = torch.Generator().manual_seed(seed)
    features, lin, t = {}, {}, 0
    for l, (mod, cin, cout, k, _, target) in enumerate(NETS[net]["convs"]):
        w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
        b = 0.05 * torch.randn(cout, generator=g)
        if l == dead_conv:
            b = torch.full((cout,), -1e4)
        features[f"features.{mod}.weight"], features[f"features.{mod}.bias"] = w.float(), b.float()
        if target:
            lin[f"{t}.1.weight"] = (torch.rand(1, cout, 1, 1, generator=g) * 0.2).float()
            t += 1
    return features, lin


def inputs(render, gt_u8):
    """(x, y) float64 (3,H,W) tensors: a float (3,H,W) render clamped to [0, 1] (NaN stays NaN), a uint8 (H,W,3)
    display image as value/255; the ground truth as value/255."""
    r = torch.as_tensor(np.asarray(render))
    x = r.permute(2, 0, 1).double() / 255 if r.dtype == torch.uint8 else torch.clamp(r.double(), 0.0, 1.0)
    return x, torch.as_tensor(np.asarray(gt_u8)).double() / 255


def conv_specs(net):
    """(module index, stride, pad, a pool follows, target) of every convolution."""
    spec = NETS[net]
    return [(mod, spec["stride1"] if mod == 0 else 1, spec["pad1"] if mod == 0 else (k - 1) // 2, pool, target)
            for mod, _, _, k, pool, target in spec["convs"]]


def z_score(x):
    """x: (B,3,H,W); the buffers in x's dtype, as lpipsPyTorch's float32 buffers are after `.to(dtype)`."""
    return (x - MEAN.to(x)[None, :, None, None]) / STD.to(x)[None, :, None, None]


def features(x, net, feats):
    """The target-layer ReLU outputs of z-scored x ((B,3,H,W)), as BaseNet.forward returns them before normalising."""
    k = NETS[net]["pool"]
    out = []
    h = z_score(x)
    for mod, s, p, pool, target in conv_specs(net):
        h = F.relu(F.conv2d(h, feats[f"features.{mod}.weight"].to(h), feats[f"features.{mod}.bias"].to(h),
                            stride=s, padding=p))
        if target:
            out.append(h)
        if pool:
            h = F.max_pool2d(h, k, 2)
    return out


def normalize(f, eps=1e-10):
    return f / (torch.sqrt(torch.sum(f ** 2, dim=1, keepdim=True)) + eps)


def head(fx, fy, lin):
    """(B,) per-image scores from the target features of both images (lists of (B,C,H,W))."""
    total = 0
    for t, (a, b) in enumerate(zip(fx, fy)):
        d = (normalize(a) - normalize(b)) ** 2
        total = total + F.conv2d(d, lin[f"{t}.1.weight"].to(d)).mean((2, 3))[:, 0]
    return total


def lpips(x, y, net, feats, lin):
    """(B,) per-image LPIPS of x against y ((B,3,H,W) in [0, 1]) in x's dtype and on x's device."""
    return head(features(x, net, feats), features(y, net, feats), lin)


def lpips64(render, gt_u8, net, feats, lin):
    """The float64 LPIPS of one view given as the kernel takes it (float (3,H,W) render or uint8 (H,W,3) display
    image; uint8 (3,H,W) ground truth), on the CPU."""
    x, y = inputs(render, gt_u8)
    return float(lpips(x[None], y[None], net, feats, lin)[0])
