"""LPIPS distance (v0.1) on the device: lpipsPyTorch's AlexNet and VGG-16 perceptual distance of one rendered view
against its uint8 ground truth (include/gab200_rasterizer.h, gab200_lpips), from weights the caller already has.

    net = LpipsNet.from_hub_cache("alex")          # the files lpipsPyTorch left in <torch hub>/checkpoints
    d = lpips(render, gt_u8, net)                  # 0-d float32 device tensor, no host wait

What is scored: the render and the ground truth as image_metrics reads them (the float render clamped to [0, 1], or
the display bytes as value/255), each z-scored with lpipsPyTorch's constants on those [0, 1] values (the reference never
rescales to [-1, 1]), torchvision's `features` up to the last target ReLU, and per target layer the mean over the
pixels of the lin-weighted squared difference of the channel-normalised features, summed over the five layers.  The
convolutions run on the tensor cores with TF32 operands (what torch's default cuDNN convolution does on an H100) and
FP32 accumulation in a fixed order; everything after them is FP32 per pixel and double across pixels.  The result is
bit-identical from call to call.  train.py's training_report uses "alex", metrics.py "vgg".
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

from . import _native as N
from .training import check_metrics_inputs

# torchvision `features` up to the last target ReLU: (module index, Cin, Cout, kernel, a pool follows, target layer).
# The targets are the ReLUs lpipsPyTorch's BaseNet returns (its target_layers count modules from 1).
_ALEX = ((0, 3, 64, 11, True, True), (3, 64, 192, 5, True, True), (6, 192, 384, 3, False, True),
         (8, 384, 256, 3, False, True), (10, 256, 256, 3, False, True))
_VGG = ((0, 3, 64, 3, False, False), (2, 64, 64, 3, True, True), (5, 64, 128, 3, False, False),
        (7, 128, 128, 3, True, True), (10, 128, 256, 3, False, False), (12, 256, 256, 3, False, False),
        (14, 256, 256, 3, True, True), (17, 256, 512, 3, False, False), (19, 512, 512, 3, False, False),
        (21, 512, 512, 3, True, True), (24, 512, 512, 3, False, False), (26, 512, 512, 3, False, False),
        (28, 512, 512, 3, False, True))
_LIN_URL = "https://raw.githubusercontent.com/richzhang/PerceptualSimilarity/master/lpips/weights/v0.1/{}.pth"
NETS = {
    "alex": dict(id=N.LPIPS_ALEX, convs=_ALEX, stride1=4, pad1=2, pool=3, min_side=31,
                 features_file="alexnet-owt-7be5be79.pth",
                 features_url="https://download.pytorch.org/models/alexnet-owt-7be5be79.pth"),
    "vgg": dict(id=N.LPIPS_VGG16, convs=_VGG, stride1=1, pad1=1, pool=2, min_side=16,
                features_file="vgg16-397923af.pth",
                features_url="https://download.pytorch.org/models/vgg16-397923af.pth"),
}


def _check_tensor(sd, key, shape, what):
    if key not in sd:
        raise KeyError(f"{what}: missing {key!r}")
    t = sd[key]
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32:
        raise TypeError(f"{what}: {key!r} must be a float32 tensor, got "
                        f"{t.dtype if isinstance(t, torch.Tensor) else type(t).__name__}")
    if tuple(t.shape) != shape:
        raise ValueError(f"{what}: {key!r} has shape {tuple(t.shape)}, expected {shape}")
    if not bool(torch.isfinite(t).all()):
        raise ValueError(f"{what}: {key!r} holds non-finite values")
    return t


class LpipsNet:
    """The packed weights of one LPIPS network on one device (gab200_lpips_pack), built once and shared by every call.

    net: "alex" or "vgg".  features: torchvision's state dict of alexnet() / vgg16() -- the `features.N.weight` /
    `features.N.bias` keys of every convolution up to the last target layer; keys outside `features.` (the
    classifier) are ignored, any other `features.` key is refused.  lin: the LPIPS v0.1 lin weights, keyed as the file
    stores them (`lin{i}.model.1.weight`) or as lpipsPyTorch renames them (`{i}.1.weight`), each (1, C_i, 1, 1).
    Every key, shape and dtype (float32) is checked, and every value must be finite."""

    def __init__(self, net: str, features: dict, lin: dict, device="cuda"):
        if net not in NETS:
            raise ValueError(f"net must be 'alex' or 'vgg', got {net!r}")
        spec = NETS[net]
        convs = spec["convs"]
        want = {}
        for mod, cin, cout, k, _, _ in convs:
            want[f"features.{mod}.weight"] = (cout, cin, k, k)
            want[f"features.{mod}.bias"] = (cout,)
        extra = sorted(k for k in features if k.startswith("features.") and k not in want)
        if extra:
            raise KeyError(f"features: unexpected keys {extra} (the {net} features up to its last target layer are "
                           f"{sorted(want)})")
        tensors = {k: _check_tensor(features, k, s, "features") for k, s in want.items()}
        chans = [cout for _, _, cout, _, _, target in convs if target]
        forms = ([f"lin{i}.model.1.weight" for i in range(5)], [f"{i}.1.weight" for i in range(5)])
        keys = set(lin)
        form = next((f for f in forms if keys == set(f)), None)
        if form is None:
            raise KeyError(f"lin: keys {sorted(keys)} are neither {forms[0]} nor {forms[1]}")
        lins = [_check_tensor(lin, k, (1, c, 1, 1), "lin") for k, c in zip(form, chans)]
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("gaussianavatars_b200 has no CPU path: LpipsNet needs a CUDA device")
        self.net, self.id = net, spec["id"]
        self.min_side = spec["min_side"]
        L = N.lib()
        nbytes = int(L.gab200_lpips_weights_bytes(self.id))
        self.weights = torch.empty(nbytes, dtype=torch.uint8, device=device)
        # "cuda" names the current device without an index; tensors report theirs (cuda:0), and the device checks
        # of lpips() and GraphedEval compare against this one
        self.device = device = self.weights.device
        w = [tensors[f"features.{c[0]}.weight"].to(device).contiguous() for c in convs]
        b = [tensors[f"features.{c[0]}.bias"].to(device).contiguous() for c in convs]
        li = [t.to(device).reshape(-1).contiguous() for t in lins]
        arr = lambda ts: (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])  # noqa: E731
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            N.check(L.gab200_lpips_pack(self.id, arr(w), arr(b), arr(li), self.weights.data_ptr(),
                                        C.c_void_p(stream)), "gab200_lpips_pack")

    @classmethod
    def from_hub_cache(cls, net: str, hub_dir: Optional[str] = None, device="cuda") -> "LpipsNet":
        """The weights lpipsPyTorch leaves in `<hub_dir>/checkpoints` (hub_dir: torch.hub.get_dir() by default):
        torchvision's `alexnet-owt-7be5be79.pth` / `vgg16-397923af.pth` and the lin file `alex.pth` / `vgg.pth`.
        Never downloads: a missing file raises FileNotFoundError naming its path and where lpipsPyTorch fetches it."""
        if net not in NETS:
            raise ValueError(f"net must be 'alex' or 'vgg', got {net!r}")
        spec = NETS[net]
        ck = os.path.join(hub_dir if hub_dir is not None else torch.hub.get_dir(), "checkpoints")
        files = ((os.path.join(ck, spec["features_file"]), spec["features_url"]),
                 (os.path.join(ck, f"{net}.pth"), _LIN_URL.format(net)))
        for path, url in files:
            if not os.path.isfile(path):
                raise FileNotFoundError(f"{path} is missing: lpipsPyTorch downloads it from {url} (this library "
                                        "downloads nothing)")
        features, lin = (torch.load(p, map_location="cpu", weights_only=True) for p, _ in files)
        return cls(net, features, lin, device)


def _size(render):
    """(H, W) of a render in either accepted layout, or None when the layout is not one of them."""
    if render.dim() == 3 and render.dtype == torch.float32 and render.shape[0] == 3:
        return int(render.shape[1]), int(render.shape[2])
    if render.dim() == 3 and render.dtype == torch.uint8 and render.shape[2] == 3:
        return int(render.shape[0]), int(render.shape[1])
    return None


def check_lpips_inputs(render: torch.Tensor, gt_u8: torch.Tensor, net: LpipsNet) -> int:
    """The checks of image_metrics, plus the network's smallest image; returns the render kind."""
    if not isinstance(net, LpipsNet):
        raise TypeError(f"net must be an LpipsNet, got {type(net).__name__}")
    hw = _size(render)
    if hw is not None and min(hw) < net.min_side:
        raise ValueError(f"LPIPS with {net.net} needs an image of at least {net.min_side}x{net.min_side} pixels, got "
                         f"{hw[1]}x{hw[0]}")
    kind = check_metrics_inputs(render, gt_u8)
    if render.device != net.device:
        raise ValueError(f"the images are on {render.device}, the LpipsNet on {net.device}")
    return kind


def lpips_scratch(net: LpipsNet, height: int, width: int) -> torch.Tensor:
    """Device scratch for one gab200_lpips call of this size: the per-CTA partial sums and two activation buffers."""
    nbytes = int(N.lib().gab200_lpips_scratch_bytes(net.id, int(height), int(width)))
    if nbytes == 0:
        raise ValueError(f"LPIPS with {net.net} needs an image of at least {net.min_side}x{net.min_side} pixels, got "
                         f"{width}x{height}")
    return torch.empty(nbytes, dtype=torch.uint8, device=net.device)


def _launch(render, gt_u8, net, table, row, skip_flag, scratch, features=None):
    kind = check_lpips_inputs(render, gt_u8, net)
    device = render.device
    if table.dtype != torch.float32 or table.dim() != 1 or table.device != device or not table.is_contiguous() or \
            table.shape[0] < 1:
        raise ValueError(f"table must be a contiguous float32 (rows,) tensor on {device}")
    for t, n in ((row, "row"), (skip_flag, "skip_flag")):
        if t is not None and (t.dtype != torch.int32 or t.device != device):
            raise TypeError(f"{n} must be an int32 tensor on {device}")
    r = render if render.is_contiguous() else render.contiguous()
    g = gt_u8 if gt_u8.is_contiguous() else gt_u8.contiguous()
    H, W = _size(r)
    need = int(N.lib().gab200_lpips_scratch_bytes(net.id, H, W))
    if scratch is None:
        scratch = lpips_scratch(net, H, W)
    elif scratch.numel() * scratch.element_size() < need or scratch.data_ptr() % 16:
        raise ValueError("LPIPS scratch too small for this image size, or not 16-byte aligned")
    a = N.LpipsArgs()
    a.abi_version, a.net, a.height, a.width, a.render_kind = N.ABI_VERSION, net.id, H, W, kind
    a.render, a.gt, a.weights, a.row = r.data_ptr(), g.data_ptr(), net.weights.data_ptr(), N.ptr(row)
    a.table, a.table_rows, a.skip_flag = table.data_ptr(), int(table.shape[0]), N.ptr(skip_flag)
    a.scratch, a.features = scratch.data_ptr(), N.ptr(features)
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device).cuda_stream
        N.check(N.lib().gab200_lpips(C.byref(a), C.c_void_p(stream)), "gab200_lpips")
    return table


def launch_lpips(render: torch.Tensor, gt_u8: torch.Tensor, net: LpipsNet, table: torch.Tensor,
                 row: Optional[torch.Tensor] = None, skip_flag: Optional[torch.Tensor] = None,
                 scratch: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Enqueues the LPIPS distance of `render` against `gt_u8` into `table[*row]` (row: a device int32, None = row 0;
    table: a (rows,) float32 device tensor) on the current stream; nothing is written when `skip_flag` (device int32)
    holds a non-zero value as the kernel runs.  Capturable: it reads nothing on the host."""
    return _launch(render, gt_u8, net, table, row, skip_flag, scratch)


@torch.no_grad()
def lpips(render: torch.Tensor, gt_u8: torch.Tensor, net: LpipsNet) -> torch.Tensor:
    """0-d float32 device tensor: the LPIPS distance of one view, with no autograd and no host wait.

    render: the float32 (3, H, W) image of render(), clamped to [0, 1] in the kernel as training_report clamps it, or
    the uint8 (H, W, 3) display image of render_display(), read as value/255 as metrics.py reads render.py's PNG.
    gt_u8: the uint8 (3, H, W) ground truth.  At least 31x31 pixels for "alex", 16x16 for "vgg".
    The value is what lpipsPyTorch's LPIPS returns for one image pair; its batch call returns the sum over the batch,
    which training_report divides by the number of views."""
    table = torch.empty(1, dtype=torch.float32, device=render.device)
    return launch_lpips(render, gt_u8, net, table)[0]


def _stages(net: str, H: int, W: int):
    """(key, C, H, W) of every stage output, in the kernel's order: "input", then the torchvision `features` index of
    each convolution's ReLU and of each pool."""
    spec = NETS[net]
    out = [("input", 4, H, W)]
    for mod, _, cout, k, pool, _ in spec["convs"]:
        s, p = (spec["stride1"], spec["pad1"]) if mod == 0 else (1, (k - 1) // 2)
        H, W = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
        out.append((mod + 1, cout, H, W))
        if pool:
            H, W = (H - spec["pool"]) // 2 + 1, (W - spec["pool"]) // 2 + 1
            out.append((mod + 2, cout, H, W))
    return out


@torch.no_grad()
def lpips_features(render: torch.Tensor, gt_u8: torch.Tensor, net: LpipsNet) -> dict:
    """Every stage of one eager gab200_lpips call, as (2, C, H, W) float32 device tensors (image 0 the render, image 1
    the ground truth), keyed "input" (the z-scored images) and by the torchvision `features` index of each
    convolution's ReLU and each pool.  The kernels are those of lpips(); only where they write differs."""
    hw = _size(render)
    check_lpips_inputs(render, gt_u8, net)
    stages = _stages(net.net, *hw)
    nbytes = int(N.lib().gab200_lpips_features_bytes(net.id, *hw))
    if nbytes != 4 * sum(2 * c * h * w for _, c, h, w in stages):
        raise RuntimeError(f"the library's LPIPS stages ({nbytes} bytes) are not those of lpips.NETS")
    buf = torch.empty(nbytes // 4, dtype=torch.float32, device=render.device)
    table = torch.empty(1, dtype=torch.float32, device=render.device)
    _launch(render, gt_u8, net, table, None, None, None, features=buf)
    out, off = {}, 0
    for key, c, h, w in stages:
        n = 2 * c * h * w
        t = buf[off:off + n].view(2, h, w, c).permute(0, 3, 1, 2)
        out[key] = t[:, :3] if key == "input" else t
        off += n
    return out

