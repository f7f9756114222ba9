"""Generates tests/golden/resize_vectors.npz by running the REAL reference loader (CameraDataset.__getitem__,
scene/__init__.py:38-62, and loadCam, utils/camera_utils.py:20-40, under /root/reference, read-only) on the CPU.  The
fixture travels to the GPU box; /root/reference does not.

    python tests/golden/make_golden_resize.py

Frames: two 41x31 RGBA frames -- one structured (gradients, a hard-edged checker that rings under the cubic, an alpha
disc with a ramp), one seeded noise with fully clear and fully opaque pixels -- each composited on a black and a white
background and resized by PILtoTorch to every target of TARGETS: down, up, one axis alone, mixed, and 1x1.  Keys
"gt_<frame>_<bg>_<W>x<H>" hold the (3, H, W) uint8 bytes of `original_image` (bytes / 255 in float32, recovered
exactly).  The loader ends its composite in `Image.fromarray(np.array(arr * 255.0, dtype=np.byte), "RGB")`, which
PIL 12 refuses; the shim of make_golden_rgba.py restores PIL < 12's reading of it for that one call.

"loader_sizes": rows (width, height, resolution, resolution_scale, image_width, image_height) of loadCam's camera
size for the capture sizes of SIZES at each (resolution, resolution_scale) of RESOLUTIONS.
"""
import os
import sys
from types import SimpleNamespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))

from tests import ref_import  # noqa: E402

ref_import.prepare()
from PIL import Image  # noqa: E402
from scene import CameraDataset  # noqa: E402  (REAL reference code)
from utils.camera_utils import loadCam  # noqa: E402  (REAL reference code)

sys.path.insert(0, HERE)
from make_golden_rgba import _fromarray_pil11  # noqa: E402

_fromarray = Image.fromarray

W, H = 41, 31
TARGETS = ((20, 15), (83, 64), (41, 12), (17, 31), (7, 90), (1, 1))
SIZES = ((1920, 1080), (3208, 2200), (1601, 1200), (802, 550), (1600, 1200), (4000, 3000), (641, 480))
RESOLUTIONS = ((-1, 1.0), (-1, 2.0), (1, 1.0), (2, 1.0), (4, 1.0), (8, 1.0), (4, 2.0), (2.0, 1.0), (800, 1.0),
               (1000.5, 1.0), (1234, 0.5))


def frames() -> dict:
    y, x = np.mgrid[0:H, 0:W]
    a = np.empty((H, W, 4), np.uint8)
    a[..., 0] = np.clip(x * 6, 0, 255)
    a[..., 1] = np.clip(y * 8, 0, 255)
    a[..., 2] = np.where(((x // 3) + (y // 3)) % 2 == 0, 255, 0)
    r = np.hypot(x - W / 2, y - H / 2)
    a[..., 3] = np.clip((14 - r) * 60, 0, 255).astype(np.uint8)
    rng = np.random.default_rng(7)
    b = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
    b[..., 3] = rng.choice(np.array([0, 255, 1, 128, 254], np.uint8), (H, W))
    return {"structured": a, "noise": b}


def loader_bytes(rgba: np.ndarray, bg, width: int, height: int) -> np.ndarray:
    """(3, height, width) uint8 ground truth of the reference loader for this frame, background and camera size."""
    cam = SimpleNamespace(image=Image.fromarray(rgba, "RGBA"), image_path=None, bg=np.array(bg),
                          image_width=width, image_height=height)
    Image.fromarray = _fromarray_pil11
    try:
        out = CameraDataset([cam])[0]
    finally:
        Image.fromarray = _fromarray
    img = out.original_image.numpy()
    assert img.shape == (3, height, width)
    u8 = np.rint(img.astype(np.float64) * 255.0)
    assert np.abs(u8 / 255.0 - img).max() < 1e-6
    return u8.astype(np.uint8)


def loader_size(width: int, height: int, resolution, resolution_scale: float) -> tuple:
    args = SimpleNamespace(resolution=resolution, data_device="cpu")
    info = SimpleNamespace(width=width, height=height, uid=0, R=np.eye(3), T=np.zeros(3), FovX=0.5, FovY=0.5,
                           bg=np.zeros(3), image=None, image_path=None, image_name="x", timestep=0)
    cam = loadCam(args, 0, info, resolution_scale)
    return cam.image_width, cam.image_height


def main():
    out = {}
    for name, rgba in frames().items():
        out["rgba_" + name] = rgba
        for bg_name, bg in (("bg0", [0, 0, 0]), ("bg1", [1, 1, 1])):
            for w, h in TARGETS:
                out[f"gt_{name}_{bg_name}_{w}x{h}"] = loader_bytes(rgba, bg, w, h)
    rows = [(w, h, r, s) + loader_size(w, h, r, s) for w, h in SIZES for r, s in RESOLUTIONS]
    out["loader_sizes"] = np.array(rows, dtype=np.float64)
    path = os.path.join(HERE, "resize_vectors.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
