"""Generates tests/golden/rgba_composite_vectors.npz by running the REAL reference loader
(CameraDataset.__getitem__, scene/__init__.py:38-62 under /root/reference, read-only) on a 256x256 RGBA frame holding
every (colour byte, alpha byte) pair in each colour channel, once on a black and once on a white background.  The
fixture travels to the GPU box; /root/reference does not.

    python tests/golden/make_golden_rgba.py

The loader ends in `Image.fromarray(np.array(arr * 255.0, dtype=np.byte), "RGB")`.  PIL 12 refuses an int8 array in
mode "RGB"; PIL < 12 took the array's buffer as the raw bytes of an RGB image.  The shim below restores exactly that
(Image.frombuffer over the int8 array's bytes) for that one call and leaves every other call to PIL.  numpy's float64
-> int8 cast wraps on x86-64, so the bytes read back as uint8 are trunc(arr * 255).

The frame's size equals the camera's, so PILtoTorch's resize is the identity (the GaussianAvatars / NeRSemble case:
802x550 frames, under the 1600-pixel rescale of utils/camera_utils.py:26-35).  `original_image` is then bytes / 255
in float32, from which round(x * 255) recovers the bytes exactly.
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

_fromarray = Image.fromarray


def _fromarray_pil11(obj, mode=None):
    """PIL < 12: an int8 array given with mode "RGB" is the raw bytes of an RGB image."""
    a = np.asarray(obj)
    if mode == "RGB" and a.dtype == np.int8 and a.ndim == 3 and a.shape[2] == 3:
        a = np.ascontiguousarray(a)
        return Image.frombuffer("RGB", (a.shape[1], a.shape[0]), a.tobytes(), "raw", "RGB", 0, 1)
    return _fromarray(obj, mode) if mode is not None else _fromarray(obj)


def every_pair_frame() -> np.ndarray:
    """(256, 256, 4) uint8: row a, column c holds alpha a and colours c, c + 85, c + 170 (mod 256), so each colour
    channel meets every (c, a) pair once."""
    c = np.arange(256, dtype=np.int64)
    a = np.arange(256, dtype=np.int64)
    rgba = np.empty((256, 256, 4), dtype=np.uint8)
    rgba[:, :, 0] = c[None, :]
    rgba[:, :, 1] = (c[None, :] + 85) % 256
    rgba[:, :, 2] = (c[None, :] + 170) % 256
    rgba[:, :, 3] = a[:, None]
    return rgba


def loader_bytes(rgba: np.ndarray, bg) -> np.ndarray:
    """(3, H, W) uint8 ground truth of the reference loader for this frame and background."""
    H, W = rgba.shape[:2]
    cam = SimpleNamespace(image=Image.fromarray(rgba, "RGBA"), image_path=None, bg=np.array(bg),
                          image_width=W, image_height=H)
    Image.fromarray = _fromarray_pil11
    try:
        out = CameraDataset([cam])[0]
    finally:
        Image.fromarray = _fromarray
    img = out.original_image.numpy()
    assert img.shape == (3, H, W)
    u8 = np.rint(img.astype(np.float64) * 255.0)
    assert np.abs(u8 / 255.0 - img).max() < 1e-6   # bytes / 255 in float32: the bytes come back exactly
    return u8.astype(np.uint8)


def main():
    rgba = every_pair_frame()
    out = {"rgba": rgba}
    for name, bg in (("bg0", [0, 0, 0]), ("bg1", [1, 1, 1])):   # dataset_readers' black / white backgrounds
        out[name] = loader_bytes(rgba, bg)
    path = os.path.join(HERE, "rgba_composite_vectors.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
