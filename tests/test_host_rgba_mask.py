"""CPU: the RGBA ground truth (gab200_composite_rgba, training.composite_rgba, GraphedFrame(rgba=True, lambda_mask=...)).

The fixture tests/golden/rgba_composite_vectors.npz holds the reference loader's own bytes for every (colour, alpha)
pair on black and white (tests/golden/make_golden_rgba.py).  Here: the float64-then-truncate restatement the kernel
implements equals them, and the nearby restatements (float32, rounding) do not -- so the GPU test against the fixture
can tell them apart.  Plus the export, the header declaration and every argument refusal that needs no device."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "rgba_composite_vectors.npz"))


def composite64(rgba: np.ndarray, bg) -> np.ndarray:
    """The loader's arithmetic in numpy's operation order, float64, then truncation: (..., H, W, 4) -> (..., 3, H, W)."""
    norm = rgba / 255.0
    arr = norm[..., :3] * norm[..., 3:4] + np.asarray(bg, dtype=np.float64) * (1 - norm[..., 3:4])
    return np.moveaxis(np.trunc(arr * 255.0).astype(np.uint8), -1, -3)


def test_fixture_covers_every_pair():
    rgba = GOLD["rgba"]
    assert rgba.shape == (256, 256, 4) and rgba.dtype == np.uint8
    for ch in range(3):
        pairs = set(zip(rgba[..., ch].ravel().tolist(), rgba[..., 3].ravel().tolist()))
        assert len(pairs) == 65536


@pytest.mark.parametrize("name,bg", [("bg0", 0.0), ("bg1", 1.0)])
def test_float64_truncation_restatement_equals_the_loader_bytes(name, bg):
    assert np.array_equal(composite64(GOLD["rgba"], [bg] * 3), GOLD[name])


@pytest.mark.parametrize("name,bg,wrong_f32", [("bg0", 0.0, 154), ("bg1", 1.0, 391)])
def test_float32_and_rounding_restatements_differ_from_the_loader(name, bg, wrong_f32):
    rgba, want = GOLD["rgba"], GOLD[name]
    norm = rgba.astype(np.float32) / np.float32(255.0)
    arr = norm[..., :3] * norm[..., 3:4] + np.float32(bg) * (np.float32(1) - norm[..., 3:4])
    f32 = np.moveaxis(np.trunc(arr * np.float32(255.0)).astype(np.uint8), -1, -3)
    # one plane per channel, each holding every pair once: count the pairs of one channel
    assert int((f32[0] != want[0]).sum()) == wrong_f32
    norm64 = rgba / 255.0
    arr64 = norm64[..., :3] * norm64[..., 3:4] + bg * (1 - norm64[..., 3:4])
    rounded = np.moveaxis(np.rint(arr64 * 255.0).astype(np.uint8), -1, -3)
    assert int((rounded != want).sum()) > 0.3 * want.size


def test_exported_and_declared():
    from gaussianavatars_b200 import _native as N
    L = N.lib()
    assert "gab200_composite_rgba" in N.EXPORTED_SYMBOLS and hasattr(L, "gab200_composite_rgba")
    hdr = open(os.path.join(ROOT, "include", "gab200_rasterizer.h")).read()
    decl = re.search(r"int32_t gab200_composite_rgba\(([^)]*)\);", hdr)
    assert decl is not None
    params = [p.split()[-1].lstrip("*") for p in decl.group(1).split(",")]
    assert params == ["views", "height", "width", "rgba", "bg", "rgb_out", "mask_out", "stream"]
    assert len(L.gab200_composite_rgba.argtypes) == 8


def test_c_abi_refusals_before_any_device_work():
    from gaussianavatars_b200 import _native as N
    L = N.lib()
    buf = (C.c_uint8 * 64)()
    f = (C.c_float * 3)()
    p, q = C.cast(buf, C.c_void_p), C.cast(f, C.c_void_p)
    invalid = -1
    assert L.gab200_composite_rgba(-1, 2, 2, p, q, p, None, None) == invalid
    assert L.gab200_composite_rgba(1, -2, 2, p, q, p, None, None) == invalid
    assert L.gab200_composite_rgba(1, 2, -2, p, q, p, None, None) == invalid
    assert L.gab200_composite_rgba(1, 2, 2, None, q, p, None, None) == invalid   # no frame
    assert L.gab200_composite_rgba(1, 2, 2, p, None, p, None, None) == invalid   # no background
    assert L.gab200_composite_rgba(1, 2, 2, p, q, None, p, None) == invalid      # no output (the mask alone is not one)


def test_composite_rgba_refusals():
    import gaussianavatars_b200 as g
    with pytest.raises(RuntimeError, match="no CPU path"):
        g.composite_rgba(torch.zeros(4, 4, 4, dtype=torch.uint8), torch.zeros(3))
    for bad in (torch.zeros(4, 4, 4, dtype=torch.float32), torch.zeros(4, 4, 3, dtype=torch.uint8),
                torch.zeros(4, 4, dtype=torch.uint8), torch.zeros(1, 2, 4, 4, 4, dtype=torch.uint8),
                np.zeros((4, 4, 4), np.uint8)):
        with pytest.raises(TypeError, match="uint8 \\(H, W, 4\\) or \\(K, H, W, 4\\)"):
            g.composite_rgba(bad, torch.zeros(3))


def test_graphed_frame_refusals():
    from gaussianavatars_b200.graph import GraphedFrame
    bg = torch.zeros(3)
    with pytest.raises(ValueError, match="loss='dL_dimage' reads none"):
        GraphedFrame(None, 8, 8, 1.0, 1.0, bg, loss="dL_dimage", rgba=True)
    for lam in (-0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="lambda_mask must be a finite value >= 0"):
            GraphedFrame(None, 8, 8, 1.0, 1.0, bg, rgba=True, lambda_mask=lam)
    with pytest.raises(ValueError, match="needs rgba=True"):
        GraphedFrame(None, 8, 8, 1.0, 1.0, bg, lambda_mask=0.1)
    with pytest.raises(ValueError, match="loss='dL_dimage' reads none"):
        GraphedFrame(None, 8, 8, 1.0, 1.0, bg, loss="dL_dimage", rgba=True, lambda_mask=0.1)
