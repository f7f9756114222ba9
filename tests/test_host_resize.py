"""CPU: the loader's resize without a GPU -- oracle/resize.py against PIL's `Image.resize` over a grid of sizes, the
oracle and loader_size against the reference loader's own output (tests/golden/resize_vectors.npz), the exports and
header declarations of gab200_resize_scratch_bytes / gab200_resize_u8, and the refusals of the C ABI and of the
Python surface."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import resize as ors

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "resize_vectors.npz"))

# (in W, in H, out W, out H): 1-pixel inputs and outputs, ratios down to 1/50, upscales, odd sizes, each axis alone
GRID = [(1, 1, 1, 5), (1, 1, 7, 3), (5, 1, 1, 1), (1, 9, 1, 4), (9, 7, 1, 1), (64, 48, 32, 24), (101, 77, 50, 38),
        (80, 60, 37, 91), (33, 21, 100, 64), (401, 275, 200, 137), (200, 150, 200, 75), (200, 150, 75, 150),
        (500, 40, 10, 40), (40, 500, 40, 10), (500, 500, 10, 10), (250, 3, 5, 3), (3, 7, 150, 350), (2, 2, 3, 3),
        (13, 11, 12, 10), (17, 19, 18, 20), (255, 129, 127, 255), (7, 300, 7, 299)]
LARGE = [(3208, 2200, 1600, 1097), (1920, 1080, 1600, 900)]


def image(W, H, channels, seed):
    """Noise, a hard-edged checker (the cubic's lobes overshoot: the clamps at 0 and 255), or flat extremes."""
    rng = np.random.default_rng(seed)
    shape = (H, W, channels) if channels > 1 else (H, W)
    kind = seed % 3
    if kind == 0:
        return rng.integers(0, 256, shape, dtype=np.uint8)
    if kind == 1:
        y, x = np.mgrid[0:H, 0:W]
        c = np.where((x // 2 + y // 3) % 2 == 0, 255, 0).astype(np.uint8)
        return np.ascontiguousarray(np.broadcast_to(c[..., None], (H, W, channels))).reshape(shape)
    return rng.choice(np.array([0, 255], np.uint8), shape)


def pil_resize(a, w, h):
    return np.asarray(Image.fromarray(a, "RGB" if a.ndim == 3 else "L").resize((w, h)))


def oracle_hwc(a, w, h):
    if a.ndim == 2:
        return ors.resize_u8(a, w, h)
    return ors.resize_u8(np.ascontiguousarray(a.transpose(2, 0, 1)), w, h).transpose(1, 2, 0)


@pytest.mark.parametrize("case", GRID, ids=lambda c: "%dx%d-%dx%d" % c)
def test_oracle_equals_pil(case):
    W, H, w, h = case
    for seed, channels in enumerate((1, 3, 1, 3, 1, 3)):
        a = image(W, H, channels, seed)
        assert np.array_equal(oracle_hwc(a, w, h), pil_resize(a, w, h)), (case, seed, channels)


@pytest.mark.parametrize("case", LARGE, ids=lambda c: "%dx%d-%dx%d" % c)
def test_oracle_equals_pil_loader_sizes(case):
    W, H, w, h = case
    a = image(W, H, 1, 0)
    assert np.array_equal(ors.resize_u8(a, w, h), pil_resize(a, w, h))


def test_oracle_plan():
    """Weights sum to 2^22 within rounding; the taps stay inside the input and the table's rows."""
    for n_in, n_out in ((3208, 1600), (2200, 1097), (33, 100), (500, 10), (1, 7), (9, 1)):
        bounds, coeffs = ors.plan(n_in, n_out)
        assert coeffs.shape == (n_out, ors.ksize(n_in, n_out))
        assert (bounds[:, 0] >= 0).all() and (bounds.sum(1) <= n_in).all() and (bounds[:, 1] <= coeffs.shape[1]).all()
        assert (np.abs(coeffs.sum(1) - (1 << 22)) <= coeffs.shape[1]).all()


def composite(rgba, bg):
    """The reference loader's composite in float64 (tests/golden/make_golden_rgba.py pins the device's to it)."""
    n = rgba / 255.0
    arr = n[:, :, :3] * n[:, :, 3:4] + np.asarray(bg, np.float64) * (1 - n[:, :, 3:4])
    return np.array(arr * 255.0).astype(np.int8).view(np.uint8).transpose(2, 0, 1)


def golden_cases():
    for key in GOLDEN.files:
        m = re.fullmatch(r"gt_(\w+)_bg(\d)_(\d+)x(\d+)", key)
        if m:
            yield key, m.group(1), float(m.group(2)), int(m.group(3)), int(m.group(4))


def test_oracle_equals_reference_loader():
    cases = list(golden_cases())
    assert len(cases) == 24
    for key, frame, bg, w, h in cases:
        gt = composite(GOLDEN["rgba_" + frame], [bg] * 3)
        assert np.array_equal(ors.resize_u8(gt, w, h), GOLDEN[key]), key


def test_loader_size_equals_reference_loadcam():
    from gaussianavatars_b200.resize import loader_size
    rows = GOLDEN["loader_sizes"]
    assert len(rows) >= 70
    for W, H, res, scale, w, h in rows:
        assert loader_size(int(W), int(H), float(res), float(scale)) == (int(w), int(h)), (W, H, res, scale)
    assert loader_size(1920, 1080) == (1600, 900)
    assert loader_size(3208, 2200) == (1600, 1097)
    assert loader_size(1601, 1200) == (1599, 1199)
    assert loader_size(802, 550) == (802, 550)
    assert loader_size(3208, 2200, 4) == (802, 550)


def test_loader_size_refusals():
    from gaussianavatars_b200.resize import loader_size
    for bad in ((0, 10), (10, -1)):
        with pytest.raises(ValueError, match="positive size"):
            loader_size(*bad)
    with pytest.raises(TypeError, match="resolution"):
        loader_size(100, 100, "2")
    with pytest.raises(TypeError, match="resolution"):
        loader_size(100, 100, True)
    for bad in (0, -2, -1.5):
        with pytest.raises(ValueError, match="resolution must be"):
            loader_size(100, 100, bad)
    with pytest.raises(ValueError, match="no pixel left"):
        loader_size(100, 1, 8)


# ---- the C ABI and the Python surface ------------------------------------------------------------------------------
SIGNATURES = {
    "gab200_resize_scratch_bytes": ("size_t", ["planes", "in_height", "in_width", "out_height", "out_width"]),
    "gab200_resize_u8": ("int32_t", ["planes", "in_height", "in_width", "out_height", "out_width", "src", "dst",
                                     "scratch", "stream"]),
}


def test_exported_and_declared():
    import gaussianavatars_b200 as g
    from gaussianavatars_b200 import _native as N
    L = N.lib()
    hdr = open(os.path.join(ROOT, "include", "gab200_rasterizer.h")).read()
    for name, (ret, params) in SIGNATURES.items():
        assert name in N.EXPORTED_SYMBOLS and hasattr(L, name)
        decl = re.search(ret + r" ?" + name + r"\(([^)]*)\);", hdr)
        assert decl is not None, name
        assert [p.split()[-1].lstrip("*") for p in decl.group(1).split(",")] == params, name
        assert len(getattr(L, name).argtypes) == len(params)
    for name in ("resize_u8", "loader_size"):
        assert name in g.__all__ and getattr(g, name).__module__ == "gaussianavatars_b200.resize"


def test_scratch_bytes():
    from gaussianavatars_b200 import _native as N
    L = N.lib()
    f = L.gab200_resize_scratch_bytes
    for bad in ((0, 4, 4, 2, 2), (1, 0, 4, 2, 2), (1, 4, 0, 2, 2), (1, 4, 4, 0, 2), (1, 4, 4, 2, -1),
                (2**31, 2, 2, 1, 1), (2**30, 4, 4, 1, 1), (2**30, 1, 1, 4, 4)):
        assert f(*bad) == 0, bad
    assert f(1, 4, 4, 4, 4) == 256                                  # a copy: no tables
    k_w, k_h = ors.ksize(3208, 1600), ors.ksize(2200, 1097)
    up = lambda n: (n + 255) // 256 * 256                           # noqa: E731
    want = up(8 * 1600) + up(4 * 1600 * k_w) + up(8 * 1097) + up(4 * 1097 * k_h) + up(4 * 2200 * 1600)
    assert f(4, 2200, 3208, 1097, 1600) == want
    assert f(4, 2200, 3208, 2200, 1600) == up(8 * 1600) + up(4 * 1600 * k_w)   # width only: no intermediate


def test_c_abi_refusals():
    from gaussianavatars_b200 import _native as N
    L = N.lib()
    buf = (C.c_uint8 * 4096)()
    base = C.addressof(buf)
    scratch = (base + 255) // 256 * 256
    p = C.c_void_p(scratch)
    for args in ((0, 4, 4, 2, 2, p, p, p), (1, 4, 4, 0, 2, p, p, p), (2**31, 2, 2, 1, 1, p, p, p),
                 (1, 4, 4, 2, 2, None, p, p), (1, 4, 4, 2, 2, p, None, p), (1, 4, 4, 2, 2, p, p, None),
                 (1, 4, 4, 2, 2, p, p, C.c_void_p(scratch + 16))):
        assert L.gab200_resize_u8(*args, None) == -1, args


def test_python_refusals():
    from gaussianavatars_b200 import composite_rgba, resize_u8
    from gaussianavatars_b200.resize import check_size
    cpu = torch.zeros(2, 4, 4, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="no CPU path"):
        resize_u8(cpu, 2, 2)
    with pytest.raises(TypeError, match="uint8"):
        resize_u8(cpu.float(), 2, 2)
    with pytest.raises(TypeError, match="uint8"):
        resize_u8(torch.zeros(4, dtype=torch.uint8), 2, 2)
    for bad in ((0, 2), (2, -1), (2.0, 2), (True, 2)):
        with pytest.raises(ValueError, match="two positive ints"):
            check_size(bad)
    for bad in (5, (1, 2, 3), None):
        with pytest.raises(TypeError, match="width, height"):
            check_size(bad)
    assert check_size((np.int64(3), 4)) == (3, 4)
    with pytest.raises(ValueError, match="two positive ints"):
        composite_rgba(torch.zeros(4, 4, 4, dtype=torch.uint8), [0, 0, 0], size=(0, 4))
    with pytest.raises(RuntimeError, match="no CPU path"):
        composite_rgba(torch.zeros(4, 4, 4, dtype=torch.uint8), [0, 0, 0], size=(2, 2))
