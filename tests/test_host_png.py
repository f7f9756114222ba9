"""CPU: the PNG encoder's surface (gab200_png_bound / gab200_png_scratch_bytes / gab200_png_encode / gab200_png_copy,
encode_png, GraphedRender / GraphedEval png=True) -- the exports, the header declarations, the C ABI's refusals before
any device work, every Python refusal -- and oracle/png.py: its filter choice against a brute-force evaluation of the
five filters, and its bound against hand-computed files."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from oracle import png as opng
from tests.test_host_frame_store import _model, no_device  # noqa: F401  (no_device: a fixture)

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
SIGNATURES = {
    "gab200_png_bound": ("int64_t", ["width", "height"]),
    "gab200_png_scratch_bytes": ("size_t", ["views", "height", "width"]),
    "gab200_png_encode": ("int32_t", ["views", "height", "width", "rgb", "scratch", "out", "out_stride", "out_len",
                                      "stream"]),
    "gab200_png_copy": ("int32_t", ["views", "src", "src_stride", "src_len", "flag", "dst", "dst_stride", "dst_len",
                                    "stream"]),
}


def test_exported_and_declared():
    import gaussianavatars_b200 as g
    from gaussianavatars_b200 import _native as N
    L = N.lib()
    hdr = open(os.path.join(ROOT, "include", "gab200_rasterizer.h")).read()
    for name, (ret, params) in SIGNATURES.items():
        assert name in N.EXPORTED_SYMBOLS and hasattr(L, name)
        decl = re.search(ret + r" " + name + r"\(([^)]*)\);", hdr)
        assert decl is not None, name
        assert [p.split()[-1].lstrip("*") for p in decl.group(1).split(",")] == params, name
        assert len(getattr(L, name).argtypes) == len(params)
    for name in ("encode_png", "png_bound"):
        assert name in g.__all__ and getattr(g, name).__module__ == "gaussianavatars_b200.png"


@pytest.mark.parametrize("W,H", [(1, 1), (700, 1), (1, 900), (550, 802), (802, 550), (1920, 1080), (11000, 5),
                                 (5461, 2), (10922, 1), (10923, 1)])
def test_bound_and_scratch_sizes(W, H):
    from gaussianavatars_b200 import _native as N
    from gaussianavatars_b200 import png_bound
    assert png_bound(W, H) == N.lib().gab200_png_bound(W, H) == opng.png_bound(W, H)
    assert N.lib().gab200_png_scratch_bytes(1, H, W) >= H * (3 * W + 1)
    assert N.lib().gab200_png_scratch_bytes(16, H, W) > N.lib().gab200_png_scratch_bytes(1, H, W)


def test_bound_by_hand():
    # 1x1: 4 filtered bytes in one stored block: 3 + 5 bits, LEN / NLEN, 4 bytes -> 9 deflate bytes; with the
    # signature 8, IHDR 25, IDAT 12 + 2 + 9 + 4, IEND 12 the file is 72 bytes, the bound one more (6 bytes per block)
    assert opng.png_bound(1, 1) == 8 + 25 + 12 + 2 + 4 + 12 + 4 + 6 == 73
    # 5461 x 2: 2 (3 * 5461 + 1) = 32768 bytes, exactly one block; 10923 x 1: 32770 bytes, two blocks
    assert opng.segments(5461, 2) == 1 and opng.png_bound(5461, 2) == 63 + 32768 + 6
    assert opng.segments(10923, 1) == 2 and opng.png_bound(10923, 1) == 63 + 32770 + 12
    # 1920 x 1080: 1080 (3 * 1920 + 1) = 6,221,880 bytes, 190 blocks
    assert opng.png_bound(1920, 1080) == 63 + 6_221_880 + 6 * 190
    with pytest.raises(ValueError):
        opng.png_bound(0, 4)


def test_c_abi_refusals_before_any_device_work():
    from gaussianavatars_b200 import _native as N
    L = N.lib()
    invalid = -1
    buf = (C.c_uint8 * 1024)()
    p = C.cast(buf, C.c_void_p)
    al = C.c_void_p((p.value + 255) & ~255)           # 256-byte aligned
    mis = C.c_void_p(al.value + 8)
    b = L.gab200_png_bound(4, 3)
    assert b == opng.png_bound(4, 3)
    for w, h in ((0, 3), (4, 0), (-1, 3), (4, -7), (2**31 - 1, 2**31 - 1), (100_000, 100_000)):
        assert L.gab200_png_bound(w, h) == invalid, (w, h)
        assert L.gab200_png_scratch_bytes(1, h, w) == 0
    assert L.gab200_png_scratch_bytes(0, 3, 4) == 0 and L.gab200_png_scratch_bytes(-2, 3, 4) == 0
    # encode: views, height, width, rgb, scratch, out, out_stride, out_len
    ok = [1, 3, 4, p, al, p, b, p]
    for i, bad in ((0, 0), (0, -1), (1, 0), (2, 0), (1, 100_000), (3, None), (4, None), (5, None), (6, b - 1),
                   (7, None), (4, mis)):
        args = list(ok)
        args[i] = bad
        assert L.gab200_png_encode(*args, None) == invalid, (i, bad)
    # copy: views, src, src_stride, src_len, flag, dst, dst_stride, dst_len
    ok = [1, al, 64, p, None, al, 64, p]
    for i, bad in ((0, 0), (1, None), (2, 0), (2, 24), (3, None), (5, None), (6, 48), (6, 72), (7, None), (1, mis),
                   (5, C.c_void_p(al.value + 4))):
        args = list(ok)
        args[i] = bad
        assert L.gab200_png_copy(*args, None) == invalid, (i, bad)


def test_encode_png_refusals():
    from gaussianavatars_b200 import encode_png
    with pytest.raises(TypeError, match="must be a torch.Tensor"):
        encode_png(np.zeros((2, 2, 3), np.uint8))
    with pytest.raises(ValueError, match="must be uint8"):
        encode_png(torch.zeros(2, 2, 3))
    for shape in ((2, 2), (2, 2, 4), (2, 2, 2, 2, 3), (2, 2, 1)):
        with pytest.raises(ValueError, match=r"must be \(H, W, 3\) or \(K, H, W, 3\)"):
            encode_png(torch.zeros(shape, dtype=torch.uint8))
    with pytest.raises(ValueError, match="must be contiguous"):
        encode_png(torch.zeros(3, 5, 3, dtype=torch.uint8).transpose(0, 1))
    with pytest.raises(ValueError, match="must be on a CUDA device"):
        encode_png(torch.zeros(3, 5, 3, dtype=torch.uint8))


def test_graphed_png_refusals(no_device):
    from gaussianavatars_b200.graph import GraphedEval, GraphedRender
    with pytest.raises(ValueError, match="png=True encodes the display image: it needs outputs 'u8' or 'both'"):
        GraphedRender(None, 8, 8, torch.zeros(3), outputs="float", png=True)
    with pytest.raises(ValueError, match="png=True encodes the display image: it needs source='u8'"):
        GraphedEval(None, 8, 8, torch.zeros(3), views=2, source="float", png=True)
    view = GraphedRender(_model(), 8, 8, torch.zeros(3), png=True)
    with pytest.raises(ValueError, match="host_png needs host_slots > 0"):
        view.host_png(0)
    plain = GraphedRender(_model(), 8, 8, torch.zeros(3), host_slots=2)
    with pytest.raises(ValueError, match="host_png needs a frame built with png=True"):
        plain.host_png(0)


# ---- the oracle's filter rule -----------------------------------------------------------------------------------------
def _brute(cur, prev):
    """All five filters byte by byte (the PNG specification's definitions), the least sum, ties to the lowest id."""
    n = len(cur)
    best = None
    for f in range(5):
        out, total = [], 0
        for i in range(n):
            x = int(cur[i])
            a = int(cur[i - 3]) if i >= 3 else 0
            b = int(prev[i]) if prev is not None else 0
            c = int(prev[i - 3]) if prev is not None and i >= 3 else 0
            if f == 0:
                pr = 0
            elif f == 1:
                pr = a
            elif f == 2:
                pr = b
            elif f == 3:
                pr = (a + b) // 2
            else:
                p = a + b - c
                pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                pr = a if pa <= pb and pa <= pc else (b if pb <= pc else c)
            v = (x - pr) % 256
            out.append(v)
            total += v if v < 128 else 256 - v
        if best is None or total < best[0]:
            best = (total, f, out)
    return best[1], np.array(best[2], np.uint8)


def _rows():
    rng = np.random.default_rng(7)
    cases = []
    for W in (1, 2, 3, 7, 40):
        n = 3 * W
        cases.append((rng.integers(0, 256, n, dtype=np.uint8), None))                          # first row, noise
        cases.append((rng.integers(0, 256, n, dtype=np.uint8), rng.integers(0, 256, n, dtype=np.uint8)))
        flat = np.full(n, 99, np.uint8)
        cases.append((flat, None))                        # None and Up tie with Sub / Avg / Paeth: lowest id
        cases.append((flat, flat.copy()))                 # all zero but None: Sub, Up, Paeth... ties
        ramp = (np.arange(n) * 5 % 256).astype(np.uint8)
        cases.append((ramp, ramp.copy()))                 # Up is exact
        cases.append((ramp, (ramp + 1).astype(np.uint8)))
        cases.append((np.zeros(n, np.uint8), None))       # every filter sums to 0: None
        cases.append((np.full(n, 128, np.uint8), np.full(n, 128, np.uint8)))   # 128 counts as 128 either way
        cases.append((rng.integers(120, 136, n, dtype=np.uint8), rng.integers(0, 256, n, dtype=np.uint8)))
    return cases


@pytest.mark.parametrize("i", range(len(_rows())))
def test_filter_choice_equals_brute_force(i):
    cur, prev = _rows()[i]
    f, row = opng.choose_filter(cur, prev)
    bf, brow = _brute(cur, prev)
    assert f == bf and np.array_equal(row, brow)


def test_filter_ties_go_to_the_lowest_id():
    flat = np.full(9, 50, np.uint8)
    # under an equal row: None 450, Sub 150, Average 75, Up 0 and Paeth 0 -> Up, the lower of the tied two
    assert [opng.row_cost(opng.filter_row(flat, flat, f)) for f in range(5)] == [450, 150, 0, 75, 0]
    assert opng.choose_filter(flat, flat)[0] == 2
    zero = np.zeros(9, np.uint8)
    assert opng.choose_filter(zero, zero)[0] == 0   # all five sum to 0


def test_filter_image_stream_layout():
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (5, 4, 3), dtype=np.uint8)
    ids, stream = opng.filter_image(img)
    assert stream.shape == (5 * 13,) and list(stream[::13]) == list(ids)
    for y in range(5):
        f, row = _brute(img[y].reshape(-1), img[y - 1].reshape(-1) if y else None)
        assert ids[y] == f and np.array_equal(stream[13 * y + 1:13 * y + 13], row)
