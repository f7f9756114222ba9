"""CPU: the PNG decoder's surface (gab200_png_status_string / gab200_png_decode_scratch_bytes / gab200_png_decode,
decode_png, FrameStore.add_png) -- the exports, the header declarations and status codes, the C ABI's refusals before
any device work, and every host-side refusal of decode_png, each naming the file and the field."""
import ctypes as C
import io
import os
import re
import struct
import zlib

import numpy as np
import pytest

from oracle import inflate as oi
from tests import png_corpus as pc
from tests.test_host_frame_store import no_device  # noqa: F401  (a fixture)

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
SIGNATURES = {
    "gab200_png_status_string": ("const char\\*", ["status"]),
    "gab200_png_decode_scratch_bytes": ("size_t", ["files", "height", "width"]),
    "gab200_png_decode": ("int32_t", ["files", "height", "width", "zdata", "zoff", "zlen", "color_type", "scratch",
                                      "out", "out_channels", "status", "stream"]),
}
STATUS_NAMES = ["OK", "ZLIB_HEADER", "BLOCK_TYPE", "STORED_LENGTH", "CODE_LENGTHS", "SYMBOL", "DISTANCE", "TRUNCATED",
                "TOO_MUCH", "TOO_LITTLE", "ADLER", "FILTER"]


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
    assert "decode_png" in g.__all__ and g.decode_png.__module__ == "gaussianavatars_b200.png"
    # the header's status codes are the oracle's, in its order
    for i, name in enumerate(STATUS_NAMES):
        assert re.search(rf"GAB200_PNG_{name} = {i},?\s", hdr), name
        assert getattr(oi, name) == i
    strings = [L.gab200_png_status_string(i).decode() for i in range(12)]
    assert len(set(strings)) == 12 and strings[0] == "ok"
    assert L.gab200_png_status_string(12).decode() == L.gab200_png_status_string(-1).decode() == "unknown PNG status"


def test_scratch_sizes():
    from gaussianavatars_b200 import _native as N
    L = N.lib()
    for F, H, W in ((1, 1, 1), (16, 550, 802), (3, 1080, 1920), (1, 7, 11000)):
        stride = (H * (1 + 4 * W) + 255) // 256 * 256
        assert L.gab200_png_decode_scratch_bytes(F, H, W) == F * stride
    for F, H, W in ((0, 4, 4), (-1, 4, 4), (1, 0, 4), (1, 4, 0), (1, -3, 4), (1, 2**16, 2**15)):
        assert L.gab200_png_decode_scratch_bytes(F, H, W) == 0, (F, H, W)


def test_c_abi_refusals_before_any_device_work():
    from gaussianavatars_b200 import _native as N
    L = N.lib()
    buf = (C.c_uint8 * 1024)()
    p = C.cast(buf, C.c_void_p)
    al = C.c_void_p((p.value + 255) & ~255)
    # files, height, width, zdata, zoff, zlen, color_type, scratch, out, out_channels, status
    ok = [1, 3, 4, p, p, p, p, al, al, 4, p]
    for i, bad in ((0, 0), (0, -2), (1, 0), (2, 0), (1, 2**28), (3, None), (4, None), (5, None), (6, None), (7, None),
                   (8, None), (9, 1), (9, 2), (9, 5), (10, None), (7, C.c_void_p(al.value + 8)),
                   (8, C.c_void_p(al.value + 2))):
        args = list(ok)
        args[i] = bad
        assert L.gab200_png_decode(*args, None) == -1, (i, bad)


def _file(color=2, depth=8, interlace=0, W=4, H=3):
    ihdr = struct.pack(">IIBBBBB", W, H, depth, color, 0, 0, interlace)
    return pc.png_file(W, H, color, zlib.compress(b"\x00" * (H * (1 + 3 * W))), ihdr=ihdr)


def test_decode_png_refusals(tmp_path):
    from gaussianavatars_b200 import decode_png
    good = _file()
    for kw, field, what in (({"color": 0}, "colour type", "grey"), ({"color": 4}, "colour type", "grey\\+alpha"),
                            ({"color": 3}, "colour type", "palette"), ({"depth": 16}, "bit depth", "16-bit"),
                            ({"interlace": 1}, "interlace method", "interlaced")):
        with pytest.raises(ValueError, match=f"file 1: IHDR {field}: {what}"):
            decode_png([good, _file(**kw)])
    path = tmp_path / "grey.png"
    path.write_bytes(_file(color=0))
    with pytest.raises(ValueError, match=re.escape(f"file 0 ({path}): IHDR colour type: grey")):
        decode_png(str(path))
    with pytest.raises(ValueError, match="file 1: IHDR width/height: 5x3, but file 0 is 4x3"):
        decode_png([good, _file(W=5)])
    with pytest.raises(ValueError, match="file 0: not a PNG file"):
        decode_png(b"GIF89a" + good[6:])
    bad_ihdr = bytearray(good)
    bad_ihdr[29] ^= 1   # IHDR's CRC
    with pytest.raises(ValueError, match="file 0: CRC of chunk b'IHDR' does not match"):
        decode_png(bytes(bad_ihdr))
    text = pc.png_file(4, 3, 2, zlib.compress(b"\x00" * 39), before=[(b"tEXt", b"a\x00b")])
    bad_text = bytearray(text)
    bad_text[33 + 8 + 3] ^= 1   # inside tEXt's body
    with pytest.raises(ValueError, match="file 0: CRC of chunk b'tEXt' does not match"):
        decode_png(bytes(bad_text))
    with pytest.raises(ValueError, match="file 0: truncated before the image data"):
        decode_png(good[:40])
    with pytest.raises(ValueError, match="file 0: IHDR: the first chunk must be a 13-byte IHDR"):
        decode_png(good[:8] + pc.chunk(b"tEXt", b"a\x00b") + good[8:])
    with pytest.raises(ValueError, match="file 0: IHDR width/height: 0x3"):
        decode_png(_file(W=0))
    with pytest.raises(ValueError, match="channels must be 3 or 4"):
        decode_png(good, channels=1)
    with pytest.raises(ValueError, match="at least one file"):
        decode_png([])
    with pytest.raises(TypeError, match="file 0 must be bytes-like or a path"):
        decode_png([3])


def test_crc_rules_follow_pil():
    """PIL checks the CRCs of the chunks before the image data, not IDAT's or IEND's: a file with a bad IDAT or IEND
    CRC passes the host walk."""
    from PIL import Image
    from gaussianavatars_b200.png import parse_png
    f = pc.png_file(4, 3, 2, zlib.compress(b"\x00" * 39))
    for at in (len(f) - 1, len(f) - 13):   # IEND's CRC, IDAT's CRC
        g = bytearray(f)
        g[at] ^= 0x10
        assert parse_png(bytes(g), "x")[3] == parse_png(f, "x")[3]
        Image.open(io.BytesIO(bytes(g))).convert("RGBA")


def test_add_png_refusals(no_device):
    from gaussianavatars_b200.frames import FrameStore
    store = FrameStore.__new__(FrameStore)
    for bad in (0, -1, 2.5, True):
        with pytest.raises(ValueError, match="batch must be a positive int"):
            store.add_png([], batch=bad)
