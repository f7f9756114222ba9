"""A plain restatement of RFC 1950/1951 inflate with zlib's validity rules (inflate.c, inftrees.c), and of the PNG
row unfilter -- the reference csrc/png_decode.cu is tested against.

    out, status, report = inflate(stream, expected=None)     # bytes, the first error (STATUS), the paths taken
    rgba, status, report = decode_idat(idat, width, height, color_type)

The status is the first error in stream order, as include/gab200_rasterizer.h's gab200_png_status lists them.  A
Huffman code is read one bit at a time (RFC 1951 3.2.2's canonical codes): a code cut off by the end of the data is
TRUNCATED; an unused code of an incomplete tree (zlib allows only an empty tree or a single code of length 1) is
SYMBOL after one bit.  A stored block copies byte by byte, each byte read before it is written, so when the data and
the room end at the same byte the data ends first.  With `expected` the stream must inflate to exactly that many bytes
(TOO_MUCH when a literal, match or stored byte would pass it, TOO_LITTLE at the end of the final block, before the
Adler-32 is read); without it the stream is checked as zlib.decompress checks it.  Nothing after the Adler-32 is read.

The report is the set of paths the stream took, named as the tests' corpus table names them.
"""
from __future__ import annotations

import numpy as np

from oracle.png import CL_ORDER, _DIST_BASE, _DIST_EXTRA, _LEN_BASE, _LEN_EXTRA

OK, ZLIB_HEADER, BLOCK_TYPE, STORED_LENGTH, CODE_LENGTHS, SYMBOL, DISTANCE, TRUNCATED, TOO_MUCH, TOO_LITTLE, ADLER, \
    FILTER = range(12)
STATUS = ("ok", "zlib header", "block type", "stored length", "code lengths", "symbol", "distance too far",
          "truncated input", "too much data", "too little data", "Adler-32", "filter type")


class _Fail(Exception):
    def __init__(self, status):
        self.status = status


class _Bits:
    def __init__(self, data: bytes):
        self.data, self.pos, self.nbits = data, 0, 8 * len(data)

    def bit(self) -> int:
        if self.pos >= self.nbits:
            raise _Fail(TRUNCATED)
        b = (self.data[self.pos >> 3] >> (self.pos & 7)) & 1
        self.pos += 1
        return b

    def bits(self, n: int) -> int:
        v = 0
        for i in range(n):
            v |= self.bit() << i
        return v

    def align(self):
        self.pos = (self.pos + 7) & ~7


class _Code:
    """A canonical Huffman code (puff's count / symbol tables); `valid` is zlib's rule for the tree's kind."""

    def __init__(self, lens, allow_incomplete: bool):
        self.count = [0] * 16
        for n in lens:
            self.count[n] += 1
        self.count[0] = 0
        left = 1
        for n in range(1, 16):
            left = 2 * left - self.count[n]
            if left < 0:
                break
        self.max = max((n for n in range(1, 16) if self.count[n]), default=0)
        self.valid = left == 0 or (left > 0 and allow_incomplete and self.max <= 1)
        offs = [0] * 16
        for n in range(1, 15):
            offs[n + 1] = offs[n] + self.count[n]
        self.symbol = [0] * sum(self.count)
        for s, n in enumerate(lens):
            if n:
                self.symbol[offs[n]] = s
                offs[n] += 1

    def decode(self, br: _Bits) -> tuple:
        """(symbol or None for an unused code, bits read)."""
        code = first = index = 0
        for n in range(1, max(self.max, 1) + 1):
            code |= br.bit()
            count = self.count[n] if n <= 15 else 0
            if code - count < first:
                return self.symbol[index + code - first], n
            index += count
            first = (first + count) << 1
            code <<= 1
        return None, max(self.max, 1)


_FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
_FIXED_DIST = [5] * 32
LIT_ROOT, DIST_ROOT = 9, 6   # the device's primary table bits: a longer code goes through a sub-table


def _dynamic(br: _Bits, report: set) -> tuple:
    hlit, hdist, hclen = br.bits(5) + 257, br.bits(5) + 1, br.bits(4) + 4
    if hlit > 286 or hdist > 30:
        raise _Fail(CODE_LENGTHS)
    report.update({f"hlit_{hlit}", f"hdist_{hdist}", f"hclen_{hclen}"})
    cl = [0] * 19
    for i in range(hclen):
        cl[CL_ORDER[i]] = br.bits(3)
    clc = _Code(cl, False)
    if not clc.valid:
        raise _Fail(CODE_LENGTHS)
    total, lens = hlit + hdist, []
    while len(lens) < total:
        sym, _ = clc.decode(br)
        if sym < 16:
            lens.append(sym)
            continue
        if sym == 16:
            rep = 3 + br.bits(2)
            if not lens:
                raise _Fail(CODE_LENGTHS)
            val = lens[-1]
            report.add({3: "rep16_min", 6: "rep16_max"}.get(rep, "rep16"))
        elif sym == 17:
            rep, val = 3 + br.bits(3), 0
            report.add({3: "rep17_min", 10: "rep17_max"}.get(rep, "rep17"))
        else:
            rep, val = 11 + br.bits(7), 0
            report.add({11: "rep18_min", 138: "rep18_max"}.get(rep, "rep18"))
        if len(lens) + rep > total:
            raise _Fail(CODE_LENGTHS)
        if len(lens) < hlit < len(lens) + rep:
            report.add("repeat_crosses_into_distances")
        lens += [val] * rep
    if lens[256] == 0:
        raise _Fail(CODE_LENGTHS)
    lit, dist = _Code(lens[:hlit], True), _Code(lens[hlit:], True)
    if not lit.valid or not dist.valid:
        raise _Fail(CODE_LENGTHS)
    if dist.max == 0:
        report.add("no_distance_codes")
    elif sum(dist.count) == 1:
        report.add("single_distance_code")
    return lit, dist


def inflate(data: bytes, expected: int | None = None) -> tuple:
    """(the inflated bytes as far as they went, status, report) of a zlib stream."""
    out, report = bytearray(), set()
    try:
        status = _inflate(_Bits(bytes(data)), out, expected, report)
    except _Fail as e:
        status = e.status
    return bytes(out), status, report


def _room(out, n, expected):
    if expected is not None and len(out) + n > expected:
        raise _Fail(TOO_MUCH)


def _inflate(br: _Bits, out: bytearray, expected, report: set) -> int:
    cmf, flg = br.bits(8), br.bits(8)
    if (cmf * 256 + flg) % 31 or cmf & 15 != 8 or cmf >> 4 > 7 or flg & 32:
        raise _Fail(ZLIB_HEADER)
    report.add(f"wbits_{(cmf >> 4) + 8}")
    fixed = None
    blocks, last, after_huffman = 0, 0, False
    while not last:
        last, btype = br.bit(), br.bits(2)
        blocks += 1
        if btype == 3:
            raise _Fail(BLOCK_TYPE)
        if btype == 0:
            if after_huffman and br.pos & 7:
                report.add("stored_after_huffman_unaligned")
            br.align()
            n, nn = br.bits(16), br.bits(16)
            if n != (~nn & 0xFFFF):
                raise _Fail(STORED_LENGTH)
            report.add({0: "stored_empty", 65535: "stored_65535"}.get(n, "stored"))
            for _ in range(n):
                b = br.bits(8)
                _room(out, 1, expected)
                out.append(b)
            after_huffman = False
            continue
        if btype == 1:
            fixed = fixed or (_Code(_FIXED_LIT, False), _Code(_FIXED_DIST, False))
            lit, dist = fixed
        else:
            lit, dist = _dynamic(br, report)
        start = len(out)
        while True:
            sym, nb = lit.decode(br)
            if sym is None:
                raise _Fail(SYMBOL)
            if btype == 2 and nb > LIT_ROOT:
                report.add(f"lit_sub_table_{nb}")
            if sym < 256:
                _room(out, 1, expected)
                out.append(sym)
                continue
            if sym == 256:
                break
            if sym > 285:
                raise _Fail(SYMBOL)
            i = sym - 257
            extra = br.bits(_LEN_EXTRA[i])
            length = _LEN_BASE[i] + extra
            ds, nb = dist.decode(br)
            if ds is None or ds > 29:
                raise _Fail(SYMBOL)
            if btype == 2 and nb > DIST_ROOT:
                report.add(f"dist_sub_table_{nb}")
            d = _DIST_BASE[ds] + br.bits(_DIST_EXTRA[ds])
            if d > len(out):
                raise _Fail(DISTANCE)
            _room(out, length, expected)
            if length == 258:
                report.add("length_258_code_285" if sym == 285 else "length_258_code_284_31")
            if d == 32768:
                report.add("distance_32768")
            if d < length:
                report.add(f"overlap_d{d}" if d <= 4 else "overlap")
            for k in range(length):
                out.append(out[-d])
        report.add(("fixed" if btype == 1 else "dynamic") + ("_empty" if len(out) == start else ""))
        after_huffman = True
    report.add("blocks_many" if blocks >= 8 else f"blocks_{blocks}")
    if expected is not None and len(out) != expected:
        raise _Fail(TOO_LITTLE)
    br.align()
    want = 0
    for _ in range(4):
        want = (want << 8) | br.bits(8)
    if want != adler32(out):
        raise _Fail(ADLER)
    return OK


def adler32(data) -> int:
    a, b = 1, 0
    arr = np.frombuffer(bytes(data), np.uint8).astype(np.int64)
    for i in range(0, len(arr), 5552):
        blk = arr[i:i + 5552]
        b = (b + len(blk) * a + int(np.cumsum(blk).sum())) % 65521
        a = (a + int(blk.sum())) % 65521
    return (b << 16) | a


def unfilter(stream: bytes, width: int, height: int, c: int) -> tuple:
    """(raw pixels (H, W, c) uint8, status, the filter types used) of a filtered stream of H rows of 1 + W c bytes
    (the PNG specification's five filters, bytes per pixel c)."""
    rs = 1 + width * c
    buf = np.frombuffer(stream, np.uint8).reshape(height, rs)
    raw = np.zeros((height, width * c), np.int64)
    used = set()
    for y in range(height):
        ft = int(buf[y, 0])
        if ft > 4:
            return None, FILTER, used
        used.add(ft)
        x = buf[y, 1:].astype(np.int64)
        up = raw[y - 1] if y else np.zeros(width * c, np.int64)
        if ft in (0, 2):
            raw[y] = (x + (up if ft == 2 else 0)) & 255
            continue
        row = raw[y]
        for i in range(width * c):
            a = int(row[i - c]) if i >= c else 0
            b = int(up[i])
            cc = int(up[i - c]) if i >= c else 0
            if ft == 1:
                p = a
            elif ft == 3:
                p = (a + b) >> 1
            else:
                pa, pb, pc = abs(b - cc), abs(a - cc), abs(a + b - 2 * cc)
                p = a if pa <= pb and pa <= pc else (b if pb <= pc else cc)
            row[i] = (int(x[i]) + p) & 255
    return raw.astype(np.uint8).reshape(height, width, c), OK, used


def decode_idat(idat: bytes, width: int, height: int, color_type: int) -> tuple:
    """(RGBA pixels (H, W, 4) uint8 or None, status, report) of a PNG's concatenated IDAT data: inflate to exactly
    H (1 + W c) bytes, then unfilter; RGB gets alpha 255.  A filter error is reported only for a valid stream."""
    c = 4 if color_type == 6 else 3
    stream, status, report = inflate(idat, height * (1 + width * c))
    if status != OK:
        return None, status, report
    raw, status, used = unfilter(stream, width, height, c)
    report |= {f"filter_{f}" for f in used}
    if status != OK:
        return None, status, report
    if c == 3:
        raw = np.concatenate([raw, np.full((height, width, 1), 255, np.uint8)], axis=2)
    return raw, OK, report
