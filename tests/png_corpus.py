"""The PNG decoder's test corpus: a deflate writer that emits exactly the blocks, codes and repeats it is told to, a
PNG writer with forced row filters, split IDATs and ancillary chunks, and the streams and files built from them
(tests/test_oracle_inflate.py checks them against zlib and PIL on the CPU, tests/test_gpu_png_decode.py against the
device).  Every stream is built from a fixed seed."""
from __future__ import annotations

import heapq
import io
import struct
import zlib

import numpy as np

from oracle import inflate as oi
from oracle.png import CL_ORDER, _DIST_BASE, _DIST_EXTRA, _LEN_BASE, _LEN_EXTRA


# ---- deflate writer -------------------------------------------------------------------------------------------------
class BitWriter:
    def __init__(self):
        self.acc, self.n, self.out = 0, 0, bytearray()

    def bits(self, v: int, n: int):
        self.acc |= (v & ((1 << n) - 1)) << self.n
        self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def code(self, code: int, n: int):   # a Huffman code, most significant bit first
        self.bits(int(format(code, f"0{n}b")[::-1], 2) if n else 0, n)

    def align(self):
        if self.n:
            self.bits(0, 8 - self.n)

    def data(self) -> bytes:
        return bytes(self.out) + (bytes([self.acc]) if self.n else b"")


def canonical(lens) -> list:
    count = [0] * 16
    for n in lens:
        count[n] += 1
    count[0] = 0
    nxt, code = [0] * 16, 0
    for n in range(1, 16):
        code = (code + count[n - 1]) << 1
        nxt[n] = code
    out = []
    for n in lens:
        out.append(nxt[n] if n else None)
        if n:
            nxt[n] += 1
    return out


def huffman(freq) -> list:
    """Code lengths of a complete prefix code over the symbols of nonzero freq (one used symbol: length 1)."""
    used = [s for s, f in enumerate(freq) if f]
    lens = [0] * len(freq)
    if len(used) == 1:
        lens[used[0]] = 1
        return lens
    heap = [(freq[s], i, [s]) for i, s in enumerate(used)]
    heapq.heapify(heap)
    k = len(heap)
    while len(heap) > 1:
        f1, _, a = heapq.heappop(heap)
        f2, _, b = heapq.heappop(heap)
        for s in a + b:
            lens[s] += 1
        heapq.heappush(heap, (f1 + f2, k, a + b))
        k += 1
    assert max(lens) <= 15
    return lens


def len_symbol(length: int, as_284: bool = False) -> tuple:
    """(symbol, extra bits, extra value) of a match length; 258 as code 285, or as 284 + 31 when as_284."""
    if length == 258:
        return (284, 5, 31) if as_284 else (285, 0, 0)
    i = max(k for k in range(28) if _LEN_BASE[k] <= length)
    return 257 + i, _LEN_EXTRA[i], length - _LEN_BASE[i]


def dist_symbol(d: int) -> tuple:
    for i in range(29, -1, -1):
        if _DIST_BASE[i] <= d:
            return i, _DIST_EXTRA[i], d - _DIST_BASE[i]
    raise ValueError(d)


def rle(lens) -> list:
    """zlib-style greedy run-length coding of code lengths: [(symbol, extra value)]."""
    out, i = [], 0
    while i < len(lens):
        v, run = lens[i], 1
        while i + run < len(lens) and lens[i + run] == v:
            run += 1
        if v == 0 and run >= 3:
            take = min(run, 138)
            out.append((18, take - 11) if take >= 11 else (17, take - 3))
            i += take
            continue
        out.append((v, 0))
        i += 1
        run -= 1
        while run >= 3:
            take = min(run, 6)
            out.append((16, take - 3))
            i += take
            run -= take
    return out


CL_EXTRA = {16: 2, 17: 3, 18: 7}


def emit(w: BitWriter, tokens, lit_codes, lit_lens, dist_codes, dist_lens):
    for t in tokens:
        if t[0] == "lit":
            w.code(lit_codes[t[1]], lit_lens[t[1]])
        else:
            _, length, d, *opt = t
            s, eb, ev = len_symbol(length, bool(opt and opt[0]))
            w.code(lit_codes[s], lit_lens[s])
            w.bits(ev, eb)
            ds, deb, dev = dist_symbol(d)
            w.code(dist_codes[ds], dist_lens[ds])
            w.bits(dev, deb)
    w.code(lit_codes[256], lit_lens[256])


def stored(w: BitWriter, data: bytes, final: bool, nlen=None):
    w.bits(int(final), 1)
    w.bits(0, 2)
    w.align()
    n = len(data)
    w.bits(n, 16)
    w.bits((~n & 0xFFFF) if nlen is None else nlen, 16)
    for b in data:
        w.bits(b, 8)


FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8


def fixed(w: BitWriter, tokens, final: bool):
    w.bits(int(final), 1)
    w.bits(1, 2)
    emit(w, tokens, canonical(FIXED_LIT), FIXED_LIT, canonical([5] * 32), [5] * 32)


CL_DEFAULT = [4] * 13 + [5] * 6   # a complete code over all 19 code-length symbols (in CL_ORDER)


def dynamic(w: BitWriter, tokens, lit_lens, dist_lens, final: bool, cl_seq=None, cl_lens=None, hclen=19,
            hlit=None, hdist=None):
    """A dynamic block: lit_lens / dist_lens (their lengths are HLIT / HDIST unless given), the code lengths as cl_seq
    (default: rle), the code-length code's lengths cl_lens by symbol (default: CL_DEFAULT in CL_ORDER)."""
    cl_seq = rle(list(lit_lens) + list(dist_lens)) if cl_seq is None else cl_seq
    if cl_lens is None:
        cl_lens = [0] * 19
        for i, s in enumerate(CL_ORDER):
            cl_lens[s] = CL_DEFAULT[i]
    w.bits(int(final), 1)
    w.bits(2, 2)
    w.bits((len(lit_lens) if hlit is None else hlit) - 257, 5)
    w.bits((len(dist_lens) if hdist is None else hdist) - 1, 5)
    w.bits(hclen - 4, 4)
    for i in range(hclen):
        w.bits(cl_lens[CL_ORDER[i]], 3)
    clc = canonical(cl_lens)
    for s, x in cl_seq:
        w.code(clc[s], cl_lens[s])
        if s >= 16:
            w.bits(x, CL_EXTRA[s])
    emit(w, tokens, canonical(lit_lens), lit_lens, canonical(dist_lens), dist_lens)


def expand(tokens) -> bytes:
    out = bytearray()
    for t in tokens:
        if t[0] == "lit":
            out.append(t[1])
        else:
            for _ in range(t[1]):
                out.append(out[-t[2]])
    return bytes(out)


def zwrap(deflate: bytes, data: bytes, header=b"\x78\x9c", adler=None) -> bytes:
    a = zlib.adler32(data) & 0xFFFFFFFF if adler is None else adler
    return header + deflate + struct.pack(">I", a)


def freq_lens(tokens, n_lit=286, n_dist=30):
    """Huffman lengths of a block's tokens (EOB counted once)."""
    lf, df = [0] * n_lit, [0] * n_dist
    lf[256] = 1
    for t in tokens:
        if t[0] == "lit":
            lf[t[1]] += 1
        else:
            lf[len_symbol(t[1], bool(t[3:] and t[3]))[0]] += 1
            df[dist_symbol(t[2])[0]] += 1
    return huffman(lf), huffman(df) if any(df) else [0] * n_dist


# ---- the crafted streams ----------------------------------------------------------------------------------------------
def crafted_streams() -> list:
    """[(name, zlib stream, the bytes it inflates to)] -- every one valid, each reaching the path it is named for."""
    rng = np.random.default_rng(11)
    out = []

    def add(name, blocks_fn, data):
        w = BitWriter()
        blocks_fn(w)
        out.append((name, zwrap(w.data(), data), data))

    noise = bytes(rng.integers(0, 256, 70000, dtype=np.uint8))
    add("stored_0_and_65535", lambda w: (stored(w, b"", False), stored(w, noise[:65535], True)), noise[:65535])
    toks = [("lit", b) for b in b"abcde"]
    add("stored_after_fixed_unaligned",
        lambda w: (fixed(w, toks, False), stored(w, b"xyz", True)), b"abcdexyz")
    add("fixed_empty_and_many_blocks",
        lambda w: ([fixed(w, [("lit", 65 + i)], False) for i in range(9)], fixed(w, [], True)),
        bytes(range(65, 74)))
    t258 = [("lit", 7), ("m", 258, 1), ("m", 258, 1, True)]
    add("length_258_fixed", lambda w: fixed(w, t258, True), expand(t258))
    l, d = freq_lens(t258)
    add("length_258_dynamic", lambda w: dynamic(w, t258, l, d, True), expand(t258))
    far = [("lit", b) for b in noise[:32768]] + [("m", 200, 32768)]
    add("distance_32768", lambda w: fixed(w, far, True), expand(far))
    ov = [("lit", 1), ("lit", 2), ("lit", 3), ("lit", 4), ("m", 100, 1), ("m", 77, 3), ("m", 150, 4)]
    add("overlap_d1_d3_d4", lambda w: fixed(w, ov, True), expand(ov))
    single = [("lit", 9), ("m", 40, 1), ("lit", 10), ("m", 3, 1)]
    ls, _ = freq_lens(single)
    add("single_distance_code", lambda w: dynamic(w, single, ls, [1], True), expand(single))
    lits = [("lit", b) for b in b"no matches at all"]
    ll, _ = freq_lens(lits)
    add("no_distance_codes", lambda w: dynamic(w, lits, ll, [0], True), expand(lits))
    # code-length repeats: 16 at 3 and 6, 18 at 138 and 11, 17 at 10 and 3, and a 17 from the literal lengths into
    # the distance lengths (the lengths are coded by rle(); the used symbols were chosen so its runs are these)
    lit_used = list(range(149, 159)) + list(range(169, 256)) + [256, 257, 258, 259, 270, 274, 275, 276]
    lf = [0] * 286
    for s in lit_used:
        lf[s] = 5
    for s in range(149, 159):
        lf[s] = 1
    rep_l = huffman(lf)
    rep_d = [0] + [1, 1]   # distance 0 unused: the zero run 277..285 + dist 0 crosses HLIT
    rep_tok = [("lit", s) for s in range(149, 159)] + [("lit", 200), ("m", 3, 2), ("m", 4, 3)]
    add("repeats", lambda w: dynamic(w, rep_tok, rep_l, rep_d, True), expand(rep_tok))
    short = [3, 3, 3, 3] + [0] * 252 + [2, 2]   # 16 at its minimum count: 3, then three repeats of it
    st = [("lit", 2), ("lit", 0), ("m", 3, 1), ("lit", 3)]
    add("repeat16_min", lambda w: dynamic(w, st, short, [1], True), expand(st))
    # 15-bit codes in both trees: literals 0..12 at lengths 1..13, 13 at 14, EOB and 257 at 15; distances 0..13 at
    # 1..14, 14 and 15 at 15 (a Fibonacci-weighted alphabet's lengths)
    fl = [0] * 286
    for s in range(13):
        fl[s] = s + 1
    fl[13], fl[256], fl[257] = 14, 15, 15
    fd = [k + 1 for k in range(14)] + [15, 15] + [0] * 14
    fib = [("lit", s) for s in range(14)] + [("lit", 0)] * 200 + [("m", 3, 150), ("lit", 13), ("m", 3, 200)]
    add("codes_15_bits", lambda w: dynamic(w, fib, fl, fd, True), expand(fib))
    # HCLEN 4 cannot make a valid block (no length but 0); it appears among the refusals
    return out


def zlib_sweep(data: bytes) -> list:
    """[(name, stream)] of zlib at every level x strategy x wbits, and with full / sync flush points."""
    out = []
    strategies = {"default": zlib.Z_DEFAULT_STRATEGY, "filtered": zlib.Z_FILTERED, "huffman": zlib.Z_HUFFMAN_ONLY,
                  "rle": zlib.Z_RLE, "fixed": zlib.Z_FIXED}
    for level in range(10):
        for sname, st in strategies.items():
            for wbits in range(9, 16):
                c = zlib.compressobj(level, zlib.DEFLATED, wbits, 8, st)
                out.append((f"zlib_l{level}_{sname}_w{wbits}", c.compress(data) + c.flush()))
    for mode, flag in (("full", zlib.Z_FULL_FLUSH), ("sync", zlib.Z_SYNC_FLUSH)):
        c = zlib.compressobj(6)
        parts = [c.compress(data[i:i + 1000]) + c.flush(flag) for i in range(0, len(data), 1000)]
        out.append((f"zlib_{mode}_flush", b"".join(parts) + c.flush()))
    return out


# ---- PNG writer ----------------------------------------------------------------------------------------------------
def filter_rows(img: np.ndarray, filters) -> bytes:
    """The filtered stream of an (H, W, c) uint8 image, row y with filter filters[y % len(filters)]."""
    H, W, c = img.shape
    rows, prev = [], np.zeros(W * c, np.int64)
    for y in range(H):
        cur = img[y].reshape(-1).astype(np.int64)
        a = np.concatenate([np.zeros(c, np.int64), cur[:-c]])
        b = prev
        cc = np.concatenate([np.zeros(c, np.int64), prev[:-c]])
        f = filters[y % len(filters)]
        if f == 0:
            p = 0
        elif f == 1:
            p = a
        elif f == 2:
            p = b
        elif f == 3:
            p = (a + b) >> 1
        else:
            pa, pb, pc = np.abs(b - cc), np.abs(a - cc), np.abs(a + b - 2 * cc)
            p = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, cc))
        rows.append(bytes([f]) + ((cur - p) & 255).astype(np.uint8).tobytes())
        prev = cur
    return b"".join(rows)


def chunk(typ: bytes, body: bytes) -> bytes:
    return struct.pack(">I", len(body)) + typ + body + struct.pack(">I", zlib.crc32(typ + body) & 0xFFFFFFFF)


def png_file(width: int, height: int, color: int, idat: bytes, split=None, before=(), ihdr=None) -> bytes:
    """A PNG file: IHDR (its 13 bytes may be given), the `before` chunks, the IDAT data as one chunk or cut at the
    sizes in `split` (0: an empty IDAT), IEND."""
    body = ihdr if ihdr is not None else struct.pack(">IIBBBBB", width, height, 8, color, 0, 0, 0)
    parts, pos = [], 0
    for n in (split or []):
        parts.append(idat[pos:pos + n])
        pos += n
    parts.append(idat[pos:])
    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", body) + b"".join(chunk(t, b) for t, b in before) +
            b"".join(chunk(b"IDAT", p) for p in parts) + chunk(b"IEND", b""))


def pil_png(img: np.ndarray, **kw) -> bytes:
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(img, "RGBA" if img.shape[2] == 4 else "RGB").save(buf, "PNG", **kw)
    return buf.getvalue()


def pil_pixels(data: bytes) -> np.ndarray:
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGBA"))


def images(seed: int = 5) -> dict:
    """Small CPU-made images: noise, flat, RGB runs (overlapping copies at d = 3 and 4), odd sizes, a long row."""
    rng = np.random.default_rng(seed)
    out = {}
    for c in (3, 4):
        out[f"noise_{c}"] = rng.integers(0, 256, (9, 13, c), dtype=np.uint8)
        out[f"flat_{c}"] = np.full((12, 10, c), 77, np.uint8)
        run = np.tile(rng.integers(0, 256, (1, 1, c), dtype=np.uint8), (6, 40, 1))
        out[f"runs_{c}"] = run
        out[f"gradient_{c}"] = (np.arange(16 * 24 * c).reshape(16, 24, c) * 7 % 256).astype(np.uint8)
        out[f"1x1_{c}"] = rng.integers(0, 256, (1, 1, c), dtype=np.uint8)
        out[f"1xN_{c}"] = rng.integers(0, 256, (1, 37, c), dtype=np.uint8)
        out[f"Nx1_{c}"] = rng.integers(0, 256, (41, 1, c), dtype=np.uint8)
        out[f"long_row_{c}"] = rng.integers(0, 256, (2, 8300 if c == 4 else 11000, c), dtype=np.uint8)
    return out


def valid_files() -> list:
    """[(name, PNG bytes, (H, W, c) pixels)] on the CPU: the test's own writer (every filter, forced per row and
    mixed; split, empty and ancillary chunks) and PIL at every level and optimize."""
    out = []
    for name, img in images().items():
        H, W, c = img.shape
        color = 6 if c == 4 else 2
        for filters in ([0], [1], [2], [3], [4], [0, 1, 2, 3, 4]):
            if len(filters) > 1 or not name.startswith("long_row"):
                stream = filter_rows(img, filters)
                out.append((f"{name}_f{''.join(map(str, filters))}", png_file(W, H, color, zlib.compress(stream, 6)),
                            img))
        stream = filter_rows(img, [4, 3, 2, 1, 0])
        idat = zlib.compress(stream, 9)
        out.append((f"{name}_split1", png_file(W, H, color, idat, split=[1] * min(len(idat), 40)), img))
        out.append((f"{name}_empty_idats", png_file(W, H, color, idat, split=[0, 0, len(idat) // 2, 0]), img))
        out.append((f"{name}_ancillary",
                    png_file(W, H, color, idat, before=[(b"tEXt", b"Comment\x00x"), (b"gAMA", b"\x00\x00\xb1\x8f")]),
                    img))
        if not name.startswith("long_row"):
            for level in range(10):
                out.append((f"{name}_pil{level}", pil_png(img, compress_level=level), img))
            out.append((f"{name}_pil_opt", pil_png(img, optimize=True), img))
    return out


# ---- refusals ---------------------------------------------------------------------------------------------------------
def _fcheck(cmf: int, flg_hi: int) -> bytes:
    flg = flg_hi & 0xE0
    flg += (31 - (cmf * 256 + flg) % 31) % 31
    return bytes([cmf, flg])


def error_streams() -> list:
    """[(name, IDAT data, width, height, colour type, expected status)]: each built to fail in one named way."""
    W, H, c = 4, 3, 3
    n = H * (1 + W * c)
    raw = bytes([0] + [10] * (W * c)) * H
    good = zlib.compress(raw)
    out = []

    def blocks(fn, data=raw, header=b"\x78\x9c", adler=None):
        w = BitWriter()
        fn(w)
        return zwrap(w.data(), data, header, adler)

    lits = [("lit", b) for b in raw]
    fl = canonical(FIXED_LIT)
    e = [("cm_not_8", _fcheck(0x77, 0) + good[2:], oi.ZLIB_HEADER),
         ("cinfo_8", _fcheck(0x88, 0) + good[2:], oi.ZLIB_HEADER),
         ("fcheck", b"\x78\x00" + good[2:], oi.ZLIB_HEADER),
         ("fdict", _fcheck(0x78, 0x20) + b"\x00\x00\x00\x01" + good[2:], oi.ZLIB_HEADER),
         ("block_type_3", b"\x78\x9c\x07\x00", oi.BLOCK_TYPE),
         ("stored_nlen", blocks(lambda w: stored(w, raw, True, nlen=0x1234)), oi.STORED_LENGTH)]
    ll, _ = freq_lens(lits)
    e.append(("hlit_287", blocks(lambda w: dynamic(w, lits, ll, [0], True, hlit=287)), oi.CODE_LENGTHS))
    e.append(("hdist_31", blocks(lambda w: dynamic(w, lits, ll, [0] * 31, True)), oi.CODE_LENGTHS))
    cl_over = [1] * 19
    e.append(("cl_oversubscribed", blocks(lambda w: dynamic(w, lits, ll, [0], True, cl_lens=cl_over)),
              oi.CODE_LENGTHS))
    cl_inc = [0] * 19
    cl_inc[0] = 1
    e.append(("cl_incomplete", blocks(lambda w: dynamic(w, lits, ll, [0], True, cl_lens=cl_inc, cl_seq=[(0, 0)] * 3)),
              oi.CODE_LENGTHS))
    e.append(("hclen_4", blocks(lambda w: dynamic(w, lits, ll, [0], True, hclen=4,
                                                  cl_lens=[2, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 2, 2],
                                                  cl_seq=[(18, 127), (18, 127), (17, 7)])), oi.CODE_LENGTHS))
    e.append(("repeat16_first", blocks(lambda w: dynamic(w, lits, ll, [0], True, cl_seq=[(16, 0)])), oi.CODE_LENGTHS))
    e.append(("repeat_past_end", blocks(lambda w: dynamic(w, lits, ll, [0], True,
                                                          cl_seq=rle(ll)[:-1] + [(18, 127)])), oi.CODE_LENGTHS))
    no_eob = list(ll)
    no_eob[256] = 0
    e.append(("no_code_256", blocks(lambda w: dynamic(w, [], no_eob, [0], True, cl_seq=rle(no_eob + [0]))),
              oi.CODE_LENGTHS))
    over = list(ll)
    over[0] = over[1] = over[2] = 1
    e.append(("lit_oversubscribed", blocks(lambda w: dynamic(w, [], over, [0], True, cl_seq=rle(over + [0]))),
              oi.CODE_LENGTHS))
    inc = [0] * 257
    inc[10] = inc[256] = 2
    e.append(("lit_incomplete", blocks(lambda w: dynamic(w, [], inc, [0], True, cl_seq=rle(inc + [0]))),
              oi.CODE_LENGTHS))
    e.append(("dist_oversubscribed", blocks(lambda w: dynamic(w, [], ll, [1, 1, 1], True,
                                                              cl_seq=rle(ll + [1, 1, 1]))), oi.CODE_LENGTHS))
    e.append(("dist_incomplete", blocks(lambda w: dynamic(w, [], ll, [2, 2, 0, 2], True,
                                                          cl_seq=rle(ll + [2, 2, 0, 2]))), oi.CODE_LENGTHS))

    def fixed_raw(w, codes):
        w.bits(1, 1)
        w.bits(1, 2)
        for s, extra in codes:
            w.code(fl[s], FIXED_LIT[s])
            for v, nb in extra:
                w.bits(v, nb)
    e.append(("fixed_286", blocks(lambda w: fixed_raw(w, [(65, []), (286, [])])), oi.SYMBOL))
    e.append(("fixed_287", blocks(lambda w: fixed_raw(w, [(65, []), (287, [])])), oi.SYMBOL))
    e.append(("dist_30", blocks(lambda w: (fixed_raw(w, [(65, []), (257, [])]), w.code(30, 5))), oi.SYMBOL))
    e.append(("dist_31", blocks(lambda w: (fixed_raw(w, [(65, []), (257, [])]), w.code(31, 5))), oi.SYMBOL))
    e.append(("empty_dist_tree_used", blocks(lambda w: dynamic(w, [("lit", 1), ("m", 3, 1)], freq_lens(
        [("lit", 1), ("m", 3, 1)])[0], [0], True)), oi.SYMBOL))
    e.append(("distance_before_first_byte", blocks(lambda w: fixed(w, [("lit", 0), ("m", 3, 2)], True)),
              oi.DISTANCE))
    e.append(("ends_inside_block", good[:len(good) // 2], oi.TRUNCATED))
    e.append(("ends_before_adler", good[:-2], oi.TRUNCATED))
    e.append(("too_much", zlib.compress(raw + b"\x00"), oi.TOO_MUCH))
    e.append(("too_little", zlib.compress(raw[:-1]), oi.TOO_LITTLE))
    e.append(("too_much_stored", blocks(lambda w: stored(w, raw + b"\x00", True), raw + b"\x00"), oi.TOO_MUCH))
    e.append(("wrong_adler", good[:-1] + bytes([good[-1] ^ 1]), oi.ADLER))
    e.append(("filter_5", zlib.compress(bytes([5]) + raw[1:]), oi.FILTER))
    for name, data, st in e:
        out.append((name, data, W, H, 2, st))
    assert all(len(x) == 6 for x in out) and n == len(raw)
    return out


def mutations(files, count: int = 300, seed: int = 2024) -> list:
    """[(name, IDAT data, width, height, colour type)]: byte flips and truncations of the given (name, IDAT, W, H,
    colour) streams, a fixed seeded set."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(count):
        name, idat, W, H, color = files[k % len(files)]
        b = bytearray(idat)
        if k % 4 == 3:
            cut = int(rng.integers(0, len(b)))
            out.append((f"{name}_cut{cut}", bytes(b[:cut]), W, H, color))
            continue
        for _ in range(1 + k % 3):
            i = int(rng.integers(0, len(b)))
            b[i] ^= 1 << int(rng.integers(0, 8))
        out.append((f"{name}_flip{k}", bytes(b), W, H, color))
    return out


def mutation_bases() -> list:
    """Small valid streams of every block kind the mutations start from."""
    rng = np.random.default_rng(9)
    img = rng.integers(0, 40, (6, 7, 4), dtype=np.uint8)
    img[:, 3:] = img[:, :1]
    stream = filter_rows(img, [0, 1, 2, 3, 4])
    out = []
    for level, st in ((0, zlib.Z_DEFAULT_STRATEGY), (1, zlib.Z_FIXED), (6, zlib.Z_DEFAULT_STRATEGY),
                      (9, zlib.Z_HUFFMAN_ONLY)):
        c = zlib.compressobj(level, zlib.DEFLATED, 15, 8, st)
        out.append((f"l{level}_s{st}", c.compress(stream) + c.flush(), 7, 6, 6))
    return out
