"""numpy restatement of the PNG encoder (gaussianavatars_b200/csrc/png.cu, DESIGN.md section 4.5), byte for byte.
TEST INFRASTRUCTURE ONLY: imported by tests/, never by the product.

The filter rule is libpng's minimum-sum-of-absolute-values heuristic: each filtered byte v counts v < 128 ? v : 256 - v,
the row takes the filter with the least sum, and a tie goes to the lowest filter id (0 None, 1 Sub, 2 Up, 3 Average,
4 Paeth).  PIL does not follow this rule exactly, so its files are not the oracle.

`encode_png` restates the rest: the filtered stream cut into 32 KiB segments; per segment the five match candidates,
the minimum match by distance, the greedy parse, the dynamic Huffman codes (leaves ordered by (count, symbol),
Moffat-Katajainen lengths, miniz's length limit), the RLE header, the exact costs and both tie rules; then the blocks
packed LSB first, the zlib stream and the chunks.  Beside the file it reports, per segment, which paths of the encoder
the segment took (`SegmentReport`), so a test can show which rare branches an input reaches.
"""
from __future__ import annotations

import dataclasses
import struct
import zlib

import numpy as np

BPP = 3                  # bytes per pixel: 8-bit RGB
SEGMENT = 32768          # filtered bytes per deflate block
WINDOW = 32768           # the deflate window: matches reach this far back, into earlier segments of the same image
ROUND = 1024             # positions whose matches are searched together (the hash table holds the rounds before)
NEAR_SCAN = 256          # positions of the current round searched back for the same 3-byte hash
HASH_BITS = 13
MAX_MATCH = 258
LIT_SYMS, DIST_SYMS, CL_SYMS = 286, 30, 19
CL_ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)
PIECE = 65536            # bytes of the IDAT chunk's type and data per CRC piece
FILTERS = ("none", "sub", "up", "average", "paeth")

# RFC 1951 section 3.2.5: (base, extra bits) of length symbols 257..285 and distance symbols 0..29
_LEN_BASE = (3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195,
             227, 258)
_LEN_EXTRA = (0,) * 8 + (1,) * 4 + (2,) * 4 + (3,) * 4 + (4,) * 4 + (5,) * 4 + (0,)
_DIST_BASE = (1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
              4097, 6145, 8193, 12289, 16385, 24577)
_DIST_EXTRA = (0, 0, 0, 0) + tuple(e for e in range(1, 14) for _ in range(2))


def _code_table(base, extra, first_sym, top):
    """(symbol, extra bits, extra value) for every value 0..top, from an RFC table of bases and extra bits."""
    sym, eb, ev = np.zeros(top + 1, np.int64), np.zeros(top + 1, np.int64), np.zeros(top + 1, np.int64)
    for i, (b, e) in enumerate(zip(base, extra)):
        hi = min(b + (1 << e), top + 1)
        sym[b:hi], eb[b:hi], ev[b:hi] = first_sym + i, e, np.arange(hi - b)
    return sym, eb, ev


_LEN_SYM, _LEN_EB, _LEN_EV = _code_table(_LEN_BASE, _LEN_EXTRA, 257, MAX_MATCH)
_DIST_SYM, _DIST_EB, _DIST_EV = _code_table(_DIST_BASE, _DIST_EXTRA, 0, WINDOW)


def filter_row(cur: np.ndarray, prev: np.ndarray | None, ftype: int) -> np.ndarray:
    """Row `cur` (3W uint8) filtered with filter `ftype` against the row above (None: the first row, all zero)."""
    x = cur.astype(np.int32)
    b = np.zeros_like(x) if prev is None else prev.astype(np.int32)
    a = np.concatenate([np.zeros(BPP, np.int32), x[:-BPP]])[:x.size]
    c = np.concatenate([np.zeros(BPP, np.int32), b[:-BPP]])[:x.size]
    if ftype == 0:
        pred = np.zeros_like(x)
    elif ftype == 1:
        pred = a
    elif ftype == 2:
        pred = b
    elif ftype == 3:
        pred = (a + b) >> 1
    elif ftype == 4:
        p = a + b - c
        pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
        pred = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
    else:
        raise ValueError(f"a PNG filter id is 0..4, got {ftype}")
    return ((x - pred) & 255).astype(np.uint8)


def row_cost(filtered: np.ndarray) -> int:
    """The heuristic's sum: every byte read as a signed magnitude."""
    v = filtered.astype(np.int64)
    return int(np.where(v < 128, v, 256 - v).sum())


def choose_filter(cur: np.ndarray, prev: np.ndarray | None) -> tuple:
    """(filter id, filtered row) the rule picks for one row."""
    best, best_row, best_cost = 0, None, None
    for f in range(5):
        row = filter_row(cur, prev, f)
        cost = row_cost(row)
        if best_cost is None or cost < best_cost:
            best, best_row, best_cost = f, row, cost
    return best, best_row


def filter_image(rgb: np.ndarray) -> tuple:
    """(filter ids (H,), filtered stream (H * (3W + 1),) uint8) of an (H, W, 3) uint8 image."""
    H, W, _ = rgb.shape
    rows = rgb.reshape(H, 3 * W)
    ids, out = np.zeros(H, np.uint8), np.zeros((H, 3 * W + 1), np.uint8)
    for y in range(H):
        f, row = choose_filter(rows[y], rows[y - 1] if y else None)
        ids[y], out[y, 0], out[y, 1:] = f, f, row
    return ids, out.reshape(-1)


def filtered_bytes(width: int, height: int) -> int:
    return height * (3 * width + 1)


def segments(width: int, height: int) -> int:
    """Deflate blocks of a file: one per SEGMENT filtered bytes, the last one shorter."""
    return -(-filtered_bytes(width, height) // SEGMENT)


def png_bound(width: int, height: int) -> int:
    """The largest file of a width x height image: signature 8, IHDR 25, IDAT chunk 12, zlib header 2 and Adler-32 4,
    IEND 12, and the deflate stream, at most every block stored (3 header bits, <= 7 bits of padding, LEN and NLEN:
    42 bits <= 6 bytes per block) -- 63 + n + 6 S."""
    if width <= 0 or height <= 0:
        raise ValueError(f"a PNG has a positive size, got {width}x{height}")
    n = filtered_bytes(width, height)
    return 63 + n + 6 * segments(width, height)


# ---- the deflate encode --------------------------------------------------------------------------------------------
def hash3(buf: np.ndarray, at: np.ndarray) -> np.ndarray:
    """The 13-bit multiplicative hash of the 3 bytes at each position `at` of `buf`."""
    v = buf[at].astype(np.uint64) | (buf[at + 1].astype(np.uint64) << 8) | (buf[at + 2].astype(np.uint64) << 16)
    return ((v * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) >> np.uint64(32 - HASH_BITS)


def min_match(dist: np.ndarray) -> np.ndarray:
    """The shortest match worth its distance: 3 up to 64, 4 up to 4096, 5 beyond."""
    return np.where(dist <= 64, 3, np.where(dist <= 4096, 4, 5))


def _match_lengths(words: np.ndarray, at: np.ndarray, dist: np.ndarray, maxlen: np.ndarray) -> np.ndarray:
    """Longest common prefix, at most maxlen, of the bytes at `at` and `dist` before; words[i] holds bytes i..i+7."""
    n = np.zeros(at.size, np.int64)
    live = np.arange(at.size)
    while live.size:
        x = words[at[live] + n[live]] ^ words[at[live] - dist[live] + n[live]]
        same = x == 0
        low = x[~same]
        n[live[~same]] += np.log2((low & (~low + np.uint64(1))).astype(np.float64)).astype(np.int64) // 8
        n[live[same]] += 8
        live = live[same]
        live = live[n[live] < maxlen[live]]
    return np.minimum(n, maxlen)


def _two_used(freq: list) -> list:
    """At least two used symbols per tree: the lowest unused symbols get a count of one."""
    freq = list(freq)
    used = sum(1 for f in freq if f)
    for s in range(len(freq)):
        if used >= 2:
            break
        if freq[s] == 0:
            freq[s], used = 1, used + 1
    return freq


def huffman_lengths(freq: list, maxbits: int) -> tuple:
    """(code lengths, deepest leaf before the limit, deepest after) of counts `freq` (two or more nonzero): leaves
    ordered by (count, symbol), Moffat and Katajainen's in-place minimum-redundancy lengths, then miniz's limit -- every
    leaf deeper than maxbits moves to maxbits, and while the Kraft sum is over, one maxbits leaf goes and the deepest
    shorter leaf splits -- with the longest codes given to the rarest leaves."""
    order = [s for _, s in sorted((f, s) for s, f in enumerate(freq) if f)]
    m = len(order)
    A = [freq[s] for s in order]
    A[0] += A[1]
    root, leaf = 0, 2
    for nxt in range(1, m - 1):          # parent pointers
        if leaf >= m or A[root] < A[leaf]:
            A[nxt], A[root] = A[root], nxt
            root += 1
        else:
            A[nxt] = A[leaf]
            leaf += 1
        if leaf >= m or (root < nxt and A[root] < A[leaf]):
            A[nxt] += A[root]
            A[root] = nxt
            root += 1
        else:
            A[nxt] += A[leaf]
            leaf += 1
    A[m - 2] = 0                         # internal depths
    for nxt in range(m - 3, -1, -1):
        A[nxt] = A[A[nxt]] + 1
    avbl, used, depth, root, nxt = 1, 0, 0, m - 2, m - 1
    while avbl > 0:                      # leaf depths
        while root >= 0 and A[root] == depth:
            used, root = used + 1, root - 1
        while avbl > used:
            A[nxt], nxt, avbl = depth, nxt - 1, avbl - 1
        avbl, depth, used = 2 * used, depth + 1, 0
    unlimited = max(A)
    count = [0] * (max(unlimited, maxbits) + 1)
    for d in A:
        count[min(d, maxbits)] += 1
    total = sum(count[i] << (maxbits - i) for i in range(1, maxbits + 1))
    while total != 1 << maxbits:
        count[maxbits] -= 1
        for i in range(maxbits - 1, 0, -1):
            if count[i]:
                count[i] -= 1
                count[i + 1] += 2
                break
        total -= 1
    lens, j = [0] * len(freq), m
    for length in range(1, maxbits + 1):
        for _ in range(count[length]):
            j -= 1
            lens[order[j]] = length
    return lens, unlimited, max(lens)


def canonical_codes(lens: list) -> list:
    """Each symbol's canonical code, bit-reversed for LSB-first packing (RFC 1951 section 3.2.2)."""
    bl = [0] * 16
    for length in lens:
        bl[length] += 1
    bl[0] = 0
    nxt, code = [0] * 16, 0
    for b in range(1, 16):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    out = []
    for length in lens:
        c = 0
        if length:
            c = int(format(nxt[length], f"0{length}b")[::-1], 2)
            nxt[length] += 1
        out.append(c)
    return out


def _fixed_lens() -> list:
    return [8] * 144 + [9] * 112 + [7] * 24 + [8] * 6


def _fixed_codes() -> list:
    """The fixed literal/length codes: canonical over all 288 symbols of RFC 1951 section 3.2.6 (286 and 287 take part
    in the code though no block uses them)."""
    return canonical_codes(_fixed_lens() + [8, 8])[:LIT_SYMS]


def run_length(seq: list) -> list:
    """The code-length sequence as (symbol, extra value) pairs: 16 repeats the previous length 3..6 times, 17 and 18
    are runs of 3..10 and 11..138 zeros."""
    out, i = [], 0
    while i < len(seq):
        v, run = seq[i], 1
        while i + run < len(seq) and seq[i + run] == v:
            run += 1
        i += run
        if v == 0:
            while run >= 11:
                r = min(run, 138)
                out.append((18, r - 11))
                run -= r
            if run >= 3:
                out.append((17, run - 3))
                run = 0
            out += [(0, 0)] * run
        else:
            out.append((v, 0))
            run -= 1
            while run >= 3:
                r = min(run, 6)
                out.append((16, r - 3))
                run -= r
            out += [(v, 0)] * run
    return out


_CL_EXTRA = {16: 2, 17: 3, 18: 7}


@dataclasses.dataclass
class SegmentReport:
    """The paths one segment took through the encoder."""
    n: int                      # filtered bytes
    kind: str                   # "stored", "fixed" or "dynamic"
    tie: str | None             # "fixed=dynamic" or "stored=huffman" when a tie rule decided the kind, else None
    huff_bits: int | None       # the rendered Huffman block (None: larger than the stored bound, never rendered)
    stored_bits: int            # the stored block at the offset the segment starts at
    fixed_bits: int
    dynamic_bits: int
    lit_depth: tuple            # (deepest leaf before the 15-bit limit, after) of the literal/length tree
    dist_depth: tuple           # ... of the distance tree
    cl_depth: tuple             # ... of the code-length tree, limit 7
    symbols: int                # symbols in the parse, end of block excluded (the doubling walk takes that many steps)
    literals: int
    longest: int                # longest match of the parse (0: none)
    farthest: int               # largest distance of the parse
    into_previous: bool         # a match reaches into the previous segment
    clipped: bool               # a match stops at the segment's end though the next segment's bytes continue it


def _segment_symbols(stream: np.ndarray, start: int, n_seg: int, row_dist: int) -> tuple:
    """(match length per position (0: a literal), its distance) of one segment: the longest of the
    five candidates 1, 3, the nearest same-hash position up to 256 back in the position's 1024-position round, the row
    above (3W + 1) and the latest same-hash position before the round, ties to the earlier candidate."""
    ws = max(0, start - WINDOW)
    n_win = start - ws
    buf = stream[ws:start + n_seg]
    n_buf = buf.size
    pad = np.concatenate([buf, np.zeros(16, np.uint8)])
    words = np.zeros(n_buf + 8, np.uint64)
    for b in range(8):
        words |= pad[b:b + n_buf + 8].astype(np.uint64) << np.uint64(8 * b)
    p = np.arange(n_seg)
    at = n_win + p
    maxlen = np.minimum(MAX_MATCH, n_seg - p)
    nh = max(n_buf - 2, 0)                       # positions with 3 bytes: all of them hashed
    hh = hash3(buf, np.arange(nh)).astype(np.int64) if nh else np.zeros(0, np.int64)
    seek = maxlen >= 3                           # (every such position is hashed)
    ps = p[seek]
    h = hh[at[seek]]
    rnd = ps // ROUND
    # nearest earlier position of the same hash in the round, at most NEAR_SCAN back
    near = np.zeros(n_seg, np.int64)
    hashed = p[at < nh]
    hr, hh_r = hashed // ROUND, hh[n_win + hashed]
    o = np.lexsort((hashed, hh_r, hr))
    srt = hashed[o]
    if srt.size > 1:
        d = srt[1:] - srt[:-1]
        ok = (hr[o][1:] == hr[o][:-1]) & (hh_r[o][1:] == hh_r[o][:-1]) & (d <= NEAR_SCAN)
        near[srt[1:][ok]] = d[ok]
    # latest position of the same hash before the round (the window and the earlier rounds)
    keys = np.sort(hh * (1 << 20) + np.arange(nh))
    q = np.searchsorted(keys, h * (1 << 20) + n_win + rnd * ROUND - 1, side="right") - 1
    hit = (q >= 0) & ((keys[np.maximum(q, 0)] >> 20) == h)
    latest = np.where(hit, at[seek] - (keys[np.maximum(q, 0)] & ((1 << 20) - 1)), 0)
    best = np.zeros(ps.size, np.int64)
    bd = np.zeros(ps.size, np.int64)
    a, ml = at[seek], maxlen[seek]
    for cand in (np.full(ps.size, 1), np.full(ps.size, 3), near[seek], np.full(ps.size, row_dist), latest):
        ok = (cand != 0) & (cand <= WINDOW) & (cand <= a)
        m = np.zeros(ps.size, np.int64)
        m[ok] = _match_lengths(words, a[ok], cand[ok], ml[ok])
        m[m < min_match(cand)] = 0
        better = m > best
        best[better], bd[better] = m[better], cand[better]
    length, dist = np.zeros(n_seg, np.int64), np.zeros(n_seg, np.int64)
    length[seek], dist[seek] = best, bd
    return length, dist


def _encode_segment(stream: np.ndarray, s: int, row_dist: int) -> dict:
    """One segment's parse, codes, costs and Huffman symbols (value, bit count), its block kind still open."""
    start = s * SEGMENT
    n_seg = min(SEGMENT, stream.size - start)
    length, dist = _segment_symbols(stream, start, n_seg, row_dist)
    # the greedy parse: next = p + max(1, len)
    lens_l, steps, p = length.tolist(), [], 0
    while p < n_seg:
        steps.append(p)
        p += max(1, lens_l[p])
    steps = np.array(steps, np.int64)
    L, D = length[steps], dist[steps]
    lit = L == 0
    lsym = np.where(lit, stream[start + steps], _LEN_SYM[L])
    dsym = _DIST_SYM[D[~lit]]
    extra = int(_LEN_EB[L[~lit]].sum() + _DIST_EB[D[~lit]].sum())
    lit_freq = np.bincount(lsym, minlength=LIT_SYMS).tolist()
    lit_freq[256] += 1                           # end of block
    dist_freq = np.bincount(dsym, minlength=DIST_SYMS).tolist()
    lit_len, *lit_depth = huffman_lengths(_two_used(lit_freq), 15)
    dist_len, *dist_depth = huffman_lengths(_two_used(dist_freq), 15)
    hlit, hdist = LIT_SYMS, DIST_SYMS
    while hlit > 257 and lit_len[hlit - 1] == 0:
        hlit -= 1
    while hdist > 1 and dist_len[hdist - 1] == 0:
        hdist -= 1
    rle = run_length(lit_len[:hlit] + dist_len[:hdist])
    cl_freq = [0] * CL_SYMS
    for sym, _ in rle:
        cl_freq[sym] += 1
    cl_len, *cl_depth = huffman_lengths(_two_used(cl_freq), 7)
    hclen = CL_SYMS
    while hclen > 4 and cl_len[CL_ORDER[hclen - 1]] == 0:
        hclen -= 1
    header = 3 + 5 + 5 + 4 + 3 * hclen + sum(cl_len[sym] + _CL_EXTRA.get(sym, 0) for sym, _ in rle)
    fixed_lens = _fixed_lens()
    dyn = header + extra + sum(f * n for f, n in zip(lit_freq, lit_len)) + sum(f * n for f, n in zip(dist_freq, dist_len))
    fix = 3 + extra + sum(f * n for f, n in zip(lit_freq, fixed_lens)) + 5 * sum(dist_freq)
    use_fixed = fix <= dyn                       # ties: the fixed block
    huff = fix if use_fixed else dyn
    # the Huffman symbols after the 3-bit block header: the header of a dynamic block, the data, end of block
    if use_fixed:
        lcode, lbits = _fixed_codes(), fixed_lens
        dcode, dbits = canonical_codes([5] * DIST_SYMS), [5] * DIST_SYMS
        head_v, head_n = [], []
    else:
        lcode, lbits, dcode, dbits = canonical_codes(lit_len), lit_len, canonical_codes(dist_len), dist_len
        ccode = canonical_codes(cl_len)
        head_v = [hlit - 257, hdist - 1, hclen - 4] + [cl_len[CL_ORDER[i]] for i in range(hclen)]
        head_n = [5, 5, 4] + [3] * hclen
        for sym, ev in rle:
            head_v += [ccode[sym], ev]
            head_n += [cl_len[sym], _CL_EXTRA.get(sym, 0)]
    lcode, lbits, dcode, dbits = (np.array(x, np.uint64) for x in (lcode, lbits, dcode, dbits))
    v, nb = lcode[lsym], lbits[lsym]
    m = ~lit
    for add_v, add_n in ((_LEN_EV[L[m]], _LEN_EB[L[m]]), (dcode[dsym], dbits[dsym]),
                         (_DIST_EV[D[m]], _DIST_EB[D[m]])):
        v[m] |= add_v.astype(np.uint64) << nb[m]
        nb[m] += add_n.astype(np.uint64)
    vals = np.concatenate([np.array(head_v, np.uint64), v, np.array([lcode[256]], np.uint64)])
    nbits = np.concatenate([np.array(head_n, np.uint64), nb, np.array([lbits[256]], np.uint64)])
    assert int(nbits.sum()) + 3 == huff
    # a match that stops at the segment's end while the stream after it still matches
    last = steps[-1]
    end = start + n_seg
    clipped = bool(length[last] and length[last] == n_seg - last < MAX_MATCH and end < stream.size and
                   stream[end] == stream[end - dist[last]])
    report = SegmentReport(
        n=n_seg, kind="", tie=None, huff_bits=huff if huff <= 42 + 8 * n_seg else None, stored_bits=0,
        fixed_bits=fix, dynamic_bits=dyn, lit_depth=tuple(lit_depth), dist_depth=tuple(dist_depth),
        cl_depth=tuple(cl_depth), symbols=int(steps.size), literals=int(lit.sum()),
        longest=int(L.max(initial=0)), farthest=int(D.max(initial=0)),
        into_previous=bool(np.any(~lit & (steps - D < 0))), clipped=clipped)
    if fix == dyn:
        report.tie = "fixed=dynamic"
    return dict(report=report, btype=1 if use_fixed else 2, vals=vals, nbits=nbits,
                adler=zlib.adler32(stream[start:end].tobytes()))


def _pack(vals: np.ndarray, nbits: np.ndarray) -> bytes:
    """The symbols' bits, LSB first, one after another (each value holds at most 57 bits)."""
    off = np.concatenate([[0], np.cumsum(nbits.astype(np.int64))[:-1]]).astype(np.int64)
    total = int(nbits.sum())
    words = np.zeros(total // 64 + 2, np.uint64)
    wi, sh = off >> 6, (off & 63).astype(np.uint64)
    np.bitwise_or.at(words, wi, vals << sh)
    spill = sh + nbits > 64
    np.bitwise_or.at(words, wi[spill] + 1, vals[spill] >> (np.uint64(64) - sh[spill]))
    return words.astype("<u8").tobytes()[:(total + 7) // 8]


def _chunk(typ: bytes, body: bytes) -> bytes:
    return struct.pack(">I", len(body)) + typ + body + struct.pack(">I", zlib.crc32(typ + body) & 0xFFFFFFFF)


def encode_png(rgb: np.ndarray, report: bool = False):
    """The file png.cu writes for an (H, W, 3) uint8 image; with report=True, (file, per-segment SegmentReport list)."""
    H, W, _ = rgb.shape
    _, stream = filter_image(rgb)
    n = stream.size
    segs = [_encode_segment(stream, s, 3 * W + 1) for s in range(segments(W, H))]
    vals, nbits, off, adler = [], [], 0, 1
    for s, g in enumerate(segs):
        r, final = g["report"], s == len(segs) - 1
        pad = (8 - ((off + 3) & 7)) & 7
        r.stored_bits = 3 + pad + 32 + 8 * r.n
        stored = r.huff_bits is None or r.stored_bits <= r.huff_bits    # ties: the stored block
        if r.huff_bits is not None and r.stored_bits == r.huff_bits:
            r.tie = "stored=huffman"
        if stored:
            r.kind = "stored"
            data = stream[s * SEGMENT:s * SEGMENT + r.n].astype(np.uint64)
            vals.append(np.concatenate([np.array([int(final), 0, r.n, r.n ^ 0xFFFF], np.uint64), data]))
            nbits.append(np.concatenate([np.array([3, pad, 16, 16], np.uint64), np.full(r.n, 8, np.uint64)]))
            off += r.stored_bits
        else:
            r.kind = "fixed" if g["btype"] == 1 else "dynamic"
            vals.append(np.concatenate([np.array([int(final) | g["btype"] << 1], np.uint64), g["vals"]]))
            nbits.append(np.concatenate([np.array([3], np.uint64), g["nbits"]]))
            off += r.huff_bits
        adler = zlib.adler32(stream[s * SEGMENT:s * SEGMENT + r.n].tobytes(), adler)
    deflate = _pack(np.concatenate(vals), np.concatenate(nbits))
    assert len(deflate) == (off + 7) // 8
    idat = b"\x78\x01" + deflate + struct.pack(">I", adler)
    data = (b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, 2, 0, 0, 0)) +
            _chunk(b"IDAT", idat) + _chunk(b"IEND", b""))
    return (data, [g["report"] for g in segs]) if report else data
