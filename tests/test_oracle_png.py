"""CPU: oracle/png.py's encode_png, the byte-for-byte restatement of the device PNG encoder, on the corpus of
tests/test_gpu_png.py -- its files pass every check the device's files pass, its parse inflates to the filtered stream,
its path report agrees with the bytes -- and the union of its path reports over the corpus reaches every rare path of
the encoder, so an edit to the corpus cannot drop one unnoticed."""
import struct
import zlib

import numpy as np
import pytest

from oracle import png as opng
from tests.test_gpu_png import CORPUS, ORACLE_BYTES, _chunks, check_stream

SMALL = sorted(k for k, v in CORPUS.items() if opng.filtered_bytes(v.shape[1], v.shape[0]) <= ORACLE_BYTES)
_CACHE = {}


def _encode(name):
    if name not in _CACHE:
        _CACHE[name] = opng.encode_png(CORPUS[name], report=True)
    return _CACHE[name]


@pytest.mark.parametrize("name", SMALL)
def test_oracle_file_passes_the_device_checks(name):
    img = CORPUS[name]
    data, report = _encode(name)
    check_stream(data, img)   # CRCs, chunk order, IHDR, zlib to its end, the filtered stream, PIL's pixels, the bound
    idat = b"".join(b for t, b in _chunks(data) if t == b"IDAT")
    assert idat[:2] == b"\x78\x01" and (0x78 * 256 + 0x01) % 31 == 0
    n = opng.filtered_bytes(img.shape[1], img.shape[0])
    assert sum(r.n for r in report) == n and len(report) == opng.segments(img.shape[1], img.shape[0])
    # the report's block sizes add up to the deflate stream
    bits = sum(r.stored_bits if r.kind == "stored" else r.huff_bits for r in report)
    assert len(idat) == 2 + (bits + 7) // 8 + 4
    # the first block's header: BFINAL when it is the only block, BTYPE its kind
    assert idat[2] & 7 == int(len(report) == 1) | {"stored": 0, "fixed": 1, "dynamic": 2}[report[0].kind] << 1
    for r in report:
        assert r.kind in ("stored", "fixed", "dynamic")
        huff = min(r.fixed_bits, r.dynamic_bits)
        assert r.huff_bits == (huff if huff <= 42 + 8 * r.n else None)
        if r.kind == "stored":
            assert r.huff_bits is None or r.stored_bits <= r.huff_bits
        else:
            assert r.huff_bits < r.stored_bits and r.huff_bits == (r.fixed_bits if r.kind == "fixed" else r.dynamic_bits)
            assert r.kind == "fixed" or r.dynamic_bits < r.fixed_bits
        assert r.literals <= r.symbols <= r.n and r.lit_depth[1] <= 15 and r.dist_depth[1] <= 15 and r.cl_depth[1] <= 7


def test_oracle_is_deterministic_and_independent_of_the_report():
    img = CORPUS["mixed_97x401"]
    assert opng.encode_png(img) == opng.encode_png(img, report=True)[0] == _encode("mixed_97x401")[0]


def test_huffman_lengths_limit_by_hand():
    # counts 1, 1, 2, 4, ..., 2^15: a chain 16 deep; the limit folds it to a complete 15-bit code, longest to rarest
    freq = [1, 1] + [1 << k for k in range(1, 16)]
    lens, unlimited, limited = opng.huffman_lengths(freq, 15)
    assert unlimited == 16 and limited == 15
    assert sum(2.0 ** -n for n in lens) == 1.0
    assert all(lens[i] >= lens[i + 1] for i in range(1, len(lens) - 1))
    assert lens[0] == lens[1] == 15
    # two symbols: one bit each; RLE of a run of zeros and repeats
    assert opng.huffman_lengths([0, 5, 0, 9], 7)[0] == [0, 1, 0, 1]
    assert opng.run_length([0] * 140 + [3] * 8 + [0] * 4 + [5, 5]) == \
        [(18, 127), (0, 0), (0, 0), (3, 0), (16, 3), (3, 0), (17, 1), (5, 0), (5, 0)]


def test_fixed_codes_decode_with_zlib():
    # a fixed block of every byte value (8- and 9-bit codes) and end of block, written with the oracle's codes, inflates
    lens, codes = opng._fixed_lens(), opng._fixed_codes()
    assert [codes[s] for s in (0, 143, 144, 255, 256, 279, 280, 285)] == \
        [int(format(c, f"0{n}b")[::-1], 2) for c, n in ((0x30, 8), (0xBF, 8), (0x190, 9), (0x1FF, 9), (0, 7),
                                                         (0x17, 7), (0xC0, 8), (0xC5, 8))]
    vals = [3] + [codes[c] for c in range(256)] + [codes[256]]
    nbits = [3] + [lens[c] for c in range(256)] + [lens[256]]
    data = opng._pack(np.array(vals, np.uint64), np.array(nbits, np.uint64))
    assert zlib.decompress(data, -15) == bytes(range(256))


# ---- which rare paths the corpus reaches ---------------------------------------------------------------------------
def _huffman(r):
    return r.kind != "stored"


PATHS = {
    # the length limit of each tree, taken by a block that renders the limited code
    "literal/length tree deeper than 15 bits": lambda r: r.kind == "dynamic" and r.lit_depth[0] > 15,
    "code-length tree deeper than 7 bits": lambda r: r.kind == "dynamic" and r.cl_depth[0] > 7,
    # the pointer-doubling parse: 2^14 + 1 or more steps need all 15 rounds
    "parse of more than 16384 symbols": lambda r: _huffman(r) and r.symbols > 1 << 14,
    "all-literal Huffman segment of 32768 symbols": lambda r: _huffman(r) and r.literals == r.symbols == 32768,
    # the window and the segment's edges
    "match at distance 32768": lambda r: _huffman(r) and r.farthest == 32768,
    "match into the previous segment": lambda r: _huffman(r) and r.into_previous,
    "258-byte match": lambda r: _huffman(r) and r.longest == 258,
    "match clipped by the segment's end": lambda r: _huffman(r) and r.clipped,
    # the block choice
    "fixed block over dynamic": lambda r: r.kind == "fixed" and r.fixed_bits < r.dynamic_bits,
    "fixed block by the fixed=dynamic tie": lambda r: r.kind == "fixed" and r.tie == "fixed=dynamic",
    "stored block over a rendered Huffman block": lambda r: r.kind == "stored" and r.huff_bits is not None and
    r.stored_bits < r.huff_bits,
    "stored block by the stored=huffman tie": lambda r: r.kind == "stored" and r.tie == "stored=huffman",
    "dynamic block": lambda r: r.kind == "dynamic",
    "stored block": lambda r: r.kind == "stored" and r.huff_bits is None,
}
FILE_PATHS = {
    "IDAT type and data end on a 64 KiB piece": lambda n: n % opng.PIECE == 0,
    "IDAT type and data end 1 byte into a 64 KiB piece": lambda n: n % opng.PIECE == 1,
}


def reached() -> dict:
    """Path -> the corpus images that reach it, from the oracle's reports."""
    out = {p: [] for p in (*PATHS, *FILE_PATHS)}
    for name in SMALL:
        data, report = _encode(name)
        for path, hit in PATHS.items():
            if any(hit(r) for r in report):
                out[path].append(name)
        idat = struct.unpack(">I", data[33:37])[0]
        for path, hit in FILE_PATHS.items():
            if hit(4 + idat):
                out[path].append(name)
    return out


def test_the_corpus_reaches_every_rare_path():
    got = reached()
    missing = [p for p, names in got.items() if not names]
    for p, names in got.items():
        print(f"{p}: {', '.join(names) or '-'}")
    assert not missing, f"no corpus image reaches: {missing}"
    # an IDAT of more than 1024 pieces is too large for the oracle: the corpus holds one (noise, stored blocks, so
    # at least its filtered bytes), and tests/test_gpu_png.py counts the device file's pieces
    assert any(opng.filtered_bytes(v.shape[1], v.shape[0]) > 1024 * opng.PIECE for v in CORPUS.values())


@pytest.mark.parametrize("name", ["de_bruijn", "fibonacci"])
def test_built_rows_take_the_sub_filter(name):
    # built from the filtered bytes they should give: the rule must pick Sub for the row, or the stream is not those
    ids, stream = opng.filter_image(CORPUS[name])
    assert ids.tolist() == [1] and stream[0] == 1
