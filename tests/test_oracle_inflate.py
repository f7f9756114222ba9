"""CPU: oracle/inflate.py against zlib and PIL over the PNG decoder's corpus (tests/png_corpus.py).  The oracle
inflates every valid stream to zlib's bytes and refuses exactly the streams zlib refuses; its unfilter gives PIL's
pixels; each crafted refusal fails in the one way it was built for; and the union of the oracle's path reports reaches
every path the corpus is meant to reach."""
import zlib

import numpy as np
import pytest

from gaussianavatars_b200.png import parse_png
from oracle import inflate as oi
from tests import png_corpus as pc

# the paths the corpus must reach (DESIGN.md 4.6, the corpus table)
PATHS = {"stored_empty", "stored_65535", "stored_after_huffman_unaligned", "fixed", "fixed_empty", "blocks_many",
         "length_258_code_285", "length_258_code_284_31", "distance_32768", "overlap_d1", "overlap_d3", "overlap_d4",
         "single_distance_code", "no_distance_codes", "rep16_min", "rep16_max", "rep17_min", "rep17_max",
         "rep18_min", "rep18_max", "repeat_crosses_into_distances", "lit_sub_table_15", "dist_sub_table_15",
         "hlit_286", "hdist_30", "hclen_4", "hclen_19", "filter_0", "filter_1", "filter_2", "filter_3", "filter_4",
         *{f"wbits_{w}" for w in range(9, 16)}}

CRAFTED = pc.crafted_streams()
ERRORS = pc.error_streams()
SWEEP_DATA = pc.filter_rows(pc.images()["gradient_4"], [0, 1, 2, 3, 4]) + bytes(range(256)) * 8


def _zlib(data):
    try:
        return zlib.decompress(data)
    except zlib.error:
        return None


@pytest.mark.parametrize("i", range(len(CRAFTED)), ids=[c[0] for c in CRAFTED])
def test_crafted_streams_equal_zlib(i):
    name, stream, data = CRAFTED[i]
    out, status, _ = oi.inflate(stream)
    assert status == oi.OK and out == data == zlib.decompress(stream)


def test_zlib_sweep_equals_zlib():
    for name, stream in pc.zlib_sweep(SWEEP_DATA):
        out, status, _ = oi.inflate(stream)
        assert status == oi.OK and out == SWEEP_DATA, name


@pytest.mark.parametrize("i", range(len(ERRORS)), ids=[e[0] for e in ERRORS])
def test_each_refusal_fails_its_one_way(i):
    name, idat, W, H, color, want = ERRORS[i]
    assert oi.decode_idat(idat, W, H, color)[1] == want
    # a zlib-level refusal is zlib's too; the size and filter refusals are the PNG's, and zlib takes the stream
    out, status, _ = oi.inflate(idat)
    z = _zlib(idat)
    if want in (oi.TOO_MUCH, oi.TOO_LITTLE, oi.FILTER):
        assert status == oi.OK and out == z
    else:
        assert status == want and z is None


def test_mutations_refused_exactly_as_zlib_refuses():
    muts = pc.mutations(pc.mutation_bases())
    assert len(muts) == 300
    refused = 0
    for name, idat, W, H, color in muts:
        out, status, _ = oi.inflate(idat)
        z = _zlib(idat)
        assert (status == oi.OK) == (z is not None), (name, oi.STATUS[status])
        if z is not None:
            assert out == z, name
        refused += status != oi.OK
    assert refused > 150   # most flips and cuts break the stream


def test_unfilter_equals_pil():
    files = pc.valid_files()
    assert len(files) == 288
    for name, data, img in files:
        W, H, color, idat = parse_png(data, name)
        rgba, status, _ = oi.decode_idat(idat, W, H, color)
        assert status == oi.OK, (name, oi.STATUS[status])
        want = pc.pil_pixels(data)
        assert np.array_equal(rgba, want), name
        assert np.array_equal(want[..., :img.shape[2]], img), name


def test_adler32_equals_zlib():
    rng = np.random.default_rng(1)
    for n in (0, 1, 5551, 5552, 5553, 100_000):
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        assert oi.adler32(data) == zlib.adler32(data)
    assert oi.adler32(b"\xff" * 200_000) == zlib.adler32(b"\xff" * 200_000)


def test_corpus_reaches_every_path():
    seen = set()
    for _, stream, _ in CRAFTED:
        seen |= oi.inflate(stream)[2]
    for _, stream in pc.zlib_sweep(SWEEP_DATA):
        seen |= oi.inflate(stream)[2]
    for _, idat, W, H, color, _ in ERRORS:
        seen |= oi.decode_idat(idat, W, H, color)[2]
    for name, data, _ in pc.valid_files():
        W, H, color, idat = parse_png(data, name)
        seen |= oi.decode_idat(idat, W, H, color)[2]
    assert PATHS - seen == set()
