"""CPU: the I_NxN H.264 oracle (tests/h264_intra4x4_oracle.py) refereed by OpenCV's bundled FFmpeg: the corpus
reaches every Intra_4x4 mode, neighbour and syntax path; the nine prediction formulas equal a direct restatement of
8.3.1.2; FFmpeg decodes the IDR-only, gop-25 and deblocked streams to the oracle's pictures byte for byte, and their
colour stays within the I_16x16 stream's PSNR floor."""
import numpy as np
import pytest

from tests import h264_corpus as hc
from tests import h264_intra4x4_corpus as c4
from tests import h264_intra4x4_oracle as I
from tests import h264_inter_corpus as ic
from tests.test_oracle_h264 import BGR_PSNR_FLOOR_DB, _decode

NEIGHBOURS = ("unavailable", "I_16x16", "I_NxN", "I_PCM", "P_L0_16x16", "P_Skip")


def _report():
    rep = set()
    for _, frames, qp, gop in c4.sequences(large=False):
        for q in (qp, min(qp + 12, 51)):
            for f in I.encode_stream(frames, q, gop):
                rep |= f["report"]
    return rep


def test_corpus_reaches_every_intra4x4_path():
    rep = _report()
    want = {("mb", "I_NxN"), ("i4_in_p",), ("i4_top_right_substituted",), ("i4_block5", "with_C"),
            ("i4_block5", "without_C"), ("prev_intra4x4_pred_mode_flag", 0), ("prev_intra4x4_pred_mode_flag", 1)}
    want |= {("i4_mode", m) for m in range(9)}
    want |= {("i4_mode_at", side, m) for side in ("top", "left", "right") for m in range(9)}
    want |= {("rem_intra4x4_pred_mode", r) for r in range(8)}
    want |= {("i4_neighbour", n) for n in NEIGHBOURS}
    want |= {("intra_cbp_luma", c) for c in range(16)} | {("intra_cbp_chroma", c) for c in range(3)}
    assert not want - rep, sorted(want - rep)


def _direct(p, mode, x, y):
    """8.3.1.2.1-9 as written, on p[(x, y)] with p[4..7, -1] already substituted."""
    if mode == 0:
        return p[x, -1]
    if mode == 1:
        return p[-1, y]
    if mode == 2:
        top, left = [p[i, -1] for i in range(4)], [p[-1, j] for j in range(4)]
        return (sum(top) + sum(left) + 4) >> 3
    if mode == 3:
        if x == 3 and y == 3:
            return (p[6, -1] + 3 * p[7, -1] + 2) >> 2
        return (p[x + y, -1] + 2 * p[x + y + 1, -1] + p[x + y + 2, -1] + 2) >> 2
    if mode == 4:
        if x > y:
            return (p[x - y - 2, -1] + 2 * p[x - y - 1, -1] + p[x - y, -1] + 2) >> 2
        if x < y:
            return (p[-1, y - x - 2] + 2 * p[-1, y - x - 1] + p[-1, y - x] + 2) >> 2
        return (p[0, -1] + 2 * p[-1, -1] + p[-1, 0] + 2) >> 2
    if mode == 5:
        z = 2 * x - y
        if z in (0, 2, 4, 6):
            return (p[x - (y >> 1) - 1, -1] + p[x - (y >> 1), -1] + 1) >> 1
        if z in (1, 3, 5):
            return (p[x - (y >> 1) - 2, -1] + 2 * p[x - (y >> 1) - 1, -1] + p[x - (y >> 1), -1] + 2) >> 2
        if z == -1:
            return (p[-1, 0] + 2 * p[-1, -1] + p[0, -1] + 2) >> 2
        return (p[-1, y - 1] + 2 * p[-1, y - 2] + p[-1, y - 3] + 2) >> 2
    if mode == 6:
        z = 2 * y - x
        if z in (0, 2, 4, 6):
            return (p[-1, y - (x >> 1) - 1] + p[-1, y - (x >> 1)] + 1) >> 1
        if z in (1, 3, 5):
            return (p[-1, y - (x >> 1) - 2] + 2 * p[-1, y - (x >> 1) - 1] + p[-1, y - (x >> 1)] + 2) >> 2
        if z == -1:
            return (p[-1, 0] + 2 * p[-1, -1] + p[0, -1] + 2) >> 2
        return (p[x - 1, -1] + 2 * p[x - 2, -1] + p[x - 3, -1] + 2) >> 2
    if mode == 7:
        if y in (0, 2):
            return (p[x + (y >> 1), -1] + p[x + (y >> 1) + 1, -1] + 1) >> 1
        return (p[x + (y >> 1), -1] + 2 * p[x + (y >> 1) + 1, -1] + p[x + (y >> 1) + 2, -1] + 2) >> 2
    z = x + 2 * y
    if z in (0, 2, 4):
        return (p[-1, y + (x >> 1)] + p[-1, y + (x >> 1) + 1] + 1) >> 1
    if z in (1, 3):
        return (p[-1, y + (x >> 1)] + 2 * p[-1, y + (x >> 1) + 1] + p[-1, y + (x >> 1) + 2] + 2) >> 2
    if z == 5:
        return (p[-1, 2] + 3 * p[-1, 3] + 2) >> 2
    return p[-1, 3]


def test_the_nine_predictions_equal_a_direct_restatement():
    rng = np.random.default_rng(0)
    for trial in range(200):
        e = rng.integers(0, 256, 13) if trial % 4 else rng.choice([0, 255], 13)
        p = {(-1, j): int(e[3 - j]) for j in range(4)}
        p[-1, -1] = int(e[4])
        p.update({(i, -1): int(e[5 + i]) for i in range(8)})
        got = I.predict4(e[None], np.array([True]), np.array([True]))[0]
        for m in range(9):
            want = [_direct(p, m, x, y) for y in range(4) for x in range(4)]
            assert list(got[m]) == want, (trial, I.MODE_NAMES[m])


def test_dc_without_neighbours_and_the_block5_rule():
    e = np.arange(13)[None] * 10
    t, f = np.array([True]), np.array([False])
    assert I.predict4(e, f, f)[0, 2, 0] == 128
    assert I.predict4(e, f, t)[0, 2, 0] == (e[0, 5:9].sum() + 2) >> 2
    assert I.predict4(e, t, f)[0, 2, 0] == (e[0, 0:4].sum() + 2) >> 2
    ok = I.available4(3, 0, t, t)[0]
    assert not ok[3] and not ok[7] and ok.sum() == 7
    assert I.available4(3, 1, t, t)[0].all()


def _check_decode(tmp_path, frames, qp, gop, deblock):
    K, H, W, _ = frames.shape
    out = I.encode_stream(frames, qp, gop, deblock=deblock)
    meta, ys = _decode(tmp_path, I.mp4([f["sample"] for f in out], W, H, qp, gop=gop))
    assert meta[0] == K and len(ys) == K
    for k, (y, f) in enumerate(zip(ys, out)):
        assert np.array_equal(y.reshape(H, W), I.crop(f["filtered"], W, H)[0]), (qp, gop, deblock, k)
    return out


@pytest.mark.parametrize("item", c4.sequences(large=False), ids=lambda it: it[0])
def test_ffmpeg_decodes_the_oracle_streams(item, tmp_path):
    name, frames, qp, gop = item
    for deblock in (False, True):
        _check_decode(tmp_path, frames, qp, gop, deblock)
        _check_decode(tmp_path, frames[:2], qp, 1, deblock)


def test_ffmpeg_decodes_a_gop25_avatar_stream(tmp_path):
    frames = ic.avatar_motion(96, 64, 27)
    for deblock in (False, True):
        out = _check_decode(tmp_path, frames, 26, 25, deblock)
        assert sum(int((f["types"] == "I4").sum()) for f in out) > 0


def test_decoded_colour_is_within_the_psnr_floor(tmp_path):
    for img in (hc.avatar_like(176, 144), hc.gradient(64, 48)):
        H, W, _ = img.shape
        for deblock in (False, True):
            out = I.encode_stream(img[None], 20, 1, deblock=deblock)
            _, frames = _decode(tmp_path, I.mp4([out[0]["sample"]], W, H, 20), rgb=True)
            mse = np.mean((frames[0][..., ::-1].astype(np.float64) - img) ** 2)
            assert 10 * np.log10(255.0 ** 2 / mse) >= BGR_PSNR_FLOOR_DB


def test_intra_cbp_table_is_a_permutation():
    assert sorted(I.INTRA_CBP_CODE) == list(range(48))
    assert I.INTRA_CBP_CODE[47] == 0 and I.INTRA_CBP_CODE[0] == 3
