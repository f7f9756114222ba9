"""CPU: tests/h264_deblock_oracle.py -- the restatement of the deblocked device H.264 stream -- refereed by OpenCV's
bundled FFmpeg, which applies the in-loop filter as a conforming decoder: every picture's luma equals the oracle's
filtered luma byte for byte at QPs across the tables, over a GOP of 40 P pictures and after a seek; the decoded colour
holds to the filtered chroma within a bound the unfiltered chroma fails; below qp 16 the filter changes nothing; intra
prediction reads the samples before the filter; and the corpus reaches every path of 8.7."""
from collections import Counter

import numpy as np
import pytest

from oracle import h264 as O
from tests import h264_corpus as hc
from tests import h264_deblock_corpus as dc
from tests import h264_deblock_oracle as D
from tests import h264_inter_corpus as ic
from tests import h264_stream_oracle as S


def _write(tmp_path, out, W, H, qp, gop, name="d.mp4"):
    path = tmp_path / name
    path.write_bytes(D.mp4([f["sample"] for f in out], W, H, qp, gop=gop))
    return path


def _luma(path, K, W, H, cv2, seek=None):
    cap = cv2.VideoCapture(str(path))
    assert cap.isOpened() and int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == K
    cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
    if seek is not None:
        cap.set(cv2.CAP_PROP_POS_FRAMES, seek)
    got = []
    for _ in range(K if seek is None else 1):
        ok, y = cap.read()
        assert ok
        got.append(y.reshape(H, W))
    return got


@pytest.mark.parametrize("item", dc.sequences(large=False), ids=lambda it: it[0])
def test_ffmpeg_decodes_the_filtered_pictures(item, tmp_path):
    cv2 = pytest.importorskip("cv2")
    name, frames, qp, gop = item
    K, H, W, _ = frames.shape
    for q in (qp, min(qp + 12, 51)):
        out = D.encode_stream(frames, q, gop)
        got = _luma(_write(tmp_path, out, W, H, q, gop), K, W, H, cv2)
        for k in range(K):
            assert np.array_equal(got[k], D.crop(out[k]["filtered"], W, H)[0]), f"{name} qp {q} frame {k}"


@pytest.mark.parametrize("qp", dc.QPS)
def test_every_table_qp_decodes_to_the_filtered_luma(qp, tmp_path):
    cv2 = pytest.importorskip("cv2")
    frames = np.concatenate([ic.avatar_motion(64, 48, 4), ic.grainy(64, 48, 3, amp=12)])
    for gop in (1, 4):
        out = D.encode_stream(frames, qp, gop)
        got = _luma(_write(tmp_path, out, 64, 48, qp, gop), len(frames), 64, 48, cv2)
        for k, y in enumerate(got):
            assert np.array_equal(y, D.crop(out[k]["filtered"], 64, 48)[0]), f"qp {qp} gop {gop} frame {k}"


def test_long_gop_reads_the_filtered_reference_and_seeks(tmp_path):
    cv2 = pytest.importorskip("cv2")
    W, H, K, gop = 96, 128, 44, 41
    base = hc.avatar_like(W, H)
    frames = np.stack([ic.shifted(base, (k % 7) - 3, (k % 5) - 2) for k in range(K)])
    out = D.encode_stream(frames, 30, gop)
    path = _write(tmp_path, out, W, H, 30, gop)
    for k, y in enumerate(_luma(path, K, W, H, cv2)):
        assert np.array_equal(y, D.crop(out[k]["filtered"], W, H)[0]), f"frame {k}"
    assert np.array_equal(_luma(path, K, W, H, cv2, seek=30)[0], D.crop(out[30]["filtered"], W, H)[0])
    # the filter changed the references the P pictures predicted from
    assert sum(not np.array_equal(f["recon"][0], f["filtered"][0]) for f in out[:gop]) >= gop // 2


def _bgr(y, cb, cr):
    """BT.601 limited range -> BGR in floating point, chroma repeated over each 2x2 block."""
    y = 1.164 * (y.astype(np.float64) - 16)
    cb, cr = (np.repeat(np.repeat(c, 2, 0), 2, 1).astype(np.float64) - 128 for c in (cb, cr))
    return np.stack([y + 2.018 * cb, y - 0.813 * cr - 0.391 * cb, y + 1.596 * cr], -1).clip(0, 255)


def test_decoded_colour_holds_to_the_filtered_chroma(tmp_path):
    cv2 = pytest.importorskip("cv2")
    W, H = 96, 64
    frames = ic.avatar_motion(W, H, 6)
    for qp in (26, 38, 45):
        out = D.encode_stream(frames, qp, 3)
        cap = cv2.VideoCapture(str(_write(tmp_path, out, W, H, qp, 3)))
        for k in range(len(frames)):
            ok, bgr = cap.read()
            assert ok
            fy, fcb, fcr = D.crop(out[k]["filtered"], W, H)
            _, ucb, ucr = D.crop(out[k]["recon"], W, H)
            # FFmpeg's conversion and upsampling differ from _bgr by under 3 levels; with the chroma before the
            # filter the worst sample is off by more
            assert np.abs(bgr - _bgr(fy, fcb, fcr)).max() <= 3, (qp, k)
            assert np.abs(bgr - _bgr(fy, ucb, ucr)).max() > 3, (qp, k)


@pytest.mark.parametrize("qp", [0, 8, 15])
def test_below_qp_16_the_filter_changes_nothing(qp):
    pairs = []
    for frames in (ic.pan(80, 64)[:4], dc.pcm_beside_intra()):
        pairs += zip(S.encode_stream(frames, qp, 3), D.encode_stream(frames, qp, 3))
    for a, b in pairs:
        assert all(np.array_equal(x, y) for x, y in zip(a["recon"], b["filtered"]))
        assert all(np.array_equal(x, y) for x, y in zip(a["recon"], b["recon"]))
        s, t = a["sample"], b["sample"]
        assert len(s) == len(t)
        # only the slice header's three filter bits: 010 -> 111
        diff = [i for i in range(len(s)) if s[i] != t[i]]
        assert diff == ([7] if s[4] == 0x65 else [6, 7])
        assert bin(int.from_bytes(s[5:8], "big") ^ int.from_bytes(t[5:8], "big")).count("1") == 2


def test_intra_prediction_reads_the_samples_before_the_filter(tmp_path):
    cv2 = pytest.importorskip("cv2")
    W, H, qp = 32, 16, 30
    img = hc.avatar_like(64, 64)[24:40, 16:48].copy()
    img[:, :16] = np.clip(img[:, :16].astype(int) + 40, 0, 255)     # a step at the macroblock edge
    out = D.encode_stream(img[None], qp, 1)
    f = out[0]
    assert (f["types"] == "I").all()
    rec, flt = f["recon"][0].astype(np.int64), f["filtered"][0].astype(np.int64)
    left_u, left_f = rec[:, 15], flt[:, 15]
    assert not np.array_equal(left_u, left_f)             # the filter moved the column macroblock 1 predicts from
    # macroblock 1 predicts from its left neighbour's last column in the mode the encode chose; the same residual on
    # a prediction from the filtered column gives other samples, so a decoder that predicted from filtered samples
    # would not output the oracle's picture
    mode = int(O.encode_frame(img, qp)["modes"][0][0, 1])
    pred = [O.predict(np.zeros((1, 16), np.int64), c[None], np.zeros(1, np.int64), np.array([False]),
                      np.array([True]), 16, False)[0, mode] for c in (left_u, left_f)]
    mb = rec[:, 16:32]
    assert not np.array_equal(np.clip(mb - pred[0] + pred[1], 0, 255), mb)
    got = _luma(_write(tmp_path, out, W, H, qp, 1), 1, W, H, cv2)[0]
    assert np.array_equal(got, D.crop(f["filtered"], W, H)[0])


def test_corpus_reaches_every_filter_path():
    paths = Counter()
    for name, frames, qp, gop in dc.sequences(large=False):
        for q in (qp, min(qp + 12, 51)):
            for f in D.encode_stream(frames, q, gop):
                paths += f["paths"]
    want = {(k, "bS", v) for k in ("luma", "chroma") for v in range(5)}
    want |= {(k, w) for k in ("luma", "chroma") for w in ("alpha_off", "beta_off", "weak")}
    want |= {(k, "tc_clip", s) for k in ("luma", "chroma") for s in "+-"}
    want |= {("luma", w) for w in ("strong", "bs4_weak", "ap_only", "aq_only")} | {("chroma", "bs4")}
    want |= {("mv_diff", a, v) for a in "xy" for v in (3, 4)}
    want |= {("pcm_edge",), ("intra_in_p",), ("border", "left"), ("border", "top")}
    assert want <= set(k for k, v in paths.items() if v), sorted(map(str, want - set(paths)))


def test_tables_have_the_standard_shape():
    assert D.ALPHA[:16] == [0] * 16 == D.BETA[:16] and D.ALPHA[16] == 4 and D.ALPHA[51] == 255 and D.BETA[51] == 18
    assert all(a <= b for a, b in zip(D.ALPHA, D.ALPHA[1:])) and all(a <= b for a, b in zip(D.BETA, D.BETA[1:]))
    for col in range(3):
        c = [t[col] for t in D.TC0]
        assert all(a <= b for a, b in zip(c, c[1:]))
    assert all(t[0] <= t[1] <= t[2] for t in D.TC0) and D.TC0[51] == (13, 17, 25)
