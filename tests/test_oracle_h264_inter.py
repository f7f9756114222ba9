"""CPU: tests/h264_stream_oracle.py -- the P-picture restatement of the device H.264 stream encode -- refereed by
OpenCV's bundled FFmpeg: its files decode with the frame count, size and rate they were written with, every frame's
luma equals the oracle's reconstruction byte for byte (P frames over a long GOP included, so nothing drifts), a seek
lands on the same bytes, and the corpus reaches the paths the P syntax has."""
import numpy as np
import pytest

from oracle import h264 as O
from tests import h264_corpus as hc
from tests import h264_inter_corpus as ic
from tests import h264_stream_oracle as S


def _decode(path, n, w, h, cv2):
    cap = cv2.VideoCapture(str(path))
    assert cap.isOpened()
    assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == n and cap.get(cv2.CAP_PROP_FPS) == 25
    assert int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)) == w and int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT)) == h
    return cap


@pytest.mark.parametrize("item", ic.sequences(large=False), ids=lambda it: it[0])
def test_ffmpeg_decodes_the_oracle_reconstruction(item, tmp_path):
    cv2 = pytest.importorskip("cv2")
    name, frames, qp, gop = item
    K, H, W, _ = frames.shape
    out = S.encode_stream(frames, qp, gop)
    path = tmp_path / "s.mp4"
    path.write_bytes(S.mp4([f["sample"] for f in out], W, H, qp, gop=gop))
    cap = _decode(path, K, W, H, cv2)
    cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
    for k in range(K):
        ok, y = cap.read()
        assert ok and np.array_equal(y.reshape(H, W), S.crop(out[k]["recon"], W, H)[0]), f"{name} frame {k}"
        if k % gop == 0:
            assert out[k]["sample"] == O.encode_frame(frames[k], qp)["sample"]


def test_long_gop_avatar_decodes_without_drift_and_seeks(tmp_path):
    cv2 = pytest.importorskip("cv2")
    W, H, K, gop = 96, 128, 48, 41
    base = hc.avatar_like(W, H)
    frames = np.stack([ic.shifted(base, (k % 7) - 3, (k % 5) - 2) for k in range(K)])
    out = S.encode_stream(frames, 20, gop)
    path = tmp_path / "long.mp4"
    path.write_bytes(S.mp4([f["sample"] for f in out], W, H, 20, gop=gop))
    cap = _decode(path, K, W, H, cv2)
    for k in range(K):
        ok, bgr = cap.read()
        assert ok
        psnr = 10 * np.log10(255 ** 2 / np.mean((bgr[..., ::-1].astype(np.float64) - frames[k]) ** 2))
        assert psnr > 30, (k, psnr)
    cap = _decode(path, K, W, H, cv2)
    cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
    for k in range(K):
        ok, y = cap.read()
        assert ok and np.array_equal(y.reshape(H, W), S.crop(out[k]["recon"], W, H)[0]), f"frame {k}"
    cap = _decode(path, K, W, H, cv2)
    cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
    cap.set(cv2.CAP_PROP_POS_FRAMES, 30)        # inside the first GOP: from the IDR at 0 through stss
    ok, y = cap.read()
    assert ok and np.array_equal(y.reshape(H, W), S.crop(out[30]["recon"], W, H)[0])


def test_identical_frames_are_all_skips():
    frames = np.stack([hc.flat(64, 48)] * 3)          # reconstructed exactly, so nothing is left to code
    out = S.encode_stream(frames, 20, 3)
    for f in out[1:]:
        assert (f["types"] == "P_Skip").all()
        b = O.Bits()
        S.p_slice_header(b, 1 if f is out[1] else 2)
        b.ue(12)                                  # the whole slice is one skip run
        assert f["sample"][4:] == b"\x61" + O.to_bytes(O.rbsp_trailing(b))


@pytest.mark.parametrize("dx,dy", [(1, 0), (0, -3), (-5, 2), (16, -16)])
def test_whole_sample_shifts_give_their_vectors(dx, dy):
    base = hc.textured(64, 64, seed=3)
    out = S.encode_stream(np.stack([base, ic.shifted(base, dx, dy)]), 14, 2)
    f = out[1]
    # content moved right by dx is predicted from dx samples left: the vector is (-4 dx, -4 dy) quarter samples
    # wherever that block lies inside the picture (elsewhere it is edge replication, which other vectors match too)
    my, mx = np.mgrid[0:4, 0:4]
    inside = (16 * mx - dx >= 0) & (16 * mx - dx <= 48) & (16 * my - dy >= 0) & (16 * my - dy <= 48)
    sel = inside & (f["types"] == "P")
    assert sel.sum() >= inside.sum() // 2
    assert (f["mvs"][sel] == (-4 * dx, -4 * dy)).all()


def test_corpus_reaches_every_p_path():
    rep = set()
    for name, frames, qp, gop in ic.sequences(large=False):
        for f in S.encode_stream(frames, qp, gop):
            rep |= f["report"]
    want = {("mb", m) for m in ("P_Skip", "P_L0_16x16", "I_16x16", "I_PCM")}
    want |= {("mb_skip_run", r) for r in ("0", "mid", "trailing", "all")}
    want |= {("mvd", v) for v in ("0", "1", "other")} | {("mvd_extreme",)} | {("luma_total", 16)}
    want |= {("mv_frac", v) for v in range(4)} | {("outside", s) for s in ("left", "right", "top", "bottom")}
    want |= {("frame_num", 15), ("emulation_prevention",)}
    assert want <= rep, sorted(map(str, want - rep))
    cbps = {k[1] for k in rep if k[0] == "inter_cbp"}
    assert len(cbps) >= 40, sorted(set(range(48)) - cbps)


def test_frame_num_wraps_and_idr_samples_are_encode_frame():
    frames = ic.drift(16, 16, [(1, 1)] * 19)
    out = S.encode_stream(frames, 20, 20)
    assert ("frame_num", 15) in out[15]["report"] and ("frame_num", 0) in out[16]["report"]
    assert out[16]["sample"][4] == 0x61 and out[16]["sample"][5] & 1 == 0 and out[16]["sample"][6] >> 5 == 0
    assert out[0]["sample"] == O.encode_frame(frames[0], 20)["sample"]
