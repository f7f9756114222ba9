"""CPU: oracle/h264.py, the restatement the device H.264 encoder is compared with, refereed by an independent decoder.
The corpus reaches every CAVLC path, mode, I_PCM and emulation prevention; OpenCV's bundled FFmpeg opens the oracle's
MP4 files with the frame count, size and rate they were written with, and its luma output (CAP_PROP_CONVERT_RGB=0)
equals the oracle's reconstruction byte for byte -- which the standard requires of any decoder when deblocking is
off; its BGR output is within a PSNR floor of the source; and the reconstruction equals a float64 restatement of the
inverse transforms."""
import numpy as np
import pytest

from oracle import h264 as O
from tests import h264_corpus as hc

WANTED = ({("coeff_token", t) for t in O.TOKEN_TABLE_NAMES} | {("level_prefix", p) for p in range(16)}
          | {("suffixLength", s) for s in range(7)} | {("total_zeros", "luma", t) for t in range(1, 16)}
          | {("total_zeros", "chromaDC", t) for t in range(1, 4)} | {("run_before", z) for z in range(1, 8)}
          | {("luma_mode", m) for m in range(4)} | {("chroma_mode", m) for m in range(4)}
          | {("mb", "I_PCM"), ("emulation_prevention",)})
BGR_PSNR_FLOOR_DB = 34.0    # at QP 20 on smooth content; a wrong colour matrix or chroma plane is far below it


def test_corpus_reaches_every_path():
    reached = set()
    for _, img, qp in hc.corpus(large=False):
        reached |= O.encode_frame(img, qp)["report"]
    assert not WANTED - reached, f"paths no corpus image reaches: {sorted(WANTED - reached, key=str)}"


def test_vlc_tables_are_prefix_free():
    def prefix_free(codes):
        words = [format(c, "0%db" % n) for c, n in codes if n]
        return len(set(words)) == len(words) and not any(a != b and b.startswith(a) for a in words for b in words)

    for t in range(4):
        assert prefix_free(zip(O.COEFF_TOKEN_CODE[t], O.COEFF_TOKEN_LEN[t])), t
    assert prefix_free(zip(O.CHROMA_DC_TOKEN_CODE, O.CHROMA_DC_TOKEN_LEN))
    for tc in range(15):
        assert len(O.TOTAL_ZEROS_LEN[tc]) == 16 - tc and prefix_free(zip(O.TOTAL_ZEROS_CODE[tc], O.TOTAL_ZEROS_LEN[tc]))
    for tc in range(3):
        assert prefix_free(zip(O.CHROMA_DC_TOTAL_ZEROS_CODE[tc], O.CHROMA_DC_TOTAL_ZEROS_LEN[tc]))
    for z in range(7):
        assert prefix_free(zip(O.RUN_BEFORE_CODE[z], O.RUN_BEFORE_LEN[z]))


def _decode(tmp_path, data, name="v.mp4", rgb=False):
    cv2 = pytest.importorskip("cv2")
    path = str(tmp_path / name)
    with open(path, "wb") as f:
        f.write(data)
    cap = cv2.VideoCapture(path)
    assert cap.isOpened()
    meta = (int(cap.get(cv2.CAP_PROP_FRAME_COUNT)), cap.get(cv2.CAP_PROP_FPS), int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)),
            int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT)))
    if not rgb:
        cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
    frames = []
    while True:
        ok, fr = cap.read()
        if not ok:
            break
        frames.append(fr)
    return meta, frames


@pytest.mark.parametrize("qp", hc.QPS)
def test_ffmpeg_decodes_the_oracle_streams_to_its_reconstruction(tmp_path, qp):
    for name, img in hc.small_images():
        H, W, _ = img.shape
        out = O.encode_frame(img, qp)
        other = O.encode_frame(img[::-1].copy(), qp)
        meta, ys = _decode(tmp_path, O.mp4([out["sample"], other["sample"], out["sample"]], W, H, qp))
        assert meta == (3, 25.0, W, H), name
        assert len(ys) == 3, name
        for y, want in zip(ys, (out, other, out)):
            assert np.array_equal(y.reshape(H, W), want["recon"][0]), f"{name} at qp {qp}"


@pytest.mark.parametrize("size", hc.LARGE_SIZES, ids=lambda s: "%dx%d" % s)
def test_ffmpeg_decodes_the_large_sizes(tmp_path, size):
    from fractions import Fraction
    W, H = size
    img = hc.avatar_like(W, H) if W < 1000 else hc.textured(W, H)
    out = O.encode_frame(img, 26)
    meta, ys = _decode(tmp_path, O.mp4([out["sample"]] * 2, W, H, 26, 30000, 1001))
    assert meta[0] == 2 and meta[2:] == (W, H) and abs(meta[1] - float(Fraction(30000, 1001))) < 1e-6
    assert all(np.array_equal(y.reshape(H, W), out["recon"][0]) for y in ys)


def test_an_i_pcm_frame_decodes_to_the_input_luma(tmp_path):
    img = hc.noise(48, 32, seed=7)
    out = O.encode_frame(img, 0)
    assert out["modes"][2].all(), "noise at QP 0 should make every macroblock I_PCM"
    _, ys = _decode(tmp_path, O.mp4([out["sample"]], 48, 32, 0))
    y, cb, cr = O.rgb_to_yuv(img)
    assert np.array_equal(ys[0].reshape(32, 48), y[:32, :48])
    assert np.array_equal(out["recon"][1], cb[:16, :24]) and np.array_equal(out["recon"][2], cr[:16, :24])


def test_decoded_colour_is_within_the_psnr_floor(tmp_path):
    for img in (hc.avatar_like(550, 802), hc.gradient(64, 48)):
        H, W, _ = img.shape
        _, frames = _decode(tmp_path, O.mp4([O.encode_frame(img, 20)["sample"]], W, H, 20), rgb=True)
        mse = np.mean((frames[0][..., ::-1].astype(np.float64) - img) ** 2)
        assert 10 * np.log10(255.0 ** 2 / mse) >= BGR_PSNR_FLOOR_DB


CI = np.array([[1, 1, 1, 1], [1, 0.5, -0.5, -1], [1, -1, -1, 1], [0.5, -1, 1, -0.5]])   # inverse core transform


def _idct_f64(d):
    """residual = floor((CI^T d CI + 32) / 64) in float64.  Exact when every >> 1 of 8.5.12.2 drops no bit, which holds
    for the dequantised coefficients below: at QP >= 24 each is a multiple of 16."""
    return np.floor((CI.T @ d.astype(np.float64) @ CI + 32) / 64)


@pytest.mark.parametrize("qp", [24, 30, 36, 45, 51])
def test_reconstruction_equals_a_float64_inverse_transform(qp):
    rng = np.random.default_rng(qp)
    M = 8
    dcl = rng.integers(-60, 61, (M, 4, 4))
    acl = rng.integers(-40, 41, (M, 4, 4, 4, 4)) * (rng.random((M, 4, 4, 4, 4)) < 0.4)
    acl[..., 0, 0] = 0
    got = O.recon_luma(dcl, acl, qp)
    ls00 = 16 * O.V[qp % 6, 0]
    hd = O.HD.astype(np.float64)
    f = hd @ dcl.astype(np.float64) @ hd
    dcy = f * ls00 * 2.0 ** (qp // 6 - 6) if qp >= 36 else np.floor((f * ls00 + 2.0 ** (5 - qp // 6)) / 2.0 ** (6 - qp // 6))
    for m in range(M):
        for by in range(4):
            for bx in range(4):
                d = acl[m, by, bx] * 16.0 * O.V[qp % 6][O.POS] * 2.0 ** (qp // 6 - 4)
                d[0, 0] = dcy[m, by, bx]
                assert np.array_equal(got[m, 4 * by:4 * by + 4, 4 * bx:4 * bx + 4], _idct_f64(d)), (m, by, bx)
    qpc = O.CHROMA_QP[qp]
    cdl = rng.integers(-60, 61, (M, 2, 2))
    cal = rng.integers(-40, 41, (M, 2, 2, 4, 4)) * (rng.random((M, 2, 2, 4, 4)) < 0.4)
    cal[..., 0, 0] = 0
    got = O.recon_chroma(cdl, cal, qpc)
    h2 = O.H2.astype(np.float64)
    dcc = np.floor(h2 @ cdl.astype(np.float64) @ h2 * 16 * O.V[qpc % 6, 0] * 2.0 ** (qpc // 6) / 32)
    for m in range(M):
        for by in range(2):
            for bx in range(2):
                d = cal[m, by, bx] * 16.0 * O.V[qpc % 6][O.POS] * 2.0 ** (qpc // 6 - 4)
                d[0, 0] = dcc[m, by, bx]
                assert np.array_equal(got[m, 4 * by:4 * by + 4, 4 * bx:4 * bx + 4], _idct_f64(d)), (m, by, bx)


def test_sizes_and_refusals():
    assert O.coded_size(550, 802) == (560, 816) and O.coded_size(1920, 1080) == (1920, 1088)
    assert O.level_idc(550, 802, 25) == 31 and O.level_idc(1920, 1080, 25) == 40
    assert O.bound(4096, 2304) > 0 and O.bound(4098, 2304) == -1 and O.bound(8688, 16) > 0 and O.bound(8704, 16) == -1
    for w, h in ((3, 2), (2, 3), (0, 2), (2, 0)):
        assert O.bound(w, h) == -1
        with pytest.raises(ValueError):
            O.encode_frame(np.zeros((max(h, 1), max(w, 1), 3), np.uint8), 20)
    with pytest.raises(ValueError):
        O.encode_frame(np.zeros((2, 2, 3), np.uint8), 52)
