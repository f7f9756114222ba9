"""GPU: the device H.264 encoder (gab200_h264_encode, VideoWriter, encode_video) against oracle/h264.py, byte for
byte: every corpus image at its QPs, batches of mixed frames, repeat runs, a CUDA graph replay, the MP4 file of a clip
longer than two batches, a GraphedRender playback loop, the refusals, and -- where OpenCV imports -- FFmpeg's decode
of the device files."""
import io

import numpy as np
import pytest
import torch

from oracle import h264 as O
from tests import h264_corpus as hc

pytestmark = pytest.mark.gpu


def device_samples(frames: torch.Tensor, qp: int) -> list:
    """The samples gab200_h264_encode writes for a CUDA (K,H,W,3) batch, as bytes (idr_pic_id 1 in each)."""
    from gaussianavatars_b200 import video as V
    K, H, W = V.check_frames(frames)
    frames = frames.view(K, H, W, 3)
    out = torch.zeros((K, V.slot_stride(W, H)), dtype=torch.uint8, device=frames.device)
    out_len = torch.empty(K, dtype=torch.int64, device=frames.device)
    V.launch_encode(frames, qp, V.scratch(K, H, W, frames.device), out, out_len)
    lens = out_len.tolist()
    host = out.cpu().numpy()
    return [host[k, :lens[k]].tobytes() for k in range(K)]


def _cuda(img):
    return torch.from_numpy(np.ascontiguousarray(img)).cuda()


@pytest.mark.parametrize("item", hc.corpus(), ids=lambda it: it[0])
def test_corpus_sample_equals_the_oracle(item):
    from gaussianavatars_b200 import video as V
    name, img, qp = item
    want = O.encode_frame(img, qp)["sample"]
    got = device_samples(_cuda(img)[None], qp)[0]
    assert len(got) <= V.video_bound(img.shape[1], img.shape[0])
    assert got == want, f"{name}: {len(got)} bytes against the oracle's {len(want)}"


def _mixed(K, w=64, h=48):
    imgs = [hc.gradient(w, h), hc.noise(w, h, seed=1), hc.stripes(w, h, True), hc.textured(w, h), hc.flat(w, h),
            hc.noise(w, h, seed=2, amp=30), hc.stripes(w, h, False)]
    return np.stack([imgs[k % len(imgs)] for k in range(K)])


@pytest.mark.parametrize("K", [1, 3, 16])
def test_batch_gives_each_frame_its_own_bytes(K):
    frames = _mixed(K)
    for qp in (0, 26):
        batch = device_samples(_cuda(frames), qp)
        for k in range(K):
            assert batch[k] == device_samples(_cuda(frames[k])[None], qp)[0], f"frame {k} of {K} at qp {qp}"
            if k < 7:
                assert batch[k] == O.encode_frame(frames[k], qp)["sample"]


def test_two_runs_are_bit_identical():
    frames = _cuda(np.stack([hc.avatar_like(550, 802), hc.textured(550, 802)]))
    assert device_samples(frames, 20) == device_samples(frames, 20)


def test_graph_replay_gives_the_eager_bytes():
    from gaussianavatars_b200 import video as V
    frames = _cuda(_mixed(4, 96, 64))
    K, H, W = V.check_frames(frames)
    eager = device_samples(frames, 24)
    src = frames.clone()
    scratch = V.scratch(K, H, W, frames.device)
    out = torch.zeros((K, V.slot_stride(W, H)), dtype=torch.uint8, device="cuda")
    out_len = torch.empty(K, dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        V.launch_encode(src, 24, scratch, out, out_len)   # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        V.launch_encode(src, 24, scratch, out, out_len)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    lens = out_len.tolist()
    assert [out[k, :lens[k]].cpu().numpy().tobytes() for k in range(K)] == eager
    src.copy_(torch.flip(frames, dims=(0,)))
    g.replay()
    lens = out_len.tolist()
    assert [out[k, :lens[k]].cpu().numpy().tobytes() for k in range(K)] == eager[::-1]


def test_video_writer_file_equals_encode_video_and_the_oracle(tmp_path):
    from fractions import Fraction

    from gaussianavatars_b200 import VideoWriter, encode_video
    clip = np.stack([hc.textured(48, 32, seed=s) if s % 3 else hc.noise(48, 32, seed=s) for s in range(37)])
    frames = _cuda(clip)
    path = tmp_path / "clip.mp4"
    with VideoWriter(str(path), 48, 32, fps=Fraction(30000, 1001), qp=18, batch=16) as vw:
        vw.add(frames[:5])
        for k in range(5, 37):
            vw.add(frames[k])
    data = path.read_bytes()
    assert data == encode_video(frames, fps=Fraction(30000, 1001), qp=18)
    want = O.mp4([O.encode_frame(f, 18)["sample"] for f in clip], 48, 32, 18, 30000, 1001)
    assert data == want


def test_graphed_render_playback_into_a_video_writer(tmp_path):
    from gaussianavatars_b200 import VideoWriter, encode_video
    from gaussianavatars_b200.graph import GraphedRender
    from tests.test_gpu_display import H_IMG, W_IMG, _flame_setup, _rig
    pc = _flame_setup(T=8)
    cams = _rig(W_IMG, H_IMG, n=8)
    player = GraphedRender(pc, W_IMG, H_IMG, torch.ones(3), outputs="u8", warm_cameras=cams, warm_timesteps=range(8))
    path = tmp_path / "renders.mp4"
    shown = []
    with VideoWriter(str(path), W_IMG, H_IMG, fps=25, qp=20, batch=4) as vw:
        for i in range(10):
            player.set_inputs(camera=cams[i % 8], timestep=i % 8)
            player.run()
            vw.add(player.display)
            shown.append(player.display.clone())
    assert path.read_bytes() == encode_video(torch.stack(shown), fps=25, qp=20)
    assert O.encode_frame(shown[3].cpu().numpy(), 20)["sample"] == device_samples(shown[3][None], 20)[0]


def test_bad_inputs_raise_before_any_launch(tmp_path):
    from gaussianavatars_b200 import VideoWriter, encode_video
    from gaussianavatars_b200 import _native as N
    good = torch.zeros((2, 32, 48, 3), dtype=torch.uint8, device="cuda")
    n0 = N.launch_count()
    bad = [(good.float(), "uint8"), (good.cpu(), "CUDA"), (good[..., :2], r"\(H, W, 3\)"),
           (torch.zeros((2, 32, 47, 3), dtype=torch.uint8, device="cuda"), "even"), (good[:, :, ::2], "contiguous"),
           (torch.zeros((1, 16, 8704, 3), dtype=torch.uint8, device="cuda"), "level 5.2")]
    for t, msg in bad:
        with pytest.raises(ValueError, match=msg):
            encode_video(t)
    with pytest.raises(ValueError, match="qp"):
        encode_video(good, qp=52)
    with pytest.raises(ValueError, match="fps"):
        encode_video(good, fps=2.5)
    vw = VideoWriter(io.BytesIO(), 48, 32)
    with pytest.raises(ValueError, match="48x32"):
        vw.add(torch.zeros((32, 50, 3), dtype=torch.uint8, device="cuda"))
    assert N.launch_count() == n0
    vw.close()
    with pytest.raises(ValueError, match="closed"):
        vw.add(good)


def test_device_files_decode_in_ffmpeg(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from gaussianavatars_b200 import VideoWriter
    clip = np.stack([hc.avatar_like(550, 802, seed=s) for s in range(5)])
    path = str(tmp_path / "avatar.mp4")
    with VideoWriter(path, 550, 802, fps=25, qp=20, batch=2) as vw:
        vw.add(_cuda(clip))
    cap = cv2.VideoCapture(path)
    assert cap.isOpened()
    assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == 5 and cap.get(cv2.CAP_PROP_FPS) == 25
    assert int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)) == 550 and int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT)) == 802
    cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
    for k in range(5):
        ok, y = cap.read()
        assert ok and np.array_equal(y.reshape(802, 550), O.encode_frame(clip[k], 20)["recon"][0]), f"frame {k}"
