"""GPU: the device H.264 stream encoder with P pictures (gab200_h264_encode_stream, VideoWriter(gop=),
encode_video(gop=)) against tests/h264_stream_oracle.py, byte for byte: every inter corpus sequence at several QPs
and GOPs, batch splits that cut a GOP, batch 1, two interleaved writers, a repeat run, a CUDA graph whose replays
continue the stream on the device, a GraphedRender playback loop decoded by FFmpeg, and IDR samples equal to
gab200_h264_encode's."""
import io

import numpy as np
import pytest
import torch

from oracle import h264 as O
from tests import h264_corpus as hc
from tests import h264_inter_corpus as ic
from tests import h264_stream_oracle as S

pytestmark = pytest.mark.gpu


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class Stream:
    """One stream's device state and buffers; encode(frames) returns the samples of the next frames."""

    def __init__(self, W, H, qp, gop, batch):
        from gaussianavatars_b200 import video as V
        self.V, self.qp, self.gop = V, qp, gop
        self.state = V.state_buffer(H, W, "cuda")
        self.scratch = V.scratch(batch, H, W, "cuda")
        self.out = torch.zeros((batch, V.slot_stride(W, H, gop)), dtype=torch.uint8, device="cuda")
        self.out_len = torch.empty(batch, dtype=torch.int64, device="cuda")

    def launch(self, frames):
        self.V.launch_encode_stream(frames, self.qp, self.gop, self.state, self.scratch, self.out, self.out_len)

    def read(self, K):
        lens = self.out_len[:K].tolist()
        host = self.out[:K].cpu().numpy()
        return [host[k, :lens[k]].tobytes() for k in range(K)]

    def encode(self, frames):
        self.launch(frames)
        return self.read(frames.shape[0])


def _device(frames, qp, gop, batch=None):
    K, H, W, _ = frames.shape
    batch = batch or K
    s = Stream(W, H, qp, gop, batch)
    got = []
    for i in range(0, K, batch):
        got += s.encode(_cuda(frames[i:i + batch]))
    return got


@pytest.mark.parametrize("item", ic.sequences(), ids=lambda it: it[0])
def test_sequence_samples_equal_the_oracle(item):
    name, frames, qp, gop = item
    for q, g in ((qp, gop), (min(qp + 12, 51), 2)):
        want = [f["sample"] for f in S.encode_stream(frames, q, g)]
        got = _device(frames, q, g)
        for k, (a, b) in enumerate(zip(got, want)):
            assert a == b, f"{name} qp {q} gop {g} frame {k}: {len(a)} bytes against the oracle's {len(b)}"


@pytest.mark.parametrize("batch", [1, 2, 3, 5])
def test_batch_splits_give_the_stream_bytes(batch):
    frames = ic.drift(64, 48, [(1, 0), (0, 1), (2, -1), (-1, 0), (0, 0), (3, 2), (1, 1)], seed=5)
    want = [f["sample"] for f in S.encode_stream(frames, 22, 3)]
    assert _device(frames, 22, 3, batch) == want


def test_idr_samples_equal_the_intra_encode():
    from tests.test_gpu_video import device_samples
    frames = ic.pan(80, 64)
    got = _device(frames, 20, 3)
    intra = device_samples(_cuda(frames), 20)
    for k in range(0, len(frames), 3):
        assert got[k] == intra[k]
    assert _device(frames, 20, 1) == intra            # gop 1 is the intra stream


def test_interleaved_writers_and_a_repeat_run(tmp_path):
    from gaussianavatars_b200 import VideoWriter
    a, b = ic.drift(48, 32, [(1, 0)] * 9, seed=2), ic.scene_cut(64, 48)
    files = []
    for run in range(2):
        pa, pb = tmp_path / f"a{run}.mp4", tmp_path / f"b{run}.mp4"
        with VideoWriter(str(pa), 48, 32, qp=20, batch=3, gop=4) as va, \
                VideoWriter(str(pb), 64, 48, qp=26, batch=2, gop=3) as vb:
            for k in range(10):
                va.add(_cuda(a[k]))
                if k < len(b):
                    vb.add(_cuda(b[k]))
        files.append((pa.read_bytes(), pb.read_bytes()))
    assert files[0] == files[1]
    assert files[0][0] == S.mp4([f["sample"] for f in S.encode_stream(a, 20, 4)], 48, 32, 20, gop=4)
    assert files[0][1] == S.mp4([f["sample"] for f in S.encode_stream(b, 26, 3)], 64, 48, 26, gop=3)


def test_graph_replays_continue_the_stream():
    frames = ic.drift(64, 48, [(1, 0), (0, 1)] * 6, seed=7)            # 13 frames
    K, gop, qp = 3, 5, 24
    want = [f["sample"] for f in S.encode_stream(frames[:12], qp, gop)]
    s = Stream(64, 48, qp, gop, K)
    src = _cuda(frames[:K]).clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        s.launch(src)                                                  # warm-up: the stream's first batch
    torch.cuda.current_stream().wait_stream(side)
    got = s.read(K)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        s.launch(src)
    for i in range(K, 12, K):
        src.copy_(_cuda(frames[i:i + K]))
        g.replay()
        got += s.read(K)
    assert got == want


def test_encode_video_gop_equals_the_oracle():
    from gaussianavatars_b200 import encode_video
    clip = ic.drift(48, 32, [(1, 1)] * 20, seed=3)
    assert encode_video(_cuda(clip), qp=20, gop=7) == \
        S.mp4([f["sample"] for f in S.encode_stream(clip, 20, 7)], 48, 32, 20, gop=7)
    assert encode_video(_cuda(clip), qp=20) == O.mp4([O.encode_frame(f, 20)["sample"] for f in clip], 48, 32, 20)


def test_graphed_render_playback_with_p_pictures(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from gaussianavatars_b200 import VideoWriter
    from gaussianavatars_b200.graph import GraphedRender
    from tests.test_gpu_display import H_IMG, W_IMG, _flame_setup, _rig
    pc = _flame_setup(T=8)
    cams = _rig(W_IMG, H_IMG, n=8)
    player = GraphedRender(pc, W_IMG, H_IMG, torch.ones(3), outputs="u8", warm_cameras=cams[:1],
                           warm_timesteps=range(8))
    path = tmp_path / "renders.mp4"
    shown = []
    with VideoWriter(str(path), W_IMG, H_IMG, fps=25, qp=20, batch=4, gop=25) as vw:
        for i in range(30):                                            # a fixed camera, the timestep advancing
            player.set_inputs(camera=cams[0], timestep=i % 8)
            player.run()
            vw.add(player.display)
            shown.append(player.display.cpu().numpy())
    out = S.encode_stream(np.stack(shown), 20, 25)
    assert path.read_bytes() == S.mp4([f["sample"] for f in out], W_IMG, H_IMG, 20, gop=25)
    cap = cv2.VideoCapture(str(path))
    assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == 30
    cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
    for k in range(30):
        ok, y = cap.read()
        assert ok and np.array_equal(y.reshape(H_IMG, W_IMG), S.crop(out[k]["recon"], W_IMG, H_IMG)[0]), k
