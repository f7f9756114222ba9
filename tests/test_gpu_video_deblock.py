"""GPU: the deblocked device H.264 stream (gab200_h264_encode_deblocked, VideoWriter(deblock=True),
encode_video(deblock=True), export_trajectory(deblock=True)) against tests/h264_deblock_oracle.py, byte for byte: every
corpus sequence at two (QP, GOP) pairs and as an IDR-only stream, the state's picture against the oracle's filtered
picture, batch splits, two interleaved writers, CUDA graph replays that continue the stream, and a GraphedRender
playback loop and a trajectory export whose files FFmpeg decodes to the filtered pictures."""
import numpy as np
import pytest
import torch

from tests import h264_deblock_corpus as dc
from tests import h264_deblock_oracle as D
from tests import h264_inter_corpus as ic

pytestmark = pytest.mark.gpu


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class Stream:
    """One deblocked stream's device state and buffers; encode(frames) returns the samples of the next frames."""

    def __init__(self, W, H, qp, gop, batch, state=True):
        from gaussianavatars_b200 import video as V
        self.V, self.qp, self.gop, self.W, self.H = V, qp, gop, W, H
        self.state = V.state_buffer(H, W, "cuda") if state else None
        self.scratch = V.deblocked_scratch(batch, H, W, gop, "cuda")
        self.out = torch.zeros((batch, V.slot_stride(W, H, gop)), dtype=torch.uint8, device="cuda")
        self.out_len = torch.empty(batch, dtype=torch.int64, device="cuda")

    def launch(self, frames):
        self.V.launch_encode_deblocked(frames, self.qp, self.gop, self.state, self.scratch, self.out, self.out_len)

    def read(self, K):
        lens = self.out_len[:K].tolist()
        host = self.out[:K].cpu().numpy()
        return [host[k, :lens[k]].tobytes() for k in range(K)]

    def encode(self, frames):
        self.launch(frames)
        return self.read(frames.shape[0])

    def picture(self):
        """The state's picture, cropped: (Y, Cb, Cr)."""
        wm, hm = (self.W + 15) // 16, (self.H + 15) // 16
        p = self.state[256:256 + 384 * wm * hm].cpu().numpy()
        y = p[:256 * wm * hm].reshape(16 * hm, 16 * wm)
        cb = p[256 * wm * hm:320 * wm * hm].reshape(8 * hm, 8 * wm)
        cr = p[320 * wm * hm:].reshape(8 * hm, 8 * wm)
        return y[:self.H, :self.W], cb[:self.H // 2, :self.W // 2], cr[:self.H // 2, :self.W // 2]


def _device(frames, qp, gop, batch=None, state=True):
    K, H, W, _ = frames.shape
    batch = batch or K
    s = Stream(W, H, qp, gop, batch, state)
    got = []
    for i in range(0, K, batch):
        got += s.encode(_cuda(frames[i:i + batch]))
    return got, s


@pytest.mark.parametrize("item", dc.sequences(), ids=lambda it: it[0])
def test_sequence_samples_and_state_equal_the_oracle(item):
    name, frames, qp, gop = item
    for q, g in ((qp, gop), (min(qp + 12, 51), 2)):
        out = D.encode_stream(frames, q, g)
        got, s = _device(frames, q, g)
        for k, (a, f) in enumerate(zip(got, out)):
            assert a == f["sample"], f"{name} qp {q} gop {g} frame {k}: {len(a)} bytes against {len(f['sample'])}"
        K, H, W, _ = frames.shape
        for a, b in zip(s.picture(), D.crop(out[-1]["filtered"], W, H)):
            assert np.array_equal(a, b), f"{name} qp {q} gop {g}: the state's picture"


@pytest.mark.parametrize("item", [it for it in dc.sequences(large=False) if it[0] in
                                  ("pan80x64", "scene_cut48x32", "pcm_beside_intra64x32", "avatar96x64@32")],
                         ids=lambda it: it[0])
def test_idr_only_stream_without_a_state(item):
    name, frames, qp, _ = item
    want = [f["sample"] for f in D.encode_stream(frames, qp, 1)]
    assert _device(frames, qp, 1, state=False)[0] == want
    assert _device(frames, qp, 1, batch=2)[0] == want


@pytest.mark.parametrize("batch", [1, 3, 16])
def test_batch_splits_give_the_stream_bytes(batch):
    frames = ic.drift(64, 48, [(1, 0), (0, 1), (2, -1), (-1, 0), (0, 0), (3, 2), (1, 1)] * 3, seed=5)   # 22 frames
    want = [f["sample"] for f in D.encode_stream(frames, 30, 9)]
    assert _device(frames, 30, 9, batch)[0] == want


def test_interleaved_writers_and_a_repeat_run(tmp_path):
    from gaussianavatars_b200 import VideoWriter
    a, b = ic.drift(48, 32, [(1, 0)] * 9, seed=2), ic.scene_cut(64, 48)
    files = []
    for run in range(2):
        pa, pb = tmp_path / f"a{run}.mp4", tmp_path / f"b{run}.mp4"
        with VideoWriter(str(pa), 48, 32, qp=28, batch=3, gop=4, deblock=True) as va, \
                VideoWriter(str(pb), 64, 48, qp=34, batch=2, gop=3, deblock=True) as vb:
            for k in range(10):
                va.add(_cuda(a[k]))
                if k < len(b):
                    vb.add(_cuda(b[k]))
        files.append((pa.read_bytes(), pb.read_bytes()))
    assert files[0] == files[1]
    assert files[0][0] == D.mp4([f["sample"] for f in D.encode_stream(a, 28, 4)], 48, 32, 28, gop=4)
    assert files[0][1] == D.mp4([f["sample"] for f in D.encode_stream(b, 34, 3)], 64, 48, 34, gop=3)


def test_graph_replays_continue_the_stream():
    frames = ic.drift(64, 48, [(1, 0), (0, 1)] * 6, seed=7)            # 13 frames
    K, gop, qp = 3, 5, 32
    want = [f["sample"] for f in D.encode_stream(frames[:12], qp, gop)]
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


def test_encode_video_deblocked_equals_the_oracle():
    from gaussianavatars_b200 import encode_video
    clip = ic.drift(48, 32, [(1, 1)] * 20, seed=3)
    for gop in (1, 7):
        assert encode_video(_cuda(clip), qp=30, gop=gop, deblock=True) == \
            D.mp4([f["sample"] for f in D.encode_stream(clip, 30, gop)], 48, 32, 30, gop=gop)


def _decoded_luma(path, K, W, H):
    cv2 = pytest.importorskip("cv2")
    cap = cv2.VideoCapture(str(path))
    assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == K
    cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
    out = []
    for _ in range(K):
        ok, y = cap.read()
        assert ok
        out.append(y.reshape(H, W))
    return out


def test_graphed_render_playback_deblocked(tmp_path):
    pytest.importorskip("cv2")
    from gaussianavatars_b200 import VideoWriter
    from gaussianavatars_b200.graph import GraphedRender
    from tests.test_gpu_display import H_IMG, W_IMG, _flame_setup, _rig
    pc = _flame_setup(T=8)
    cams = _rig(W_IMG, H_IMG, n=8)
    player = GraphedRender(pc, W_IMG, H_IMG, torch.ones(3), outputs="u8", warm_cameras=cams[:1],
                           warm_timesteps=range(8))
    path = tmp_path / "renders.mp4"
    shown = []
    with VideoWriter(str(path), W_IMG, H_IMG, fps=25, qp=30, batch=4, gop=25, deblock=True) as vw:
        for i in range(30):                                            # a fixed camera, the timestep advancing
            player.set_inputs(camera=cams[0], timestep=i % 8)
            player.run()
            vw.add(player.display)
            shown.append(player.display.cpu().numpy())
    out = D.encode_stream(np.stack(shown), 30, 25)
    assert path.read_bytes() == D.mp4([f["sample"] for f in out], W_IMG, H_IMG, 30, gop=25)
    for k, y in enumerate(_decoded_luma(path, 30, W_IMG, H_IMG)):
        assert np.array_equal(y, D.crop(out[k]["filtered"], W_IMG, H_IMG)[0]), k


def test_trajectory_export_deblocked_decodes(tmp_path):
    pytest.importorskip("cv2")
    from PIL import Image
    from gaussianavatars_b200.trajectory import export_trajectory
    from tests.test_gpu_trajectory import _model, _path
    pc, path = _model(), _path()
    video = tmp_path / "traj.mp4"
    res = export_trajectory(pc, path, str(tmp_path / "png"), bg=torch.ones(3, device="cuda"), video=str(video), gop=5,
                            qp=30, batch=16, deblock=True)
    K = res["frames"]
    frames = np.stack([np.asarray(Image.open(tmp_path / "png" / f"{k:05d}.png").convert("RGB")) for k in range(K)])
    out = D.encode_stream(frames, 30, 5)
    assert video.read_bytes() == D.mp4([f["sample"] for f in out], path.W, path.H, 30, gop=5)
    for k, y in enumerate(_decoded_luma(video, K, path.W, path.H)):
        assert np.array_equal(y, D.crop(out[k]["filtered"], path.W, path.H)[0]), k
