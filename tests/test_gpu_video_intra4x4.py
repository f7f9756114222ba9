"""GPU: the I_NxN device H.264 stream (gab200_h264_encode_flags with GAB200_H264_INTRA4X4, VideoWriter(intra4x4=True),
encode_video(intra4x4=True), export_trajectory(intra4x4=True)) against tests/h264_intra4x4_oracle.py, byte for byte:
every corpus sequence at two QPs, IDR-only and with gop 25, with and without the filter, the state's picture against
the oracle's, the flags entry without the option against the existing entries, batch splits, two interleaved
writers, CUDA graph replays that continue the stream, and a GraphedRender playback loop and a trajectory export whose
files FFmpeg decodes to the oracle's pictures."""
import numpy as np
import pytest
import torch

from tests import h264_intra4x4_corpus as c4
from tests import h264_intra4x4_oracle as I
from tests import h264_inter_corpus as ic

pytestmark = pytest.mark.gpu


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class Stream:
    """One stream's device state and buffers through gab200_h264_encode_flags; encode(frames) returns the samples of
    the next frames."""

    def __init__(self, W, H, qp, gop, batch, deblock=False, intra4x4=True, state=True):
        from gaussianavatars_b200 import video as V
        self.V, self.qp, self.gop, self.W, self.H = V, qp, gop, W, H
        self.deblock, self.intra4x4 = deblock, intra4x4
        self.state = V.state_buffer(H, W, "cuda") if state else None
        self.scratch = V.flags_scratch(batch, H, W, gop, deblock, intra4x4, "cuda")
        self.out = torch.zeros((batch, V.slot_stride(W, H, gop)), dtype=torch.uint8, device="cuda")
        self.out_len = torch.empty(batch, dtype=torch.int64, device="cuda")

    def launch(self, frames):
        self.V.launch_encode_flags(frames, self.qp, self.gop, self.deblock, self.intra4x4, self.state, self.scratch,
                                   self.out, self.out_len)

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


def _device(frames, qp, gop, deblock=False, batch=None, state=True, intra4x4=True):
    K, H, W, _ = frames.shape
    batch = batch or K
    s = Stream(W, H, qp, gop, batch, deblock, intra4x4, state)
    got = []
    for i in range(0, K, batch):
        got += s.encode(_cuda(frames[i:i + batch]))
    return got, s


@pytest.mark.parametrize("item", c4.sequences(large=False), ids=lambda it: it[0])
def test_sequence_samples_and_state_equal_the_oracle(item):
    name, frames, qp, _ = item
    K, H, W, _ = frames.shape
    for q in (qp, min(qp + 12, 51)):
        for gop in (1, 25):
            for deblock in (False, True):
                out = I.encode_stream(frames, q, gop, deblock=deblock)
                got, s = _device(frames, q, gop, deblock)
                where = f"{name} qp {q} gop {gop} deblock {deblock}"
                for k, (a, f) in enumerate(zip(got, out)):
                    assert a == f["sample"], f"{where} frame {k}: {len(a)} bytes against {len(f['sample'])}"
                for a, b in zip(s.picture(), I.crop(out[-1]["filtered"], W, H)):
                    assert np.array_equal(a, b), f"{where}: the state's picture"


def test_the_large_avatar_equals_the_oracle():
    name, frames, qp, gop = c4.sequences()[-1]
    out = I.encode_stream(frames, qp, gop)
    got, _ = _device(frames, qp, gop)
    assert got == [f["sample"] for f in out]
    assert sum(int((f["types"] == "I4").sum()) for f in out) > 0


@pytest.mark.parametrize("item", [it for it in c4.sequences(large=False) if it[0] in
                                  ("pan80x64", "pcm_beside_intra64x32", "avatar96x64@32", "directions_motion80x64")],
                         ids=lambda it: it[0])
def test_flags_without_intra4x4_give_the_existing_entries_bytes(item):
    from gaussianavatars_b200 import video as V
    name, frames, qp, gop = item
    K, H, W, _ = frames.shape
    x = _cuda(frames)
    stride = V.slot_stride(W, H, gop)
    out = torch.zeros((K, stride), dtype=torch.uint8, device="cuda")
    out_len = torch.empty(K, dtype=torch.int64, device="cuda")

    def read():
        lens = out_len.tolist()
        host = out.cpu().numpy()
        return [host[k, :lens[k]].tobytes() for k in range(K)]

    V.launch_encode(x, qp, V.scratch(K, H, W, "cuda"), out, out_len)
    assert _device(frames, qp, 1, state=False, intra4x4=False)[0] == read()
    V.launch_encode_stream(x, qp, gop, V.state_buffer(H, W, "cuda"), V.scratch(K, H, W, "cuda"), out, out_len)
    assert _device(frames, qp, gop, intra4x4=False)[0] == read()
    V.launch_encode_deblocked(x, qp, gop, V.state_buffer(H, W, "cuda"), V.deblocked_scratch(K, H, W, gop, "cuda"), out,
                              out_len)
    assert _device(frames, qp, gop, deblock=True, intra4x4=False)[0] == read()


@pytest.mark.parametrize("batch", [1, 3, 16])
def test_batch_splits_give_the_stream_bytes(batch):
    frames = c4.moving_directions(64, 48, 3)
    frames = np.concatenate([frames, ic.drift(64, 48, [(1, 0), (0, 1), (2, -1)] * 3, seed=5)])   # 13 frames
    for deblock in (False, True):
        want = [f["sample"] for f in I.encode_stream(frames, 24, 9, deblock=deblock)]
        assert _device(frames, 24, 9, deblock, batch)[0] == want


def test_interleaved_writers_and_a_repeat_run(tmp_path):
    from gaussianavatars_b200 import VideoWriter
    a, b = ic.drift(48, 32, [(1, 0)] * 9, seed=2), c4.moving_directions(64, 48, 3)
    files = []
    for run in range(2):
        pa, pb = tmp_path / f"a{run}.mp4", tmp_path / f"b{run}.mp4"
        with VideoWriter(str(pa), 48, 32, qp=28, batch=3, gop=4, intra4x4=True) as va, \
                VideoWriter(str(pb), 64, 48, qp=22, batch=2, gop=1, deblock=True, intra4x4=True) as vb:
            for k in range(10):
                va.add(_cuda(a[k]))
                if k < len(b):
                    vb.add(_cuda(b[k]))
        files.append((pa.read_bytes(), pb.read_bytes()))
    assert files[0] == files[1]
    assert files[0][0] == I.mp4([f["sample"] for f in I.encode_stream(a, 28, 4)], 48, 32, 28, gop=4)
    assert files[0][1] == I.mp4([f["sample"] for f in I.encode_stream(b, 22, 1, deblock=True)], 64, 48, 22, gop=1)


def test_graph_replays_continue_the_stream():
    frames = ic.drift(64, 48, [(1, 0), (0, 1)] * 6, seed=7)            # 13 frames
    K, gop, qp = 3, 5, 26
    for deblock in (False, True):
        want = [f["sample"] for f in I.encode_stream(frames[:12], qp, gop, deblock=deblock)]
        s = Stream(64, 48, qp, gop, K, deblock)
        src = _cuda(frames[:K]).clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            s.launch(src)                                              # warm-up: the stream's first batch
        torch.cuda.current_stream().wait_stream(side)
        got = s.read(K)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            s.launch(src)
        for i in range(K, 12, K):
            src.copy_(_cuda(frames[i:i + K]))
            g.replay()
            got += s.read(K)
        assert got == want, deblock


def test_encode_video_intra4x4_equals_the_oracle():
    from gaussianavatars_b200 import encode_video
    clip = ic.drift(48, 32, [(1, 1)] * 20, seed=3)
    for gop in (1, 7):
        for deblock in (False, True):
            assert encode_video(_cuda(clip), qp=24, gop=gop, deblock=deblock, intra4x4=True) == \
                I.mp4([f["sample"] for f in I.encode_stream(clip, 24, gop, deblock=deblock)], 48, 32, 24, gop=gop)


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


def test_graphed_render_playback_intra4x4(tmp_path):
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
    with VideoWriter(str(path), W_IMG, H_IMG, fps=25, qp=20, batch=4, gop=25, intra4x4=True) as vw:
        for i in range(30):                                            # a fixed camera, the timestep advancing
            player.set_inputs(camera=cams[0], timestep=i % 8)
            player.run()
            vw.add(player.display)
            shown.append(player.display.cpu().numpy())
    out = I.encode_stream(np.stack(shown), 20, 25)
    assert path.read_bytes() == I.mp4([f["sample"] for f in out], W_IMG, H_IMG, 20, gop=25)
    for k, y in enumerate(_decoded_luma(path, 30, W_IMG, H_IMG)):
        assert np.array_equal(y, I.crop(out[k]["filtered"], W_IMG, H_IMG)[0]), k


def test_trajectory_export_intra4x4_decodes(tmp_path):
    pytest.importorskip("cv2")
    from PIL import Image
    from gaussianavatars_b200.trajectory import export_trajectory
    from tests.test_gpu_trajectory import _model, _path
    pc, path = _model(), _path()
    video = tmp_path / "traj.mp4"
    res = export_trajectory(pc, path, str(tmp_path / "png"), bg=torch.ones(3, device="cuda"), video=str(video), gop=5,
                            qp=26, batch=16, deblock=True, intra4x4=True)
    K = res["frames"]
    frames = np.stack([np.asarray(Image.open(tmp_path / "png" / f"{k:05d}.png").convert("RGB")) for k in range(K)])
    out = I.encode_stream(frames, 26, 5, deblock=True)
    assert video.read_bytes() == I.mp4([f["sample"] for f in out], path.W, path.H, 26, gop=5)
    for k, y in enumerate(_decoded_luma(video, K, path.W, path.H)):
        assert np.array_equal(y, I.crop(out[k]["filtered"], path.W, path.H)[0]), k
