"""-m gpu: PNG files written on the device (csrc/png.cu, gaussianavatars_b200.png.encode_png) and by the playback and
evaluation replays (GraphedRender / GraphedEval png=True, host_png).

Every file is checked four ways -- PIL opens it as RGB of the right size with the input's pixels; zlib inflates the
IDAT data to its end with nothing left over (the Adler-32); every chunk's CRC-32 is zlib.crc32 of its type and data;
the chunk order and the IHDR fields -- every row's filter byte is oracle/png.py's choice, and, for every image of at
most ORACLE_BYTES filtered bytes, the file is oracle/png.py's encode_png byte for byte.

CORPUS holds natural images (flat, gradient, noise, mixed rows) and images built to force the encoder's rare paths: a
literal tree and a code-length tree past their length limits, an all-literal segment that still compresses, matches at
exactly 32768 and into the previous segment, both block-choice ties, and IDAT chunks that end on and one byte past a
64 KiB CRC piece or span more than 1024 of them.  tests/test_oracle_png.py shows from the oracle's path report, on the
CPU, that the corpus reaches every one of them."""
import io
import struct
import zlib

import numpy as np
import pytest
import torch

from oracle import png as opng

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


def _chunks(data: bytes) -> list:
    assert data[:8] == b"\x89PNG\r\n\x1a\n", "signature"
    pos, out = 8, []
    while pos < len(data):
        n, = struct.unpack(">I", data[pos:pos + 4])
        typ, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        crc, = struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])
        assert crc == zlib.crc32(typ + body) & 0xFFFFFFFF, f"CRC of {typ}"
        out.append((typ, body))
        pos += 12 + n
    assert pos == len(data)
    return out


# The largest image (filtered bytes) whose file is compared with the oracle's byte for byte: the oracle takes 1-2 s per
# MB of filtered stream on one CPU core (0.4 s for the 400x300 noise image, 2.8 s for an 802x550 display frame), so the
# 1080p display frame (6.2 MB) and noise_4800 (69 MB) get the other checks only.
ORACLE_BYTES = 1 << 21


def check_file(data: bytes, img: np.ndarray):
    """check_stream, and the file is the oracle's when the image is at most ORACLE_BYTES filtered bytes."""
    check_stream(data, img)
    if opng.filtered_bytes(img.shape[1], img.shape[0]) <= ORACLE_BYTES:
        assert data == opng.encode_png(img), "the file is not the oracle's, byte for byte"


def check_stream(data: bytes, img: np.ndarray):
    """The four checks, the filters against the oracle, and the bound."""
    from PIL import Image
    from gaussianavatars_b200 import png_bound
    H, W = img.shape[:2]
    chunks = _chunks(data)
    types = [t for t, _ in chunks]
    assert types[0] == b"IHDR" and types[-1] == b"IEND" and set(types[1:-1]) == {b"IDAT"}, types
    assert struct.unpack(">IIBBBBB", chunks[0][1]) == (W, H, 8, 2, 0, 0, 0)
    assert chunks[-1][1] == b""
    d = zlib.decompressobj()
    raw = d.decompress(b"".join(b for t, b in chunks if t == b"IDAT"))
    assert d.eof and d.unused_data == b"", "the zlib stream does not end where the IDAT data ends"
    ids, filtered = opng.filter_image(img)
    assert raw == filtered.tobytes(), "the filtered stream is not the oracle's (filter choice or filtered bytes)"
    im = Image.open(io.BytesIO(data))
    im.load()
    assert im.mode == "RGB" and im.size == (W, H)
    assert np.array_equal(np.asarray(im), img), "pixels differ"
    assert len(data) <= png_bound(W, H) == opng.png_bound(W, H)


def _encode(img: np.ndarray) -> bytes:
    from gaussianavatars_b200 import encode_png
    return encode_png(torch.from_numpy(np.ascontiguousarray(img)).to(DEV))


def _gradient(H, W):
    y, x = np.mgrid[0:H, 0:W]
    return np.stack([x * 255 // max(W - 1, 1), y * 255 // max(H - 1, 1), (x + y) % 256], -1).astype(np.uint8)


def _mixed(H, W, seed):
    """Rows of noise, flat rows and gradient rows: blocks of every kind, at varied bit offsets."""
    rng = np.random.default_rng(seed)
    img = _gradient(H, W)
    rows = rng.random(H)
    img[rows < 0.3] = rng.integers(0, 256, (int((rows < 0.3).sum()), W, 3), dtype=np.uint8)
    img[(rows >= 0.3) & (rows < 0.5)] = 200
    return img


def _from_sub(f) -> np.ndarray:
    """A one-row image whose Sub-filtered bytes are f (3W of them): each channel is the running sum of its bytes.  The
    filter rule picks Sub when f is small signed bytes; the images below assert that it does."""
    f = np.asarray(f, np.int64)
    return (f.reshape(-1, 3).cumsum(0) & 255).astype(np.uint8)[None]


def _de_bruijn(k: int, n: int) -> np.ndarray:
    """The lexicographically least de Bruijn sequence B(k, n): every n-symbol word once, read cyclically."""
    a, seq = [0] * (k * n), []

    def db(t, p):
        if t > n:
            if n % p == 0:
                seq.extend(a[1:p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, k):
                a[t] = j
                db(t + 1, t)
    db(1, 1)
    return np.array(seq, np.int64)


def _de_bruijn_row(W: int) -> np.ndarray:
    """A 1 x W image whose filtered stream is B(32, 3) over the small signed bytes -16..15, cycled: the filter byte (1,
    Sub) and the row make the first 32768 bytes, in which no 3 bytes repeat -- a segment of 32768 literals that still
    compresses (5-bit codes), whose parse needs all 15 doubling rounds -- and every later byte repeats the one 32768
    before it: matches at exactly the window's distance, 258 long, into the previous segment."""
    v = _de_bruijn(32, 3)
    v = np.where(v < 16, v, v + 224)
    v = np.roll(v, -int(np.argmax(v == 1)))           # starts with the filter byte
    return _from_sub(np.resize(np.roll(v, -1), 3 * W))


def _fibonacci_bytes(n: int, seed: int) -> np.ndarray:
    """n filtered bytes: 160 small signed values drawn uniformly and 12 more with counts 1, 2, 3, 5, ..., 233.  With the
    end-of-block symbol's count of one the rare twelve form one chain, 17 deep under the body's 8, past the 15-bit
    limit."""
    rng = np.random.default_rng(seed)
    fib = [1, 2]
    while len(fib) < 12:
        fib.append(fib[-1] + fib[-2])
    body, chain = np.arange(-80, 80) & 255, np.arange(80, 92)
    return rng.permutation(np.concatenate([np.repeat(chain, fib), rng.choice(body, n - sum(fib))]))


def _hex(h: int, w: int, data: str) -> np.ndarray:
    return np.frombuffer(bytes.fromhex(data), np.uint8).reshape(h, w, 3).copy()


def _flat_tail(W: int, T: int, seed: int) -> np.ndarray:
    """A noise row whose last T pixels are flat."""
    img = np.random.default_rng(seed).integers(0, 256, (1, W, 3), dtype=np.uint8)
    img[:, W - T:] = 7
    return img


_rng = np.random.default_rng(1)
CORPUS = {
    "white": np.full((48, 64, 3), 255, np.uint8),
    "black": np.zeros((31, 17, 3), np.uint8),
    "one_colour": np.full((40, 23, 3), [12, 200, 77], np.uint8),
    "1x1": _rng.integers(0, 256, (1, 1, 3), dtype=np.uint8),
    "1xN": _rng.integers(0, 256, (1, 1000, 3), dtype=np.uint8),
    "Nx1": _gradient(1500, 1),
    "noise": _rng.integers(0, 256, (400, 300, 3), dtype=np.uint8),
    "gradient": _gradient(300, 257),
    "wide_11000": _mixed(5, 11000, 2),          # 3W + 1 > 32768: the previous row is beyond the window
    "one_full_segment": _mixed(2, 5461, 3),     # exactly 32768 filtered bytes
    "segment_minus_1": _mixed(1, 10922, 4),     # 32767
    "segment_plus_2": _mixed(1, 10923, 5),      # 32770
    **{f"mixed_{h}x{w}": _mixed(h, w, h * w) for h, w in ((97, 401), (128, 512), (211, 173), (300, 333), (64, 1030))},
    # built for the rare paths (tests/test_oracle_png.py names the path each one reaches)
    "de_bruijn": _de_bruijn_row(21846),
    "fibonacci": _from_sub(_fibonacci_bytes(3 * 10922, 0)),
    # found by a seeded search over tiny images: the fixed and dynamic costs tie (304 bits), and fixed wins over
    # stored (336); a Huffman block of exactly the stored block's 480 bits; one of 818 bits, 2 over stored, rendered
    # and then dropped
    "tie_fixed_dynamic": _hex(1, 12, "349d34f07cf004073407bd347cbdbd9d047c04f0079d7c07bd04bdd9bd9d9df07cf0047c"),
    "tie_stored_huffman": _hex(1, 18, "dad195a4f5cd87d9e4ce8d7ebae99ba4eeffda9cf3d2e1f67aa0cfe8d38a81e49cbf8cfdbafd8d"
                                      "c3a9db7c94f1d4f4d1b3f0b5af88be"),
    "stored_over_huffman": _hex(1, 32, "c426e5487322659f79b0a96af63a36f8ba697baa942ba38e4d91ffb0a7fc23effb4afe82d954bd"
                                       "3421cb1ed55341c753943d2a214848b14ec89cf0b6f32bb34193f176181c82d516b3a853535fef"
                                       "4fb5c761d83c302fab815a34fca77046c63e"),
    # IDAT type + data: 65536 bytes (2 stored blocks: n + 5 S + 6 = 65532 data bytes) and 65537 bytes, one byte into
    # a second png_assemble_kernel piece
    "idat_65536": np.random.default_rng(3).integers(0, 256, (2, 10919, 3), dtype=np.uint8),
    "idat_65537": _flat_tail(21845, 20, 3),
    # 69 MB of stored blocks: 1055 pieces, so each png_finish_kernel thread combines a run of two
    "noise_4800": np.random.default_rng(4).integers(0, 256, (4800, 4800, 3), dtype=np.uint8),
}


@pytest.mark.parametrize("name", sorted(CORPUS))
def test_round_trip_filters_bound_and_determinism(name):
    img = CORPUS[name]
    data = _encode(img)
    check_file(data, img)
    assert _encode(img) == data, "two encodes of the same input differ"
    if name == "noise_4800":   # png_finish_kernel's threads each combine a run of pieces
        idat, = struct.unpack(">I", data[33:37])
        assert -(-(4 + idat) // opng.PIECE) > 1024


def test_noise_takes_stored_blocks():
    img = CORPUS["noise"]
    n = opng.filtered_bytes(img.shape[1], img.shape[0])
    # stored: the filtered bytes plus 5 or 6 bytes per block, and the fixed chunk overhead
    assert len(_encode(img)) <= 57 + n + 6 * opng.segments(img.shape[1], img.shape[0])


def test_a_batch_of_16_different_images():
    from gaussianavatars_b200 import encode_png
    imgs = np.stack([_mixed(120, 150, s) if s % 3 else _rng.integers(0, 256, (120, 150, 3), dtype=np.uint8)
                     for s in range(16)])
    imgs[5] = 255
    files = encode_png(torch.from_numpy(imgs).to(DEV))
    assert isinstance(files, list) and len(files) == 16
    for k in range(16):
        check_file(files[k], imgs[k])
        assert files[k] == _encode(imgs[k]), f"view {k} of the batch differs from its own encode"


def test_a_batch_whose_views_take_different_paths():
    """One launch of four views of one shape, each its own mix of block kinds and segment paths: the de Bruijn row
    (32768 literals, then matches at 32768), Fibonacci bytes (the literal tree past 15 bits), noise (stored) and a flat
    image.  Each view's file is its own encode's and the oracle's."""
    from gaussianavatars_b200 import encode_png
    W = 21846
    fib = _from_sub(np.concatenate([_fibonacci_bytes(3 * 10922, 0), _fibonacci_bytes(3 * W - 3 * 10922, 1)]))
    imgs = np.stack([_de_bruijn_row(W), fib, np.random.default_rng(5).integers(0, 256, (1, W, 3), np.uint8),
                     np.full((1, W, 3), 200, np.uint8)])
    # per segment: block kind, literal tree past its limit, all literals, farthest match
    paths = [tuple((r.kind, r.lit_depth[0] > 15, r.literals == r.symbols, r.farthest) for r in rep)
             for rep in (opng.encode_png(img, report=True)[1] for img in imgs)]
    assert len(set(paths)) == 4 and [p[0][0] for p in paths] == ["dynamic", "dynamic", "stored", "dynamic"], paths
    assert paths[0][0][2] and paths[0][1][3] == 32768 and paths[1][0][1]
    files = encode_png(torch.from_numpy(imgs).to(DEV))
    for k in range(4):
        check_file(files[k], imgs[k])
        assert files[k] == _encode(imgs[k]), f"view {k} of the batch differs from its own encode"


def test_refusals_on_the_device():
    from gaussianavatars_b200 import encode_png
    t = torch.zeros(4, 5, 3, dtype=torch.uint8, device=DEV)
    with pytest.raises(ValueError, match="contiguous"):
        encode_png(t.transpose(0, 1))
    with pytest.raises(ValueError, match="uint8"):
        encode_png(t.float())


# ---- display frames of the synthetic avatar -------------------------------------------------------------------------
def avatar_display(P, W, H, azimuth=15.0, seed=0):
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.model import MeshBoundGaussians
    from gaussianavatars_b200.renderer import render_display
    verts, faces = syn.head_mesh()
    params = syn.avatar_splats(P, n_faces=faces.shape[0], seed=seed, sh_degree=3)
    pc = MeshBoundGaussians(params, 3, verts, faces, pose_fn=syn.pose_mesh, device=DEV)
    pc.select_mesh_by_timestep(0)
    cam = syn.orbit_camera(W, H, r=1.0, fovy_deg=20.0, azimuth_deg=azimuth)
    with torch.no_grad():
        return render_display(cam, pc, Pipe, torch.ones(3, device=DEV))["display_u8"].contiguous()


@pytest.mark.parametrize("P,W,H", [(89_000, 802, 550), (100_000, 1920, 1080)])
def test_avatar_display_frames_are_no_larger_than_pil_level_1(P, W, H):
    from PIL import Image
    disp = avatar_display(P, W, H)
    img = disp.cpu().numpy()
    data = _encode(img)
    check_file(data, img)
    sizes = {}
    for level in (1, 6):
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format="PNG", compress_level=level)
        sizes[level] = buf.tell()
    print(f"[png {W}x{H}] {len(data)} bytes, PIL level 1 {sizes[1]}, level 6 {sizes[6]}")
    assert len(data) <= sizes[1], f"{len(data)} bytes, PIL's compress_level=1 file {sizes[1]}"


# ---- the replays ----------------------------------------------------------------------------------------------------
def _decode(data: bytes) -> torch.Tensor:
    from PIL import Image
    return torch.from_numpy(np.asarray(Image.open(io.BytesIO(data)).convert("RGB")).copy())


def test_graphed_render_png_over_a_flame_sequence():
    from gaussianavatars_b200 import encode_png
    from gaussianavatars_b200.graph import GraphedRender
    from tests.test_gpu_display import H_IMG, W_IMG, _flame_setup, _rig
    pc = _flame_setup(T=8)
    cams = _rig(W_IMG, H_IMG, n=8)
    kw = dict(warm_cameras=cams, warm_timesteps=range(8))
    view = GraphedRender(pc, W_IMG, H_IMG, torch.ones(3), outputs="u8", host_slots=2, png=True, **kw)
    plain = GraphedRender(pc, W_IMG, H_IMG, torch.ones(3), outputs="u8", host_slots=2, **kw)
    frames = []
    for i in range(16):
        for v in (view, plain):
            v.set_inputs(camera=cams[i % 8], timestep=(3 * i) % 8)
            v.run()
        frames.append(view.display.clone())
        if i >= 1:   # a consumer one replay behind
            data = view.host_png(i - 1)
            assert torch.equal(_decode(data), frames[i - 1].cpu()), f"replay {i - 1}"
            check_file(data, frames[i - 1].cpu().numpy())
            assert data == encode_png(frames[i - 1]), "the replay's file is not encode_png of its display"
        assert torch.equal(view.host_frame(i), plain.host_frame(i)), "host_frame changed with png=True"
    assert view.captures == plain.captures == 1 and not view.overflowed()


def test_graphed_render_png_with_the_mesh_overlay():
    from gaussianavatars_b200.graph import GraphedRender
    from tests.test_gpu_display import H_IMG, W_IMG, _flame_setup, _rig
    pc = _flame_setup(T=8)
    cams = _rig(W_IMG, H_IMG, n=4)
    view = GraphedRender(pc, W_IMG, H_IMG, torch.ones(3), outputs="u8", host_slots=2, png=True, warm_cameras=cams,
                         warm_timesteps=range(8), mesh_opacity=0.5)
    for i in range(6):
        view.set_inputs(camera=cams[i % 4], timestep=i, mesh_opacity=0.3 + 0.1 * i)
        view.run()
        want = view.display.clone()
        data = view.host_png(i)
        assert torch.equal(_decode(data), want.cpu()), f"replay {i} with the overlay"
    assert view.captures == 1


def test_graphed_render_png_16_views_per_replay():
    from gaussianavatars_b200.graph import GraphedRender
    from tests.test_gpu_display import H_IMG, W_IMG, _flame_setup, _rig
    pc = _flame_setup(T=4)
    cams = _rig(W_IMG, H_IMG, n=16)
    view = GraphedRender(pc, W_IMG, H_IMG, torch.ones(3), outputs="both", host_slots=2, png=True,
                         views_per_replay=16, warm_cameras=[cams], warm_timesteps=range(4))
    for t in range(3):
        view.set_inputs(cameras=cams, timestep=t)
        view.run()
        want = view.display.clone()
        files = view.host_png(t)
        assert isinstance(files, list) and len(files) == 16
        for k in range(16):
            assert torch.equal(_decode(files[k]), want[k].cpu()), f"replay {t}, view {k}"
        assert len(set(files)) > 1
    assert view.captures == 1


def test_host_png_refuses_an_overflowed_replay():
    from gaussianavatars_b200.graph import GraphedRender
    from tests.test_gpu_display import H_IMG, W_IMG, _flame_setup, _rig
    pc = _flame_setup(T=6)
    cam = _rig(W_IMG, H_IMG, n=4)[1]
    view = GraphedRender(pc, W_IMG, H_IMG, torch.ones(3), outputs="u8", host_slots=2, png=True, capacity=2000)
    view.set_inputs(camera=cam, timestep=1)
    view.run(check=False)
    assert view.overflowed()
    with pytest.raises(RuntimeError, match="replay 0 overflowed its instance capacity"):
        view.host_png(0)
    view.run(check=True)   # regrows, re-captures, replays
    assert not view.overflowed()
    assert torch.equal(_decode(view.host_png(1)), view.display.cpu())


def test_graphed_eval_scores_are_unchanged_by_png():
    from gaussianavatars_b200.graph import GraphedEval
    from tests.test_gpu_metrics import H_IMG, W_IMG, _models, _rig, _truth_u8
    pc, truth, _ = _models(T=8)
    cams = _rig(W_IMG, H_IMG, n=6)
    bg = torch.ones(3)
    gts = [_truth_u8(truth, c, i, bg) for i, c in enumerate(cams)]
    evs = [GraphedEval(pc, W_IMG, H_IMG, bg, views=6, source="u8", host_slots=2, png=p, warm_cameras=cams,
                       warm_timesteps=range(6)) for p in (False, True)]
    for i in range(6):
        for ev in evs:
            ev.set_inputs(camera=cams[i], timestep=i, gt_u8=gts[i], view=i)
            ev.run()
        assert torch.equal(_decode(evs[1].host_png(i)), evs[0].host_frame(i)), f"view {i}"
    a, b = evs[0].scores(), evs[1].scores()
    assert torch.equal(a["per_view"], b["per_view"])
    assert evs[1].captures == 1
