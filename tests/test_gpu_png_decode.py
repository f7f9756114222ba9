"""-m gpu: PNG files read on the device (gaussianavatars_b200.png.decode_png, gab200_png_decode,
FrameStore.add_png).

  * every valid file of the corpus (tests/png_corpus.py: the test's own writer with every filter, split / empty /
    ancillary chunks; PIL at every level and optimize; RGB and RGBA; 1x1, 1xN, Nx1 and rows longer than 32 KiB) and
    PIL and encode_png files of synthetic avatar frames at 802x550 and 1080p decode to PIL's convert("RGBA") pixels,
    and with channels=3 to their first three channels;
  * decode_png(encode_png(x)) == x;
  * every crafted stream (each deflate path the corpus names, framed as one row so that the whole stream is decoded),
    every crafted refusal and 300 seeded flips and cuts get exactly oracle/inflate.py's status, and decode_png raises
    naming the first such file;
  * one launch of RGB and RGBA files from different compressors with one corrupt file gives each valid file the
    bytes of its single-file decode;
  * FrameStore.add_png stores the bytes and nbytes of PIL + add_rgba; image_metrics and lpips over a decoded
    render / gt pair equal the same calls over PIL-read arrays."""
import math
import zlib

import numpy as np
import pytest
import torch

from oracle import inflate as oi
from tests import png_corpus as pc

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


def _decode(files, channels=4):
    from gaussianavatars_b200 import decode_png
    return decode_png(files, channels, DEV).cpu().numpy()


def _status(files):
    from gaussianavatars_b200.png import decode_png_status
    return decode_png_status(files, 4, DEV)


# ---- valid files ----------------------------------------------------------------------------------------------------
VALID = pc.valid_files()


@pytest.mark.parametrize("channels", [4, 3])
def test_corpus_files_decode_to_pil_pixels(channels):
    for name, data, img in VALID:
        want = pc.pil_pixels(data)[..., :channels]
        got = _decode(data, channels)
        assert got.shape == want.shape and np.array_equal(got, want), name


def _avatar(P, W, H, azimuth, seed=0):
    """(display RGB, RGBA with the alpha plane's bytes) of a synthetic avatar frame."""
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.model import MeshBoundGaussians
    from gaussianavatars_b200.renderer import render_display
    verts, faces = syn.head_mesh()
    params = syn.avatar_splats(P, n_faces=faces.shape[0], seed=seed, sh_degree=3)
    pc_ = MeshBoundGaussians(params, 3, verts, faces, pose_fn=syn.pose_mesh, device=DEV)
    pc_.select_mesh_by_timestep(0)
    cam = syn.orbit_camera(W, H, r=1.0, fovy_deg=20.0, azimuth_deg=azimuth)
    with torch.no_grad():
        out = render_display(cam, pc_, Pipe, torch.ones(3, device=DEV), depth_alpha=True)
    rgb = out["display_u8"]
    a = (out["alpha"][0] * 255 + 0.5).clamp(0, 255).to(torch.uint8)
    return rgb.cpu().numpy(), torch.cat([rgb, a[..., None]], 2).cpu().numpy()


@pytest.mark.parametrize("P,W,H", [(89_000, 802, 550), (100_000, 1920, 1080)])
def test_avatar_frames_pil_and_encode_png(P, W, H):
    from gaussianavatars_b200 import encode_png
    rgb, rgba = _avatar(P, W, H, 15.0)
    files = []
    levels = range(10) if W < 1000 else (0, 1, 6, 9)
    for img in (rgb, rgba):
        files += [pc.pil_png(img, compress_level=lv) for lv in levels] + [pc.pil_png(img, optimize=True)]
    files.append(encode_png(torch.from_numpy(rgb).to(DEV).contiguous()))
    for f in files:
        want = pc.pil_pixels(f)
        assert np.array_equal(_decode(f), want)
        assert np.array_equal(_decode(f, 3), want[..., :3])
    # one batch of one colour type per compressor: the same bytes
    batch = _decode(files[:4])
    assert all(np.array_equal(batch[i], pc.pil_pixels(files[i])) for i in range(4))


def test_decode_of_encode_is_identity():
    from gaussianavatars_b200 import encode_png
    rng = np.random.default_rng(4)
    for H, W in ((1, 1), (1, 700), (900, 1), (64, 64), (5, 11000), (550, 802)):
        x = torch.from_numpy(rng.integers(0, 256, (3, H, W, 3), dtype=np.uint8)).to(DEV)
        x[1] = x[1, :1, :1]                                    # flat
        x[2] = torch.arange(H * W * 3, device=DEV).reshape(H, W, 3).to(torch.uint8)   # gradient
        files = encode_png(x.contiguous())
        assert torch.equal(_status(files)[0], torch.cat([x, torch.full((3, H, W, 1), 255, dtype=torch.uint8,
                                                                        device=DEV)], 3))
        from gaussianavatars_b200 import decode_png
        assert torch.equal(decode_png(files, 3, DEV), x)
    rgb, _ = _avatar(100_000, 1920, 1080, -20.0, seed=3)
    x = torch.from_numpy(rgb).to(DEV).contiguous()
    from gaussianavatars_b200 import decode_png
    assert torch.equal(decode_png(encode_png(x), 3, DEV), x)


# ---- statuses against the oracle ------------------------------------------------------------------------------------
def _framed(stream: bytes, data: bytes) -> list:
    """(IDAT, W, H, colour) framings of a stream that inflates to `data`: one row that fits it exactly when one does
    (so the Adler-32 and the filter are reached), and one row too wide and one too narrow."""
    out = []
    for c, color in ((3, 2), (4, 6)):
        if len(data) > 1 and (len(data) - 1) % c == 0:
            out.append((stream, (len(data) - 1) // c, 1, color))
    out.append((stream, len(data) // 3 + 2, 1, 2))
    if len(data) > 8:
        out.append((stream, (len(data) - 5) // 4, 1, 6))
    return out


def _cases():
    cases = []
    for name, stream, data in pc.crafted_streams():
        cases += [(f"{name}_{k}", *f) for k, f in enumerate(_framed(stream, data))]
    for name, stream in pc.zlib_sweep(bytes(range(256)) * 40)[::7]:
        cases += [(f"{name}_{k}", *f) for k, f in enumerate(_framed(stream, bytes(range(256)) * 40))]
    cases += [(n, idat, W, H, color) for n, idat, W, H, color, _ in pc.error_streams()]
    cases += pc.mutations(pc.mutation_bases())
    return cases


def test_every_stream_gets_the_oracles_status():
    cases = _cases()
    by_size = {}
    for name, idat, W, H, color in cases:
        by_size.setdefault((W, H), []).append((name, idat, color))
    seen = set()
    for (W, H), group in by_size.items():
        files = [pc.png_file(W, H, color, idat) for _, idat, color in group]
        px, st, _ = _status(files)
        for (name, idat, color), s, got in zip(group, st, px):
            want, ws, _ = oi.decode_idat(idat, W, H, color)
            assert s == ws, (name, oi.STATUS[s], oi.STATUS[ws])
            if ws == oi.OK:
                assert np.array_equal(got.cpu().numpy(), want), name
            seen.add(ws)
    assert seen == set(range(12))   # every status, OK included, was met


def test_decode_png_raises_naming_the_first_bad_file(tmp_path):
    from gaussianavatars_b200 import decode_png
    W, H = 4, 3
    good = pc.png_file(W, H, 2, zlib.compress(b"\x00" * (H * (1 + 3 * W))))
    bad = {n: pc.png_file(W, H, c, idat) for n, idat, _, _, c, _ in pc.error_streams()}
    path = tmp_path / "f.png"
    path.write_bytes(bad["wrong_adler"])
    with pytest.raises(ValueError, match=r"file 2 \(.*f\.png\): Adler-32 mismatch \(status 10\)"):
        decode_png([good, good, str(path), bad["fixed_286"]], device=DEV)
    with pytest.raises(ValueError, match=r"file 1: distance too far back \(status 6\)"):
        decode_png([good, bad["distance_before_first_byte"], bad["filter_5"]], device=DEV)
    with pytest.raises(ValueError, match=r"file 0: invalid row filter type \(status 11\)"):
        decode_png(bad["filter_5"], device=DEV)


def test_mixed_launch_equals_single_decodes():
    rng = np.random.default_rng(8)
    H, W = 37, 53
    files = []
    for k in range(12):
        c = 4 if k % 2 else 3
        img = rng.integers(0, 60, (H, W, c), dtype=np.uint8)
        img[:, W // 2:] = img[:, :1]
        if k % 3 == 0:
            files.append(pc.pil_png(img, compress_level=k % 10))
        elif k % 3 == 1:
            files.append(pc.png_file(W, H, 6 if c == 4 else 2, zlib.compress(pc.filter_rows(img, [4, 1, 0]), 1),
                                     split=[5, 0, 9]))
        else:
            co = zlib.compressobj(9, zlib.DEFLATED, 10, 9, zlib.Z_RLE)
            files.append(pc.png_file(W, H, 6 if c == 4 else 2, co.compress(pc.filter_rows(img, [3])) + co.flush()))
    corrupt = bytearray(files[5])
    corrupt[60] ^= 0xFF
    files[5] = bytes(corrupt)
    px, st, _ = _status(files)
    assert st[5] != 0 and st.count(0) == 11
    for k, f in enumerate(files):
        if k != 5:
            assert np.array_equal(px[k].cpu().numpy(), _decode(f)), k


# ---- the callers ----------------------------------------------------------------------------------------------------
def test_frame_store_add_png_equals_pil_and_add_rgba(tmp_path):
    from gaussianavatars_b200 import FrameStore
    from PIL import Image
    _, rgba = _avatar(20_000, 160, 112, 10.0)
    frames = [rgba, rgba[::-1].copy(), np.ascontiguousarray(rgba[..., :3])]
    paths = []
    for i, f in enumerate(frames):
        p = tmp_path / f"{i}.png"
        Image.fromarray(f).save(p)
        paths.append(str(p))
    bg = [1.0, 1.0, 1.0]
    a, b = FrameStore(160, 112, bg, DEV), FrameStore(160, 112, bg, DEV)
    ids_a = a.add_png(paths, batch=2)
    ids_b = b.add_rgba(torch.from_numpy(np.stack([np.asarray(Image.open(p).convert("RGBA")) for p in paths])))
    assert ids_a == ids_b == [0, 1, 2] and a.nbytes == b.nbytes
    for x, y in zip(a.decode(ids_a), b.decode(ids_b)):
        assert torch.equal(x, y)
    with pytest.raises(ValueError, match="files 0..2 are 160x112, the store holds 32x32 frames"):
        FrameStore(32, 32, bg, DEV).add_png(paths)


def test_metrics_over_decoded_pairs_equal_pil_reads():
    from gaussianavatars_b200 import LpipsNet, decode_png, image_metrics, lpips
    from tests import lpips_oracle as ol
    W, H = 160, 112
    render, _ = _avatar(30_000, W, H, 0.0)
    gt, _ = _avatar(30_000, W, H, 4.0, seed=1)
    files = [pc.pil_png(render), pc.pil_png(gt, compress_level=9)]
    dec = decode_png(files, 3, DEV)
    pil = [torch.from_numpy(pc.pil_pixels(f)[..., :3].copy()).to(DEV) for f in files]
    feats, lin = ol.seeded_weights("vgg", ol.SEED["vgg"])
    net = LpipsNet("vgg", feats, lin, DEV)
    m_dev = image_metrics(dec[0], dec[1].permute(2, 0, 1).contiguous())
    m_pil = image_metrics(pil[0], pil[1].permute(2, 0, 1).contiguous())
    assert torch.equal(m_dev, m_pil)
    l_dev = lpips(dec[0], dec[1].permute(2, 0, 1).contiguous(), net)
    l_pil = lpips(pil[0], pil[1].permute(2, 0, 1).contiguous(), net)
    assert torch.equal(l_dev, l_pil) and math.isfinite(float(l_dev))
