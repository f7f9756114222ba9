"""-m gpu: the loader's resize on the device (csrc/resize.cu, gaussianavatars_b200.resize, composite_rgba(size=),
FrameStore.add_png(resize=True)).

  * resize_u8 == oracle/resize.py == PIL's `Image.resize`, byte for byte, on the CPU tests' grid of sizes (1-pixel
    inputs and outputs, ratios down to 1/50, upscales, odd sizes, each axis alone), at 3208x2200 -> 1600x1097 and
    1920x1080 -> 1600x900, for "RGB" images as planar channels and "L" images, batched over frames, and on a row wider
    than the kernel stages in shared memory;
  * composite_rgba(size=) gives the reference loader's bytes (tests/golden/resize_vectors.npz), eagerly and replayed
    from a CUDA graph fed new frames;
  * add_png(resize=True) + decode equals the host pipeline -- PIL open, convert("RGBA"), the loader's composite, PIL's
    resize, and PIL's "L" resize of the alpha bytes for the mask -- for RGB and RGBA files, and at the size of the
    store it gives the bytes of resize=False;
  * one GraphedFrame(frames=store) replay on a resized store equals the eager iteration on the resized frame."""
import functools
import io
import re

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import resize as ors
from tests import test_gpu_rgba_mask as RM
from tests import test_gpu_train_graph as TG
from tests.test_host_resize import GOLDEN, GRID, LARGE, composite, golden_cases, image, pil_resize

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
LAM = 0.1


def _g():
    import gaussianavatars_b200 as g
    return g


def _device_resize(planes: np.ndarray, w: int, h: int) -> np.ndarray:
    return _g().resize_u8(torch.from_numpy(np.array(planes)).to(DEV), w, h).cpu().numpy()


# ---- the kernels ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", GRID + LARGE, ids=lambda c: "%dx%d-%dx%d" % c)
def test_kernel_equals_oracle_and_pil(case):
    W, H, w, h = case
    small = W * H <= 600 * 600
    rgb = [image(W, H, 3, s) for s in ((0, 1, 2) if small else (0,))]
    planes = np.ascontiguousarray(np.stack([a.transpose(2, 0, 1) for a in rgb]))  # (F, 3, H, W)
    got = _device_resize(planes, w, h)
    assert got.shape == (len(rgb), 3, h, w)
    for f, a in enumerate(rgb):
        assert np.array_equal(got[f].transpose(1, 2, 0), pil_resize(a, w, h)), (case, f)
    if small:
        assert np.array_equal(got, ors.resize_u8(planes, w, h))
    grey = image(W, H, 1, 1)
    assert np.array_equal(_device_resize(grey, w, h), pil_resize(grey, w, h)), case


def test_kernel_many_planes_and_a_wide_row():
    """256 frames x 4 planes in one call; a 50,001-pixel row, read from global memory instead of shared."""
    rng = np.random.default_rng(3)
    planes = rng.integers(0, 256, (256, 4, 23, 37), dtype=np.uint8)
    for w, h in ((16, 9), (37, 50), (80, 23)):
        assert np.array_equal(_device_resize(planes, w, h), ors.resize_u8(planes, w, h)), (w, h)
    wide = image(50001, 3, 1, 0)
    for w, h in ((700, 5), (700, 3), (60000, 2)):
        assert np.array_equal(_device_resize(wide, w, h), pil_resize(wide, w, h)), (w, h)


def test_same_size_is_a_copy_and_empty_batches():
    g = _g()
    a = torch.randint(0, 256, (2, 3, 17, 9), dtype=torch.uint8, device=DEV)
    out = g.resize_u8(a, 9, 17)
    assert torch.equal(out, a) and out.data_ptr() != a.data_ptr()
    t = a.transpose(-1, -2)                                                      # strided: made contiguous first
    assert torch.equal(g.resize_u8(t, 5, 11).cpu(), torch.from_numpy(ors.resize_u8(t.cpu().numpy(), 5, 11)))
    assert g.resize_u8(a[:0], 4, 4).shape == (0, 3, 4, 4)


# ---- composite_rgba(size=) -----------------------------------------------------------------------------------------
def test_composite_size_equals_the_reference_loader():
    g = _g()
    cases = list(golden_cases())
    assert len(cases) == 24
    for key, frame, bg, w, h in cases:
        rgba = torch.from_numpy(GOLDEN["rgba_" + frame]).to(DEV)
        gt, mask = g.composite_rgba(rgba, torch.full((3,), bg), size=(w, h))
        assert torch.equal(gt.cpu(), torch.from_numpy(GOLDEN[key])), key
        want_mask = pil_resize(GOLDEN["rgba_" + frame][..., 3], w, h)
        assert np.array_equal(mask[0].cpu().numpy(), want_mask), key


def test_composite_size_is_capturable():
    g = _g()
    bg = torch.tensor([1.0, 0.0, 1.0], device=DEV)
    frames = RM._rgba(6, 61, 45, seed=5).to(DEV)
    static = frames[:3].clone()
    want = g.composite_rgba(static, bg, size=(30, 70))                           # eager, and the warm-up
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gt, mask = g.composite_rgba(static, bg, size=(30, 70))
    for batch in (frames[:3], frames[3:]):
        static.copy_(batch)
        graph.replay()
        torch.cuda.synchronize()
        eager = g.composite_rgba(batch, bg, size=(30, 70))
        assert torch.equal(gt, eager[0]) and torch.equal(mask, eager[1])
    assert gt.shape == want[0].shape == (3, 3, 70, 30) and mask.shape == (3, 1, 70, 30)
    for f in range(3):
        rgba = frames[3 + f].cpu().numpy()
        assert np.array_equal(gt[f].cpu().numpy(), _host_gt(rgba, [1.0, 0.0, 1.0], 30, 70))


# ---- FrameStore.add_png(resize=True) -------------------------------------------------------------------------------
def _host_gt(rgba: np.ndarray, bg, w, h) -> np.ndarray:
    """(3, h, w): the loader's composite at the file's size, then PIL's resize of the "RGB" image."""
    c = composite(rgba, bg)
    img = Image.frombuffer("RGB", (rgba.shape[1], rgba.shape[0]), np.ascontiguousarray(c.transpose(1, 2, 0)).tobytes(),
                           "raw", "RGB", 0, 1)
    return np.asarray(img.resize((w, h))).transpose(2, 0, 1)


def _host_frame(data: bytes, bg, w, h) -> tuple:
    rgba = np.asarray(Image.open(io.BytesIO(data)).convert("RGBA"))
    mask = np.asarray(Image.fromarray(rgba[..., 3], "L").resize((w, h)))
    return _host_gt(rgba, bg, w, h), mask[None]


def _png(rgba: np.ndarray, mode: str) -> bytes:
    buf = io.BytesIO()
    Image.fromarray(rgba if mode == "RGBA" else np.ascontiguousarray(rgba[..., :3]), mode).save(buf, "PNG",
                                                                                               compress_level=1)
    return buf.getvalue()


@pytest.mark.parametrize("W,H,w,h", [(203, 151, 100, 75), (64, 48, 97, 60), (3208, 2200, 1600, 1097),
                                     (1920, 1080, 1600, 900)])
def test_add_png_resize_equals_the_host_pipeline(W, H, w, h):
    g = _g()
    bg = [1.0, 1.0, 1.0] if W % 2 else [0.0, 0.0, 0.0]
    F = 4 if W * H < 10**6 else 1
    rgba = RM._rgba(F, H, W, seed=W).numpy()
    files = [_png(rgba[f], mode) for f in range(F) for mode in ("RGBA", "RGB")]
    store = g.FrameStore(w, h, bg, DEV)
    ids = store.add_png(files, batch=3, resize=True)
    gt, mask = store.decode(ids)
    gt, mask = gt.cpu().numpy(), mask.cpu().numpy()
    for i, data in enumerate(files):
        want_gt, want_mask = _host_frame(data, bg, w, h)
        assert np.array_equal(gt[i], want_gt), (W, H, i)
        assert np.array_equal(mask[i], want_mask), (W, H, i)
    if F == 1:
        assert g.loader_size(W, H) == (w, h)


def test_add_png_resize_at_the_store_size_and_refusals():
    g = _g()
    rgba = RM._rgba(3, 40, 56, seed=9).numpy()
    files = [_png(a, "RGBA") for a in rgba]
    a, b = g.FrameStore(56, 40, [1, 1, 1], DEV), g.FrameStore(56, 40, [1, 1, 1], DEV)
    ia, ib = a.add_png(files, resize=True), b.add_png(files)
    for x, y in zip(a.decode(ia), b.decode(ib)):
        assert torch.equal(x, y)
    assert a.nbytes == b.nbytes and torch.equal(a.arena[:a._used], b.arena[:b._used])
    small = g.FrameStore(28, 20, [1, 1, 1], DEV)
    with pytest.raises(ValueError, match=re.escape("56x40, the store holds 28x20 frames (resize=True")):
        small.add_png(files)
    with pytest.raises(ValueError, match="one size per call"):
        small.add_png(files + [_png(RM._rgba(1, 20, 28, seed=1).numpy()[0], "RGBA")], resize=True)
    with pytest.raises(ValueError, match="uint8 \\(3, 20, 28\\)"):
        small.add_rgba(torch.from_numpy(rgba))
    ids = small.add_rgba(torch.from_numpy(rgba), resize=True)
    assert torch.equal(small.decode(ids)[0], g.composite_rgba(torch.from_numpy(rgba).to(DEV), [1, 1, 1],
                                                              size=(28, 20))[0])


# ---- the captured training iteration on a resized store -------------------------------------------------------------
def test_replay_on_a_resized_store_equals_the_eager_iteration(monkeypatch):
    g = _g()
    sc, _ = RM._single_view_setup()
    W, H = sc["W"], sc["H"]
    pc = TG._trainable(sc)
    store = g.FrameStore(W, H, sc["bg"], DEV)
    rgba = RM._rgba(2, H * 5 // 3 + 1, W * 7 // 4 + 3, seed=90)
    store.add_rgba(rgba, resize=True)
    fr = RM._single_frame(pc, sc, frames=store, lambda_mask=LAM)
    fr.set_inputs(frames=1)
    pc.optimizer.init_state()
    snap = TG._snapshot(pc)
    fr.capture()
    fr.run(check=True)
    torch.cuda.synchronize()
    want_gt, want_mask = g.composite_rgba(rgba[1].to(DEV), sc["bg"].to(DEV), size=(W, H))
    assert torch.equal(fr.gt, want_gt) and torch.equal(fr.mask, want_mask)
    # the eager iteration, its frame composited and resized as the store's was
    monkeypatch.setattr(g, "composite_rgba", functools.partial(g.composite_rgba, size=(W, H)))
    img, alpha, loss, pc_e = RM._eager_mask_iteration_single(sc, snap, sc["verts"], rgba[1].to(DEV),
                                                             pc.active_sh_degree)
    assert torch.equal(fr.image, img) and torch.equal(fr.alpha, alpha)
    assert abs(float(fr.loss) - loss) <= 1e-6 * loss
    TG._grads_close([p.grad for p in pc.parameters()], [p.grad for p in pc_e.parameters()])
    RM._check_step_exact(fr, pc, snap, "resized store replay")
    assert fr.captures == 1
