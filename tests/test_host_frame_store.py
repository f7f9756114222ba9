"""CPU: the frame store's surface (gab200_frame_encode_plan / gab200_frame_encode / gab200_frame_decode, FrameStore,
GraphedFrame(frames=store)) -- the exports, the header declarations, the C ABI's argument refusals, every Python
refusal, and what makes a frame that reads a store re-capture.  No device: the GraphedFrame tests stub the capture
as tests/test_host_graph_keys.py does, and the store is a host stand-in with the attributes a frame reads."""
import contextlib
import ctypes as C
import os
import re
from types import SimpleNamespace

import pytest
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
PARAMS = ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest")
W, H = 40, 24
SIGNATURES = {
    "gab200_frame_encode_plan": ["frames", "height", "width", "gt", "mask", "record_units", "stream"],
    "gab200_frame_encode": ["frames", "height", "width", "gt", "mask", "frame_base", "tile_off", "arena", "stream"],
    "gab200_frame_decode": ["views", "height", "width", "ids", "arena", "frame_base", "tile_off", "gt_out", "mask_out",
                            "stream"],
}


def test_exported_and_declared():
    import gaussianavatars_b200 as g
    from gaussianavatars_b200 import _native as N
    L = N.lib()
    hdr = open(os.path.join(ROOT, "include", "gab200_rasterizer.h")).read()
    for name, params in SIGNATURES.items():
        assert name in N.EXPORTED_SYMBOLS and hasattr(L, name)
        decl = re.search(r"int32_t " + name + r"\(([^)]*)\);", hdr)
        assert decl is not None, name
        assert [p.split()[-1].lstrip("*") for p in decl.group(1).split(",")] == params, name
        assert len(getattr(L, name).argtypes) == len(params)
    assert "FrameStore" in g.__all__ and g.FrameStore.__module__ == "gaussianavatars_b200.frames"
    assert L.gab200_abi_version() == 3


def test_c_abi_refusals_before_any_device_work():
    from gaussianavatars_b200 import _native as N
    L = N.lib()
    buf = (C.c_uint8 * 256)()
    p = C.cast(buf, C.c_void_p)
    invalid = -1
    # plan: frames, height, width, gt, mask, record_units
    assert L.gab200_frame_encode_plan(-1, 2, 2, p, None, p, None) == invalid
    assert L.gab200_frame_encode_plan(1, -2, 2, p, None, p, None) == invalid
    assert L.gab200_frame_encode_plan(1, 2, -2, p, None, p, None) == invalid
    assert L.gab200_frame_encode_plan(1, 2, 2, None, p, p, None) == invalid    # no ground truth (a mask alone is not one)
    assert L.gab200_frame_encode_plan(1, 2, 2, p, None, None, None) == invalid  # nowhere to write the sizes
    # encode: ... frame_base, tile_off, arena
    assert L.gab200_frame_encode(-1, 2, 2, p, None, p, p, p, None) == invalid
    assert L.gab200_frame_encode(1, 2, -2, p, None, p, p, p, None) == invalid
    for k in range(3):   # frame_base, tile_off or arena missing
        args = [p, p, p]
        args[k] = None
        assert L.gab200_frame_encode(1, 2, 2, p, None, *args, None) == invalid
    assert L.gab200_frame_encode(1, 2, 2, None, None, p, p, p, None) == invalid
    # decode: views, height, width, ids, arena, frame_base, tile_off, gt_out, mask_out
    assert L.gab200_frame_decode(-1, 2, 2, p, p, p, p, p, None, None) == invalid
    assert L.gab200_frame_decode(1, -2, 2, p, p, p, p, p, None, None) == invalid
    assert L.gab200_frame_decode(1, 2, -2, p, p, p, p, p, None, None) == invalid
    for k in range(5):   # ids, arena, frame_base, tile_off or gt_out missing (the mask alone is not an output)
        args = [p, p, p, p, p]
        args[k] = None
        assert L.gab200_frame_decode(1, 2, 2, *args, p, None) == invalid


def test_frame_store_construction_refusals():
    import gaussianavatars_b200 as g
    with pytest.raises(ValueError, match="positive size"):
        g.FrameStore(0, 8, [0, 0, 0], "cuda:0")
    with pytest.raises(ValueError, match="positive size"):
        g.FrameStore(8, -1, [0, 0, 0], "cuda:0")
    with pytest.raises(ValueError, match="bg must hold 3 values"):
        g.FrameStore(8, 8, [0, 0], "cuda:0")
    with pytest.raises(RuntimeError, match="no CPU path"):
        g.FrameStore(8, 8, [0, 0, 0], "cpu")


# ---- a host stand-in of a store and a stubbed GraphedFrame ---------------------------------------------------------
def _store(n=3, bg=(0.0, 0.0, 0.0), w=W, h=H):
    from gaussianavatars_b200.frames import FrameStore, _tiles
    s = FrameStore.__new__(FrameStore)
    s.W, s.H, s.device, s.bg = w, h, torch.device("cpu"), torch.tensor(bg, dtype=torch.float32)
    s.n_tiles, s._n, s._used = _tiles(h, w), n, 8 * n
    s.arena = torch.zeros(64, dtype=torch.uint8)
    s.frame_base = torch.zeros(4, dtype=torch.int64)
    s.tile_off = torch.zeros(4 * s.n_tiles, dtype=torch.int32)
    return s


class _NoGraph:
    def replay(self):
        pass


@pytest.fixture()
def no_device(monkeypatch):
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", _NoGraph)
    monkeypatch.setattr(torch.cuda, "graph", lambda g: contextlib.nullcontext())


def _model(P=4):
    pc = SimpleNamespace(active_sh_degree=0, binding=torch.zeros(P, dtype=torch.int32), verts_rest=torch.zeros(5, 3))
    for n in PARAMS:
        setattr(pc, n, torch.nn.Parameter(torch.zeros(P, 3)))
    pc.parameters = lambda: [getattr(pc, n) for n in PARAMS]
    return pc


def _frame(store, K=1, **kw):
    from gaussianavatars_b200.graph import GraphedFrame
    fr = GraphedFrame(_model(), W, H, 0.7, 0.5, torch.zeros(3), frames=store, views_per_replay=K, **kw)
    fr._learn_capacity = lambda: (0, (0, 0))
    fr._body = lambda *a, **k: None
    return fr


def test_store_id_checks():
    s = _store(n=3)
    assert s.check_ids(2) == [2] and s.check_ids([0, 2, 0]) == [0, 2, 0]
    assert s.check_ids(torch.tensor([1, 1])) == [1, 1]
    for bad in (3, -1, [0, 3], [1.0], True, [None]):
        with pytest.raises(ValueError, match="frame ids index the store's 3 frames"):
            s.check_ids(bad)
    assert len(s) == 3 and s.raw_nbytes == 3 * 4 * W * H and s.nbytes == 24 + 3 * (8 + 4 * s.n_tiles)


def test_graphed_frame_refusals_without_a_model():
    from gaussianavatars_b200.graph import GraphedFrame
    bg = torch.zeros(3)
    with pytest.raises(ValueError, match="use one of them"):
        GraphedFrame(None, 8, 8, 1.0, 1.0, bg, rgba=True, frames=object())
    with pytest.raises(ValueError, match="loss='dL_dimage' reads none"):
        GraphedFrame(None, 8, 8, 1.0, 1.0, bg, loss="dL_dimage", frames=object())
    # a frame built without a store still needs rgba=True for the mask term
    with pytest.raises(ValueError, match="needs rgba=True"):
        GraphedFrame(None, 8, 8, 1.0, 1.0, bg, lambda_mask=0.1)


def test_graphed_frame_store_refusals(no_device):
    with pytest.raises(ValueError, match="must be a gaussianavatars_b200.FrameStore"):
        _frame(object())
    with pytest.raises(ValueError, match="the frame store holds 41x24 frames"):
        _frame(_store(w=W + 1))
    with pytest.raises(ValueError, match="the backgrounds must be equal"):
        _frame(_store(bg=(1.0, 1.0, 1.0)))
    with pytest.raises(ValueError, match="holds no frames"):
        _frame(_store(n=0))
    fr = _frame(_store(), lambda_mask=0.1)   # the store's mask feeds the mask term
    assert fr.mask.shape == (1, H, W) and fr.gt.shape == (3, H, W) and fr.gt_rgba is None and fr.gt_stage is None
    with pytest.raises(ValueError, match="give frames=, not gt_u8 / gt_rgba"):
        fr.set_inputs(gt_u8=torch.zeros(3, H, W, dtype=torch.uint8))
    with pytest.raises(ValueError, match="give frames=, not gt_u8 / gt_rgba"):
        fr.set_inputs(gt_rgba=torch.zeros(H, W, 4, dtype=torch.uint8))
    for bad in (3, -1, [0, 1], True):
        with pytest.raises(ValueError, match="frame ids|1 views per replay"):
            fr.set_inputs(frames=bad)
    fr.set_inputs(frames=2)
    assert fr.frame_ids.tolist() == [2]
    k4 = _frame(_store(), K=4)
    assert k4.frame_ids.shape == (4,) and k4.mask.shape == (4, 1, H, W)
    with pytest.raises(ValueError, match="give 4 frame ids"):
        k4.set_inputs(frames=1)
    with pytest.raises(ValueError, match="got 3 frame ids"):
        k4.set_inputs(frames=[0, 1, 2])
    with pytest.raises(ValueError, match="frame ids index"):
        k4.set_inputs(frames=[0, 1, 2, 3])
    k4.set_inputs(frames=[2, 0, 2, 1])
    assert k4.frame_ids.tolist() == [2, 0, 2, 1]
    with pytest.raises(ValueError, match="stage_frames needs"):
        k4.stage_frames([0, 0, 0, 0])
    from gaussianavatars_b200.graph import GraphedFrame
    plain = GraphedFrame(_model(), W, H, 0.7, 0.5, torch.zeros(3))
    with pytest.raises(ValueError, match="needs a GraphedFrame built with frames=store"):
        plain.set_inputs(frames=0)


def test_prefetching_pair_must_agree_on_the_store(no_device, monkeypatch):
    from gaussianavatars_b200.graph import GraphedFrame
    monkeypatch.setattr(torch.cuda, "Stream", lambda device=None: None)
    a = _frame(_store(), host_inputs=True)
    b = GraphedFrame(_model(), W, H, 0.7, 0.5, torch.zeros(3), host_inputs=True)
    assert a.frames_stage.shape == (1,) and a.frames_stage.dtype == torch.int32 and b.frames_stage is None
    with pytest.raises(ValueError, match="frames= on both or on neither"):
        a.prefetch_for(b)
    with pytest.raises(ValueError, match="frames= on both or on neither"):
        b.prefetch_for(a)
    a.stage_frames(2)
    assert a.frames_stage.tolist() == [2]
    with pytest.raises(ValueError, match="frame ids index"):
        a.stage_frames(3)


def test_ids_never_recapture_and_a_grown_store_does(no_device):
    s = _store()
    fr = _frame(s)
    fr.run()
    assert fr.captures == 1
    for i in (0, 2, 1):
        fr.set_inputs(frames=i)
        fr.run()
    assert fr.captures == 1
    s._n += 1   # frames added into the store's spare room: nothing moved
    fr.run()
    assert fr.captures == 1
    s.arena = torch.zeros(128, dtype=torch.uint8)   # the arena grew (reallocated)
    fr.run()
    assert fr.captures == 2
    s.tile_off = torch.zeros(8 * s.n_tiles, dtype=torch.int32)   # the index grew
    fr.run()
    fr.run()
    assert fr.captures == 3
