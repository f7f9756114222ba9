"""CPU: the evaluation surface -- the gab200_image_metrics entry points (exports, ctypes signatures against the header,
argument checks that reject before any device work, the scratch size), the input checks of image_metrics and the
host-side behaviour of GraphedEval (its checks, the NaN table, how scores() forms the means) -- no GPU."""
import ctypes as C
import math
import os
import re
from types import SimpleNamespace

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DUMMY = 0x1000   # never dereferenced: every call below is rejected during argument validation


def _hdr():
    return open(os.path.join(ROOT, "include", "gab200_rasterizer.h")).read()


def test_metrics_entry_points_are_exported_with_the_header_signatures():
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    for s in ("gab200_image_metrics", "gab200_image_metrics_scratch_bytes"):
        assert s in N.EXPORTED_SYMBOLS and hasattr(L, s)
    assert L.gab200_abi_version() == N.ABI_VERSION == 3
    assert L.gab200_image_metrics.restype is C.c_int32
    assert L.gab200_image_metrics.argtypes == [C.POINTER(N.MetricsArgs), C.c_void_p]
    assert L.gab200_image_metrics_scratch_bytes.restype is C.c_size_t
    assert L.gab200_image_metrics_scratch_bytes.argtypes == [C.c_int32, C.c_int32]
    hdr = _hdr()
    m = re.search(r"int32_t gab200_image_metrics\(([^)]*)\);", hdr)
    assert m and [p.strip() for p in m.group(1).split(",")] == ["const gab200_metrics_args* args", "void* stream"]
    m = re.search(r"size_t gab200_image_metrics_scratch_bytes\(([^)]*)\);", hdr)
    assert m and [p.strip() for p in m.group(1).split(",")] == ["int32_t height", "int32_t width"]
    assert re.search(r"#define GAB200_METRICS_FIELDS (\d+)", hdr).group(1) == str(N.METRICS_FIELDS) == "4"
    assert re.search(r"GAB200_METRICS_FLOAT_CHW = (\d+)", hdr).group(1) == str(N.METRICS_FLOAT_CHW)
    assert re.search(r"GAB200_METRICS_U8_HWC = (\d+)", hdr).group(1) == str(N.METRICS_U8_HWC)


def test_metrics_args_mirror_the_header_struct():
    from gaussianavatars_b200 import _native as N

    body = re.search(r"typedef struct gab200_metrics_args \{(.*?)\} gab200_metrics_args;", _hdr(), re.S).group(1)
    names = []
    for line in body.splitlines():
        decl = line.split("/*")[0].strip().rstrip(";")
        if decl:
            names += [n.strip().lstrip("*") for n in decl.split(None, 1)[1].split(",")] if " " in decl else []
    names = [n.split()[-1].lstrip("*") for n in names]
    assert names == [f for f, _ in N.MetricsArgs._fields_]
    assert C.sizeof(N.MetricsArgs) == 72


def test_scratch_size_is_three_doubles_per_channel_and_tile():
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    assert L.gab200_image_metrics_scratch_bytes(45, 70) == 2 * 3 * 3 * 3 * 8     # 2 x 3 tiles of 32 x 32
    assert L.gab200_image_metrics_scratch_bytes(1080, 1920) == 34 * 60 * 3 * 3 * 8
    assert L.gab200_image_metrics_scratch_bytes(0, 70) == 0 and L.gab200_image_metrics_scratch_bytes(45, -1) == 0


def _args(**kw):
    from gaussianavatars_b200 import _native as N

    a = N.MetricsArgs()
    a.abi_version, a.height, a.width, a.render_kind = N.ABI_VERSION, 17, 33, N.METRICS_FLOAT_CHW
    a.render = a.gt = a.table = a.scratch = DUMMY
    a.table_rows = 4
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("bad", [
    dict(render=None), dict(gt=None), dict(table=None), dict(scratch=None), dict(scratch=DUMMY + 4),
    dict(height=0), dict(width=0), dict(height=-3), dict(table_rows=0), dict(table_rows=-1),
    dict(render_kind=2), dict(render_kind=-1), dict(abi_version=2),
], ids=lambda d: "-".join(f"{k}={v}" for k, v in d.items()))
def test_image_metrics_rejects_invalid_arguments(bad):
    from gaussianavatars_b200 import _native as N

    assert N.lib().gab200_image_metrics(C.byref(_args(**bad)), None) == -1
    assert N.lib().gab200_image_metrics(None, None) == -1


def test_image_metrics_checks_its_inputs():
    from gaussianavatars_b200.training import image_metrics

    gt = torch.zeros((3, 17, 33), dtype=torch.uint8)
    for render, err in ((torch.zeros((3, 17, 33), dtype=torch.float64), TypeError),   # not float32
                        (torch.zeros((4, 17, 33)), TypeError),                         # not 3 channels
                        (torch.zeros((17, 33, 3)), TypeError),                         # float HWC
                        (torch.zeros((3, 17, 33), dtype=torch.uint8), TypeError),      # uint8 CHW
                        (torch.zeros((1, 3, 17, 33)), TypeError)):
        with pytest.raises(err):
            image_metrics(render, gt)
    img = torch.zeros((3, 17, 33))
    with pytest.raises(TypeError, match="uint8"):
        image_metrics(img, gt.float())
    with pytest.raises(ValueError, match="shape"):
        image_metrics(img, torch.zeros((3, 17, 32), dtype=torch.uint8))
    with pytest.raises(ValueError, match="shape"):
        image_metrics(torch.zeros((17, 33, 3), dtype=torch.uint8), torch.zeros((3, 33, 17), dtype=torch.uint8))
    with pytest.raises(RuntimeError, match="CPU"):   # well-formed, but there is no CPU path
        image_metrics(img, gt)


def _pc():
    return SimpleNamespace(_xyz=torch.zeros(4, 3), verts_rest=torch.zeros(5, 3))


def test_graphed_eval_argument_checks():
    from gaussianavatars_b200.graph import GraphedEval
    from gaussianavatars_b200 import synthetic as syn

    with pytest.raises(ValueError, match="source"):
        GraphedEval(_pc(), 64, 48, torch.zeros(3), views=4, source="png")
    with pytest.raises(ValueError, match="host_slots"):
        GraphedEval(_pc(), 64, 48, torch.zeros(3), views=4, source="float", host_slots=2)
    with pytest.raises(ValueError, match="views"):
        GraphedEval(_pc(), 64, 48, torch.zeros(3), views=0)
    ev = GraphedEval(_pc(), 64, 48, torch.zeros(3), views=4, source="u8", host_slots=2)
    assert ev.outputs == "u8" and ev.table.shape == (4, 4) and torch.isnan(ev.table).all()
    assert ev.gt.shape == (3, 48, 64) and ev.gt.dtype == torch.uint8
    ev.set_inputs(view=3)
    assert int(ev.view) == 3
    for v in (4, -1):
        with pytest.raises(IndexError):
            ev.set_inputs(view=v)
    assert int(ev.view) == 3
    with pytest.raises(ValueError, match="gt_u8"):
        ev.set_inputs(gt_u8=torch.zeros((3, 48, 63), dtype=torch.uint8))
    with pytest.raises(ValueError, match="gt_u8"):
        ev.set_inputs(gt_u8=torch.zeros((48, 64, 3), dtype=torch.uint8))
    with pytest.raises(ValueError, match="gt_u8"):
        ev.set_inputs(gt_u8=torch.zeros((3, 48, 64)))
    gt = torch.randint(0, 256, (3, 48, 64), dtype=torch.uint8)
    ev.set_inputs(gt_u8=gt, view=1)
    assert torch.equal(ev.gt, gt) and int(ev.view) == 1
    # a camera of another size: the ground truth is checked against the NEW size and the buffer follows it
    cam = syn.orbit_camera(80, 60)
    with pytest.raises(ValueError, match="gt_u8"):
        ev.set_inputs(camera=cam, gt_u8=gt)
    gt2 = torch.randint(0, 256, (3, 60, 80), dtype=torch.uint8)
    ev.set_inputs(camera=cam, gt_u8=gt2)
    assert (ev.W, ev.H) == (80, 60) and torch.equal(ev.gt, gt2)


def test_scores_raise_on_missing_rows_and_form_training_report_means():
    from gaussianavatars_b200.graph import GraphedEval

    ev = GraphedEval(_pc(), 64, 48, torch.zeros(3), views=3)
    with pytest.raises(RuntimeError, match=r"rows \[0, 1, 2\].*regrow"):
        ev.scores()
    rows = torch.tensor([[0.1, 20.5, 20.25, 0.7], [0.2, 21.5, 21.0, 0.8], [0.3, math.inf, math.inf, 1.0]])
    ev.table[:2] = rows[:2]
    with pytest.raises(RuntimeError, match=r"rows \[2\]"):
        ev.scores()
    s = ev.scores(n=2)
    assert torch.equal(s["per_view"], rows[:2])
    r32 = rows[:2].tolist()
    assert s["l1"] == (0.0 + r32[0][0] + r32[1][0]) / 2     # the float32 values summed in double
    assert s["psnr"] == (r32[0][1] + r32[1][1]) / 2 and s["psnr_all"] == (r32[0][2] + r32[1][2]) / 2
    assert s["ssim"] == (r32[0][3] + r32[1][3]) / 2
    ev.table[2] = rows[2]
    assert ev.scores()["psnr"] == math.inf
    with pytest.raises(IndexError):
        ev.scores(n=4)
    ev.reset()
    assert torch.isnan(ev.table).all()
