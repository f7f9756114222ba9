"""CPU: the K-view mesh overlay's C ABI (gab200_mesh_render_views, gab200_mesh_views_scratch_bytes: export, signature,
every refusal before any device work), the checks of mesh_overlay_views and of the graph constructors that draw it,
and the state key of a K-view GraphedRender / a GraphedEval with the mesh -- no compute calls (no GPU)."""
import ctypes as C
import os
import re

import pytest
import torch

from gaussianavatars_b200 import _native as N
from tests.test_host_mesh import BAD, _args, _mesh_render, _no_device  # noqa: F401  (_no_device: a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 0x10000


def _declaration(name):
    hdr = open(os.path.join(ROOT, "include", "gab200_rasterizer.h")).read()
    m = re.search(r"(\w+) " + name + r"\(([^)]*)\);", hdr)
    assert m, f"{name} is not declared in the header"
    return m.group(1), [" ".join(p.split()) for p in m.group(2).split(",")]


def test_the_two_entry_points_are_exported_with_the_header_signatures():
    L = N.lib()
    for s in ("gab200_mesh_render_views", "gab200_mesh_views_scratch_bytes"):
        assert s in N.EXPORTED_SYMBOLS and hasattr(L, s)
    assert _declaration("gab200_mesh_render_views") == \
        ("int32_t", ["const gab200_mesh_args* args", "int32_t views", "void* stream"])
    assert _declaration("gab200_mesh_views_scratch_bytes") == \
        ("size_t", ["int32_t views", "int32_t num_faces", "int32_t width", "int32_t height"])
    f = L.gab200_mesh_render_views
    assert f.restype is C.c_int32 and f.argtypes == [C.POINTER(N.MeshArgs), C.c_int32, C.c_void_p]
    g = L.gab200_mesh_views_scratch_bytes
    assert g.restype is C.c_size_t and g.argtypes == [C.c_int32] * 4
    assert L.gab200_abi_version() == N.ABI_VERSION == 3   # new entry points, the argument struct is unchanged


VIEWS_BAD = {
    "clip_space": dict(pos_kind=N.MESH_POS_CLIP), "out_rgba": dict(out_rgba=FAKE), "out_float": dict(out_float=FAKE),
    "out_rast": dict(out_rast=FAKE), "in_rast": dict(in_rast=FAKE), "in_color": dict(in_color=FAKE, channels=4),
    "out_color": dict(out_color=FAKE, in_color=FAKE, channels=4), "no_out_u8": dict(out_u8=None, out_rgba=FAKE),
    "no_base": dict(base=None), "no_opacity": dict(opacity=None), "base_none_kind": dict(base_kind=N.MESH_BASE_NONE),
}


@pytest.mark.parametrize("name", sorted(VIEWS_BAD) + [f"single:{n}" for n in sorted(BAD)])
def test_invalid_arguments_are_refused_before_any_device_work(name):
    L = N.lib()
    kw = BAD[name[7:]] if name.startswith("single:") else VIEWS_BAD[name]
    launches = L.gab200_launch_count()
    for views in (1, 4):
        assert L.gab200_mesh_render_views(C.byref(_args(**kw)), views, None) == -1
    assert L.gab200_launch_count() == launches


@pytest.mark.parametrize("views", [0, -1, N.MAX_VIEWS + 1])
def test_views_outside_the_range_are_refused(views):
    L = N.lib()
    assert L.gab200_mesh_render_views(C.byref(_args()), views, None) == -1
    assert L.gab200_mesh_views_scratch_bytes(views, 100, 64, 48) == 0
    assert L.gab200_mesh_render_views(None, 1, None) == -1


def test_too_many_face_records_are_refused():
    L = N.lib()
    F = (2**31 - 1) // 3 + 1
    assert L.gab200_mesh_render_views(C.byref(_args(F=F)), 3, None) == -1
    assert L.gab200_mesh_views_scratch_bytes(3, F, 64, 48) == 0


def test_valid_arguments_pass_validation_and_scratch_is_k_views_of_one():
    L = N.lib()
    launches = L.gab200_launch_count()
    if not torch.cuda.is_available():   # validated, then refused for want of an sm_90 device: nothing launched
        for views in (1, 2, 16, N.MAX_VIEWS):
            assert L.gab200_mesh_render_views(C.byref(_args()), views, None) == -4
        assert L.gab200_mesh_render_views(C.byref(_args(lighting=N.MESH_LIGHT_CONSTANT, antialias=0,
                                                          adjacency=None, face_colors=FAKE,
                                                          base_kind=N.MESH_BASE_FLOAT_CHW, error_flag=FAKE)),
                                          3, None) == -4
    assert L.gab200_launch_count() == launches
    one = L.gab200_mesh_scratch_bytes(100, 64, 48)
    assert L.gab200_mesh_views_scratch_bytes(1, 100, 64, 48) == one
    s4 = L.gab200_mesh_views_scratch_bytes(4, 100, 64, 48)
    assert s4 % 256 == 0 and s4 >= 4 * (8 * 64 * 48 + 304 * 100)
    assert L.gab200_mesh_views_scratch_bytes(4, 100, 64, 96) > s4
    assert L.gab200_mesh_views_scratch_bytes(4, 0, 64, 48) == 0
    assert L.gab200_mesh_views_scratch_bytes(4, 100, 16385, 48) == 0
    # the header's figure: 16 views of the 9,996-face head at 1080p
    big = L.gab200_mesh_views_scratch_bytes(16, 9996, 1920, 1080)
    assert 300e6 < big < 330e6


def test_mesh_overlay_views_checks_its_arguments():
    from gaussianavatars_b200 import mesh_overlay_views
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.renderer import camera_table

    cams = [syn.orbit_camera(32, 24, azimuth_deg=a) for a in (0.0, 30.0)]
    v, f = torch.zeros(5, 3), torch.tensor([[0, 1, 2]])
    base = torch.zeros(2, 3, 24, 32, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="no CPU path"):           # every check passed, then the device one
        mesh_overlay_views(v, f, cams, base)
    with pytest.raises(RuntimeError, match="no CPU path"):
        mesh_overlay_views(v, f, camera_table(cams, "cpu"), base.float())
    for bad in (torch.zeros(3, 24, 32), torch.zeros(2, 4, 24, 32), torch.zeros(2, 3, 24, 32, dtype=torch.float64),
                torch.zeros(2, 3, 24, 32, dtype=torch.int32)):
        with pytest.raises(ValueError, match=r"base must be \(K,3,H,W\) float32 or uint8"):
            mesh_overlay_views(v, f, cams, bad)
    with pytest.raises(ValueError, match="base holds 1"):
        mesh_overlay_views(v, f, [], torch.zeros(0, 3, 24, 32))
    with pytest.raises(ValueError, match="image size"):
        mesh_overlay_views(v, f, cams, torch.zeros(2, 3, 24, 16385))
    with pytest.raises(ValueError, match="1 cameras for 2 base planes"):
        mesh_overlay_views(v, f, cams[:1], base)
    with pytest.raises(ValueError, match="a camera is 32x24, base is 32x20"):
        mesh_overlay_views(v, f, cams, torch.zeros(2, 3, 20, 32))
    for table in (camera_table(cams, "cpu")[:1], camera_table(cams, "cpu")[:, :35], camera_table(cams, "cpu").double()):
        with pytest.raises(ValueError, match="camera table of 2 views"):
            mesh_overlay_views(v, f, table, base)
    with pytest.raises(ValueError, match="one mesh per call"):
        mesh_overlay_views(torch.zeros(2, 5, 3), f, cams, base)


# ---- the graphs, with the capture stubbed out (no device, no graph) -----------------------------------------------
def _model(P=4):
    from types import SimpleNamespace
    names = ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest")
    pc = SimpleNamespace(active_sh_degree=0, binding=torch.zeros(P, dtype=torch.int32), verts_rest=torch.zeros(5, 3),
                         faces=torch.tensor([[0, 1, 2], [2, 1, 3], [0, 2, 4]]))
    for n in names:
        setattr(pc, n, torch.nn.Parameter(torch.zeros(P, 3)))
    pc.parameters = lambda: [getattr(pc, n) for n in names]
    return pc


def _captured(fr):
    fr._learn_capacity = lambda: (0, (0, 0))
    fr._body = lambda *a, **k: None
    return fr.capture()


def test_graph_constructors_accept_k_views_with_the_mesh_and_check_it(_no_device):
    from gaussianavatars_b200.graph import GraphedEval, GraphedRender
    pc = _model()
    view = GraphedRender(pc, 64, 48, torch.zeros(3), views_per_replay=3, mesh_opacity=0.5)
    assert view.K == 3 and view.mesh and view.cam.shape == (3, 37)
    with pytest.raises(ValueError, match="outputs 'u8' or 'both'"):
        GraphedRender(pc, 64, 48, torch.zeros(3), views_per_replay=3, mesh_opacity=0.5, outputs="float")
    with pytest.raises(ValueError, match="face_colors must be"):
        GraphedRender(pc, 64, 48, torch.zeros(3), views_per_replay=3, mesh_opacity=0.5, face_colors=torch.rand(4, 3))
    pc.faces = pc.faces.float()
    with pytest.raises(ValueError, match="integer faces"):
        GraphedRender(pc, 64, 48, torch.zeros(3), views_per_replay=3, mesh_opacity=0.5)
    pc.faces = pc.faces.long()
    with pytest.raises(ValueError, match="source='u8'"):
        GraphedEval(pc, 64, 48, torch.zeros(3), views=4, source="float", mesh_opacity=0.5)
    with pytest.raises(ValueError, match="mesh_lighting"):
        GraphedEval(pc, 64, 48, torch.zeros(3), views=4, source="u8", mesh_opacity=0.5, mesh_lighting="world")
    ev = GraphedEval(pc, 64, 48, torch.zeros(3), views=4, source="u8", views_per_replay=2, mesh_opacity=0.5)
    assert ev.mesh and ev.outputs == "u8" and ev.mesh_display is None
    with pytest.raises(ValueError, match=r"gt_u8 must be a uint8 \(2, 3, 48, 64\)"):
        ev.set_inputs(gt_u8=torch.zeros(2, 3, 48, 64))
    with pytest.raises(ValueError, match="host_mesh_png needs"):
        GraphedEval(pc, 64, 48, torch.zeros(3), views=4, source="u8", png=True).host_mesh_png()
    with pytest.raises(ValueError, match="built with mesh_opacity"):
        GraphedEval(pc, 64, 48, torch.zeros(3), views=4, source="u8").set_inputs(mesh_opacity=0.5)


def test_k_view_mesh_inputs_never_recapture_and_the_key_follows_the_mesh(_no_device):
    from gaussianavatars_b200.graph import GraphedEval, GraphedRender
    for make in (lambda pc: GraphedRender(pc, 64, 48, torch.zeros(3), views_per_replay=3, mesh_opacity=0.5),
                 lambda pc: GraphedEval(pc, 64, 48, torch.zeros(3), views=6, source="u8", views_per_replay=3,
                                        mesh_opacity=0.5)):
        pc = _model()
        fr = _captured(make(pc))
        assert not fr._stale()
        fr.set_inputs(mesh_opacity=0.25)
        assert not fr._stale() and torch.equal(fr._opacity, torch.tensor([0.25, 0.75]))
        fr.set_inputs(face_colors=torch.rand(3, 3))     # a colour buffer the capture did not have
        assert fr._stale()
        fr.capture()
        fr.set_inputs(face_colors=torch.rand(1, 3, 3))  # written into that buffer
        assert not fr._stale()
        pc.faces[0, 0] = 3                               # topology edited in place: the adjacency is rebuilt
        assert fr._stale()
        fr.capture()
        pc.faces = pc.faces.clone()                      # a new faces tensor
        assert fr._stale()
        fr.capture()
        fr.mesh_lighting = "constant"                    # the lighting is baked into the launch
        assert fr._stale()


def test_a_plain_eval_key_has_no_mesh_entries(_no_device):
    from gaussianavatars_b200.graph import GraphedEval
    pc = _model()
    plain = _captured(GraphedEval(pc, 64, 48, torch.zeros(3), views=2, source="u8"))
    pc.faces = pc.faces.clone()
    assert not plain._stale()


def test_the_sweep_parses_and_plans_without_a_device():
    import importlib.util
    spec = importlib.util.spec_from_file_location("mesh_views_sweep", os.path.join(ROOT, "scripts", "mesh_views_sweep.py"))
    sweep = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sweep)
    a = sweep.parse(["--sizes", "64x48,32x24", "--ks", "1,2", "--eval-ks", "1,2", "--records", "4", "--splats", "1000"])
    assert a.sizes == [(64, 48), (32, 24)] and a.ks == [1, 2] and a.records == 4
    plans = list(sweep.plan(a))
    assert [p["plan"] for p in plans] == ["64x48", "32x24"]
    L = N.lib()
    assert plans[0]["mesh_views_scratch_bytes"] == {k: L.gab200_mesh_views_scratch_bytes(k, 9996, 64, 48) for k in (1, 2)}
    with pytest.raises(SystemExit):
        sweep.parse(["--records", "5", "--eval-ks", "4"])
    with pytest.raises(SystemExit):
        sweep.parse(["--ks", "0"])
