"""CPU: the mesh overlay's C ABI (struct layout against gcc, argument validation before any device work), the Python
surface's input checks, and the nvdiffrast import shim resolving to this library -- no compute calls (no GPU)."""
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch

from gaussianavatars_b200 import _native as N

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
HEADER = os.path.join(ROOT, "include", "gab200_rasterizer.h")


def test_mesh_args_layout_matches_the_c_struct(tmp_path):
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{HEADER}"', "int main(){",
             'printf("size %zu\\n", sizeof(gab200_mesh_args));']
    for fname, _ in N.MeshArgs._fields_:
        lines.append(f'printf("{fname} %zu\\n", offsetof(gab200_mesh_args, {fname}));')
    lines.append("return 0;}")
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.run(["/usr/bin/gcc", str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
               if l.strip())
    assert int(got["size"]) == C.sizeof(N.MeshArgs)
    for fname, _ in N.MeshArgs._fields_:
        assert int(got[fname]) == getattr(N.MeshArgs, fname).offset, fname


def _args(**kw):
    """A well-formed POS_WORLD u8 composite request with fake (never dereferenced) device pointers."""
    a = N.MeshArgs()
    a.abi_version, a.V, a.F, a.width, a.height = N.ABI_VERSION, 10, 4, 64, 48
    a.pos_kind, a.lighting, a.antialias, a.base_kind = N.MESH_POS_WORLD, N.MESH_LIGHT_FRONT, 1, N.MESH_BASE_U8_CHW
    fake = 0x10000
    a.verts = a.faces = a.adjacency = a.camera = a.base = a.opacity = a.out_u8 = fake
    a.scratch = 0x20000
    for k, v in kw.items():
        setattr(a, k, v)
    return a


BAD = {
    "abi": dict(abi_version=N.ABI_VERSION + 1), "no_faces": dict(F=0), "neg_V": dict(V=0), "wide": dict(width=16385),
    "tall": dict(height=0), "no_verts": dict(verts=None), "no_scratch": dict(scratch=None),
    "unaligned_scratch": dict(scratch=0x20010), "pos_kind": dict(pos_kind=2), "lighting": dict(lighting=5),
    "base_kind": dict(base_kind=3), "aa_without_adjacency": dict(adjacency=None), "no_camera": dict(camera=None),
    "no_output": dict(out_u8=None), "composite_without_base": dict(base=None),
    "composite_without_opacity": dict(opacity=None), "composite_in_clip_space": dict(pos_kind=N.MESH_POS_CLIP),
    "color_without_input": dict(out_color=0x10000, channels=4), "too_many_channels":
        dict(out_color=0x10000, in_color=0x10000, channels=65),
}


@pytest.mark.parametrize("name", sorted(BAD))
def test_invalid_mesh_arguments_are_refused_before_any_device_work(name):
    L = N.lib()
    assert L.gab200_mesh_render(C.byref(_args(**BAD[name])), None) == -1
    assert L.gab200_mesh_render(None, None) == -1


def test_valid_arguments_pass_validation_and_scratch_is_a_pure_function_of_the_sizes():
    L = N.lib()
    launches = L.gab200_launch_count()
    if not torch.cuda.is_available():   # validated, then refused for want of an sm_90 device: nothing launched
        assert L.gab200_mesh_render(C.byref(_args()), None) == -4
    assert L.gab200_launch_count() == launches
    s = L.gab200_mesh_scratch_bytes(100, 64, 48)
    assert s > 0 and s % 256 == 0
    assert s == L.gab200_mesh_scratch_bytes(100, 64, 48)
    assert L.gab200_mesh_scratch_bytes(100, 64, 96) > s and L.gab200_mesh_scratch_bytes(200, 64, 48) > s
    assert L.gab200_mesh_scratch_bytes(0, 64, 48) == 0 and L.gab200_mesh_scratch_bytes(1, 16385, 1) == 0


def test_python_surface_checks_inputs():
    from gaussianavatars_b200 import MeshRenderer, mesh_overlay
    from gaussianavatars_b200 import synthetic as syn

    cam = syn.orbit_camera(32, 24)
    v = torch.zeros(5, 3)
    f = torch.tensor([[0, 1, 2]])
    base = torch.zeros(3, 24, 32)
    with pytest.raises(RuntimeError, match="no CPU path"):
        mesh_overlay(v, f, cam, base)
    with pytest.raises(ValueError, match="one mesh per call"):
        mesh_overlay(torch.zeros(2, 5, 3), f, cam, base)
    with pytest.raises(ValueError, match="out must be"):
        mesh_overlay(v, f, cam, base, out="png")
    with pytest.raises(NotImplementedError):
        MeshRenderer(lighting_type="world")


def test_nvdiffrast_shim_resolves_to_this_library_and_refuses_batches():
    code = ("import sys; sys.path.insert(0, %r)\n"
            "import nvdiffrast.torch as dr, torch\n"
            "print(dr.__file__)\n"
            "try:\n"
            "    dr.rasterize(dr.RasterizeCudaContext(), torch.zeros(2, 3, 4), torch.zeros(1, 3, dtype=torch.int32), (8, 8))\n"
            "except ValueError as e:\n"
            "    print('refused', e)\n") % os.path.join(ROOT, "gaussianavatars_b200", "compat")
    out = subprocess.run([sys.executable, "-c", code], check=True, capture_output=True, text=True, cwd="/").stdout
    assert os.path.join(ROOT, "gaussianavatars_b200", "compat", "nvdiffrast", "torch.py") in out
    assert "refused" in out and "one image per call" in out


# ---- GraphedRender(mesh_opacity=...): what re-captures, with the capture stubbed out (no device, no graph) ----------
@pytest.fixture
def _no_device(monkeypatch):
    import contextlib

    class _NoGraph:
        def replay(self):
            pass

    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", _NoGraph)
    monkeypatch.setattr(torch.cuda, "graph", lambda g: contextlib.nullcontext())


def _mesh_render(**kw):
    from types import SimpleNamespace

    from gaussianavatars_b200.graph import GraphedRender

    P = 4
    names = ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest")
    pc = SimpleNamespace(active_sh_degree=0, binding=torch.zeros(P, dtype=torch.int32), verts_rest=torch.zeros(5, 3),
                         faces=torch.tensor([[0, 1, 2], [2, 1, 3], [0, 2, 4]]))
    for n in names:
        setattr(pc, n, torch.nn.Parameter(torch.zeros(P, 3)))
    pc.parameters = lambda: [getattr(pc, n) for n in names]
    fr = GraphedRender(pc, 64, 48, torch.zeros(3), **kw)
    fr._learn_capacity = lambda: (0, (0, 0))
    fr._body = lambda *a, **k: None
    return fr.capture()


def test_mesh_opacity_and_face_colours_never_recapture(_no_device):
    fr = _mesh_render(mesh_opacity=0.5, face_colors=torch.rand(3, 3))
    fr.set_inputs(mesh_opacity=0.3, face_colors=torch.rand(1, 3, 3))
    assert not fr._stale()
    assert torch.equal(fr._opacity, torch.tensor([0.3, 0.7], dtype=torch.float32))


def test_mesh_state_key_follows_faces_and_the_colour_buffer(_no_device):
    fr = _mesh_render(mesh_opacity=0.5)
    assert not fr._stale()
    fr.set_inputs(face_colors=torch.rand(3, 3))       # a colour buffer the capture did not have
    assert fr._stale()
    fr.capture()
    fr.pc.faces[0, 0] = 3                              # topology edited in place: the adjacency is rebuilt
    assert fr._stale()
    fr.capture()
    fr.pc.faces = fr.pc.faces.clone()                  # a new faces tensor
    assert fr._stale()


def test_mesh_overlay_arguments_are_checked(_no_device):
    with pytest.raises(ValueError, match="outputs 'u8' or 'both'"):
        _mesh_render(mesh_opacity=0.5, outputs="float")
    with pytest.raises(ValueError, match="mesh_lighting"):
        _mesh_render(mesh_opacity=0.5, mesh_lighting="world")
    with pytest.raises(ValueError, match="face_colors must be"):
        _mesh_render(mesh_opacity=0.5, face_colors=torch.rand(4, 3))
    with pytest.raises(ValueError, match="built with mesh_opacity"):
        _mesh_render().set_inputs(mesh_opacity=0.5)
