"""CPU: the FLAME operator's yardstick and host surface -- the torch restatement (tests/flame_oracle.py) against the
fixture generated from the real reference (tests/golden/make_golden_flame.py), the new C ABI (exports, struct layouts,
argument checks), the Python argument checks, the reference's FLAME optimizer groups, and the synthetic assets."""
import ctypes as C
import os
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests import flame_oracle as fo
from tests import ref_import

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
HEADER = os.path.join(ROOT, "include", "gab200_rasterizer.h")
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "flame_vectors.npz"))
ASSET_KEYS = ("v_template", "shapedirs", "posedirs", "J_regressor", "lbs_weights")


def _gold_assets(dtype):
    a = {k: torch.tensor(GOLD[k], dtype=dtype) for k in ASSET_KEYS}
    a["parents"] = GOLD["parents"].tolist()
    return a


def _gold_params(dtype, requires_grad=False):
    p = {k[len("param_"):]: torch.tensor(GOLD[k], dtype=dtype) for k in GOLD.files if k.startswith("param_")}
    for k in fo.POSED:
        p[k].requires_grad_(requires_grad)
    return p


def test_oracle_matches_the_reference_fixture_in_float64():
    a = _gold_assets(torch.float64)
    T = GOLD["verts"].shape[0]
    worst = 0.0
    for t in range(T):
        p = _gold_params(torch.float64, requires_grad=True)
        verts, cano, joints = fo.select_mesh_by_timestep(a, p, t)
        (verts * torch.tensor(GOLD["C"][t][None])).sum().backward()
        for got, name in ((verts[0], "verts"), (cano[0], "verts_cano"), (joints[0], "joints")):
            ref = GOLD[name][t]
            err = float(np.abs(got.detach().numpy() - ref).max() / np.abs(ref).max())
            worst = max(worst, err)
            assert err <= 1e-12, (t, name, err)
        for k in fo.POSED:
            ref = GOLD[f"grad_{k}"][t]
            g = p[k].grad.numpy()
            assert np.abs(g - ref).max() <= 1e-12 * np.abs(ref).max(), (t, k)
            assert not np.delete(g, t, axis=0).any(), "rows other than the timestep's must be exactly zero"
    print(f"oracle vs reference fixture: worst relative error {worst:.2e}")


def test_rodrigues_as_written_is_exactly_identity_at_zero_with_a_finite_gradient():
    r = torch.zeros(1, 3, dtype=torch.float64, requires_grad=True)
    R = fo.batch_rodrigues(r)
    assert torch.equal(R.detach(), torch.eye(3, dtype=torch.float64)[None])
    (R * torch.arange(9, dtype=torch.float64).view(1, 3, 3)).sum().backward()
    assert torch.isfinite(r.grad).all() and r.grad.abs().max() > 0


def test_new_entry_points_are_exported_and_abi_version_is_unchanged():
    from gaussianavatars_b200 import _native as N

    lib = N.lib()
    for s in ("gab200_flame_scratch_bytes", "gab200_flame_prepare", "gab200_flame_forward", "gab200_flame_backward"):
        assert s in N.EXPORTED_SYMBOLS and hasattr(lib, s)
    assert lib.gab200_abi_version() == N.ABI_VERSION == 3
    # the prepared constants: v_base, the expression basis, J_base, JS and the backward's partials, 256-B carved
    V, NE = 5000, 100
    assert lib.gab200_flame_scratch_bytes(V, NE) >= 4 * (3 * V + NE * 3 * V + 15 + 15 * NE)
    assert lib.gab200_flame_scratch_bytes(V, NE) % 256 == 0


@pytest.mark.parametrize("name", ["FlameAssets", "FlameFrameArgs", "FlameGrads"])
def test_flame_struct_mirrors_match_the_c_layout(tmp_path, name):
    from gaussianavatars_b200 import _native as N

    ct = getattr(N, name)
    cname = {"FlameAssets": "gab200_flame_assets", "FlameFrameArgs": "gab200_flame_frame_args",
             "FlameGrads": "gab200_flame_grads"}[name]
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{HEADER}"', "int main(){",
             f'printf("{cname} %zu\\n", sizeof({cname}));']
    lines += [f'printf("{cname}.{f} %zu\\n", offsetof({cname}, {f}));' for f, _ in ct._fields_]
    lines += [f'printf("consts %d %d %d %d\\n", GAB200_FLAME_J, GAB200_FLAME_POSE_BASIS, GAB200_FLAME_MAX_EXPR, '
              f'GAB200_FLAME_FRAME_FLOATS);', "return 0;}"]
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.run(["/usr/bin/gcc", str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {l.split()[0]: l.split()[1:] for l in out if l.strip()}
    assert int(got[cname][0]) == C.sizeof(ct)
    for f, _ in ct._fields_:
        assert int(got[f"{cname}.{f}"][0]) == getattr(ct, f).offset, f
    assert [int(x) for x in got["consts"]] == [N.FLAME_J, N.FLAME_POSE_BASIS, N.FLAME_MAX_EXPR, N.FLAME_FRAME_FLOATS]


def _assets_struct(**over):
    from gaussianavatars_b200 import _native as N

    a = N.FlameAssets()
    a.abi_version, a.V, a.n_shape, a.n_expr, a.J = N.ABI_VERSION, 64, 300, 100, 5
    for i, p in enumerate([-1, 0, 1, 1, 1]):
        a.parents[i] = p
    a.v_template = a.shapedirs = a.posedirs = a.J_regressor = a.lbs_weights = 256
    for k, v in over.items():
        if k == "parents":
            for i, p in enumerate(v):
                a.parents[i] = p
        else:
            setattr(a, k, v)
    return a


def test_the_c_abi_rejects_other_skeletons_and_bad_arguments_before_any_launch():
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    shape = C.c_void_p(256)
    for bad in (dict(J=4), dict(J=6), dict(parents=[0, 0, 1, 1, 1]), dict(parents=[-1, 0, 2, 1, 1]),
                dict(parents=[-1, 0, 1, 4, 1]), dict(n_expr=101), dict(n_expr=-1), dict(V=0), dict(abi_version=2),
                dict(posedirs=None)):
        a = _assets_struct(**bad)
        assert L.gab200_flame_prepare(C.byref(a), shape, None, C.c_void_p(256), None) == -1, bad
    a = _assets_struct()
    assert L.gab200_flame_prepare(C.byref(a), shape, None, C.c_void_p(257), None) == -1   # scratch not 256-B aligned
    assert L.gab200_flame_prepare(C.byref(a), None, None, C.c_void_p(256), None) == -1    # n_shape > 0 needs shape
    g = N.FlameFrameArgs()
    g.abi_version, g.T, g.assets, g.scratch = N.ABI_VERSION, 4, C.pointer(a), 256
    assert L.gab200_flame_forward(C.byref(g), C.c_void_p(256), None, None) == -1             # no timestep / params
    grads = N.FlameGrads()
    assert L.gab200_flame_backward(C.byref(g), C.c_void_p(256), None, C.byref(grads), None) == -1
    assert L.gab200_flame_forward(None, None, None, None) == -1


def _small_arrays(V=64, n_shape=300, n_expr=100, J=5):
    return dict(v_template=torch.zeros(V, 3), shapedirs=torch.zeros(V, 3, n_shape + n_expr),
                posedirs=torch.zeros(36, 3 * V), J_regressor=torch.zeros(J, V), parents=[-1, 0, 1, 1, 1][:J] + [1] * (J - 5),
                lbs_weights=torch.zeros(V, J), faces=torch.zeros(4, 3, dtype=torch.long), n_shape=n_shape, n_expr=n_expr)


def test_flame_lbs_rejects_what_is_not_flame_before_touching_a_device():
    from gaussianavatars_b200.flame import FlameLBS

    with pytest.raises(ValueError, match="5 joints"):
        FlameLBS.from_arrays(**_small_arrays(J=4))
    with pytest.raises(ValueError, match="5 joints"):
        FlameLBS.from_arrays(**_small_arrays(J=6))
    for parents in ([0, 0, 1, 1, 1], [-1, 0, 3, 1, 1], [-1, 1, 1, 1, 1]):
        kw = _small_arrays()
        kw["parents"] = parents
        with pytest.raises(ValueError, match="topologically"):
            FlameLBS.from_arrays(**kw)
    kw = _small_arrays()
    kw["n_expr"] = 50                      # shapedirs carries 300 + 100 components
    with pytest.raises(ValueError, match="shapedirs"):
        FlameLBS.from_arrays(**kw)
    with pytest.raises(ValueError, match="n_expr"):
        FlameLBS.from_arrays(**_small_arrays(n_expr=120))
    with pytest.raises(RuntimeError, match="no CPU path"):
        FlameLBS.from_arrays(**_small_arrays(), device="cpu")


def test_timesteps_are_checked_on_the_host():
    from gaussianavatars_b200.flame import timestep_tensor
    from gaussianavatars_b200.graph import GraphedFrame

    for t in (-1, 4, 100):
        with pytest.raises(IndexError):
            timestep_tensor(t, 4, torch.device("cpu"))
    with pytest.raises(TypeError):
        timestep_tensor(torch.zeros(1, dtype=torch.int64), 4, torch.device("cpu"))
    fr = GraphedFrame.__new__(GraphedFrame)     # the host-side checks only: no device buffers
    fr.flame, fr.num_timesteps, fr.timestep = object(), 4, torch.zeros(1, dtype=torch.int32)
    for t in (-1, 4):
        with pytest.raises(IndexError):
            fr.set_inputs(timestep=t)
    with pytest.raises(ValueError, match="timestep"):
        fr.set_inputs(verts=torch.zeros(3, 3))
    fr.set_inputs(timestep=3)
    assert int(fr.timestep[0]) == 3
    fr.flame = None
    with pytest.raises(ValueError, match="FLAME"):
        fr.set_inputs(timestep=0)


def test_flame_param_groups_are_the_reference_groups():
    from gaussianavatars_b200 import flame_param_groups

    fp = {k: torch.zeros(4, w) for k, w in (("expr", 100), ("rotation", 3), ("neck_pose", 3), ("jaw_pose", 3),
                                            ("eyes_pose", 6), ("translation", 3))}
    fp["shape"] = torch.zeros(300)
    groups = flame_param_groups(fp)
    assert [g["name"] for g in groups] == ["pose", "trans", "expr"]
    assert [g["lr"] for g in groups] == [1e-5, 1e-6, 1e-3]
    assert [len(g["params"]) for g in groups] == [4, 1, 1]
    assert groups[0]["params"][0] is fp["rotation"] and groups[0]["params"][3] is fp["eyes_pose"]
    assert all(p.requires_grad for g in groups for p in g["params"]) and not fp["shape"].requires_grad
    if ref_import.available():
        from argparse import ArgumentParser
        ref_import.prepare()
        from arguments import OptimizationParams   # REAL reference defaults (arguments/__init__.py:95-97)
        op = OptimizationParams(ArgumentParser())
        assert [op.flame_pose_lr, op.flame_trans_lr, op.flame_expr_lr] == [1e-5, 1e-6, 1e-3]


def test_synthetic_flame_assets_have_flame_layouts():
    from gaussianavatars_b200 import synthetic as syn

    a = syn.flame_like_assets(0)
    V = a["v_template"].shape[0]
    assert 5000 <= V <= 5200
    assert a["shapedirs"].shape == (V, 3, 400) and a["posedirs"].shape == (36, 3 * V)
    assert a["J_regressor"].shape == (5, V) and a["lbs_weights"].shape == (V, 5)
    assert a["parents"].tolist() == [-1, 0, 1, 1, 1]
    assert torch.allclose(a["lbs_weights"].sum(1), torch.ones(V), atol=1e-6)
    assert torch.allclose(a["J_regressor"].sum(1), torch.ones(5), atol=1e-6)
    seq = syn.flame_like_sequence(8, seed=1, V=V)
    assert seq["expr"].shape == (8, 100) and seq["eyes_pose"].shape == (8, 6) and seq["static_offset"].shape == (1, V, 3)
    # the demo's magnitudes move the mesh by millimetres to centimetres
    fa = fo.assets_as(dict(a, parents=a["parents"].tolist()), torch.float64)
    v, cano, _ = fo.select_mesh_by_timestep(fa, seq, 3)
    d = (cano[0] - fa["v_template"]).norm(dim=1)
    assert 1e-3 < float(d.max()) < 5e-2, float(d.max())
