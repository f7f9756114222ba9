"""Generates tests/golden/flame_vectors.npz by IMPORTING the real reference FLAME forward (flame_model/flame.py
FlameHead.forward, flame_model/lbs.py lbs) and calling FlameHead.forward unbound on a namespace that carries seeded
synthetic buffers of FLAME's layouts (the licensed flame2023.pkl is not needed: the operator is dense algebra over
arrays of known shapes).  Small V keeps the fixture small; n_shape = 300 and n_expr = 100 are FLAME's.

Timesteps: the 4 rows of demo_flame_param_head.npz, a row whose neck / jaw / eyes are exactly zero, and a row with
rotations near 2.5 rad.  For every timestep t the fixture holds, in float64: verts, verts_cano, the posed joints, and
the autograd gradients of the seeded linear functional sum(C_t * verts) w.r.t. every (T, .) tensor.

    python tests/golden/make_golden_flame.py
"""
import os
import sys
from types import SimpleNamespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)

from tests import ref_import  # noqa: E402

V, N_SHAPE, N_EXPR = 64, 300, 100
POSED = ("expr", "rotation", "neck_pose", "jaw_pose", "eyes_pose", "translation")


def assets(rng):
    x = rng.normal(0, 0.08, size=(V, 3))
    shapedirs = rng.normal(0, 1e-3, size=(V, 3, N_SHAPE + N_EXPR))
    posedirs = rng.normal(0, 2e-3, size=(36, 3 * V))
    J_regressor = rng.uniform(0, 1, size=(5, V)) ** 4
    J_regressor /= J_regressor.sum(1, keepdims=True)
    w = rng.uniform(0, 1, size=(V, 5)) ** 3
    w /= w.sum(1, keepdims=True)
    f32 = lambda a: a.astype(np.float32)   # noqa: E731  the fixture's values are exactly float32 numbers
    return dict(v_template=f32(x), shapedirs=f32(shapedirs), posedirs=f32(posedirs), J_regressor=f32(J_regressor),
                lbs_weights=f32(w), parents=np.array([-1, 0, 1, 1, 1], np.int64))


def params(rng):
    demo = np.load(os.path.join(HERE, "demo_flame_param_head.npz"))
    p = {k: demo[k].astype(np.float32) for k in ("shape", *POSED)}
    p["static_offset"] = demo["static_offset"].astype(np.float32)            # (1, 64, 3)
    zero = {k: np.zeros_like(p[k][:1]) for k in POSED}                        # neck / jaw / eyes exactly 0
    zero["expr"], zero["rotation"], zero["translation"] = p["expr"][:1], p["rotation"][:1], p["translation"][:1]
    big = {k: p[k][1:2].copy() for k in POSED}                                # rotations near 2.5 rad
    for k, n in (("rotation", 3), ("neck_pose", 3), ("jaw_pose", 3), ("eyes_pose", 6)):
        d = rng.normal(size=n).reshape(-1, 3)
        big[k] = (2.5 * d / np.linalg.norm(d, axis=1, keepdims=True)).reshape(1, n).astype(np.float32)
    for k in POSED:
        p[k] = np.concatenate([p[k], zero[k], big[k]], 0)
    return p


def main():
    ref_import.prepare()
    import torch
    from flame_model.flame import FlameHead  # noqa: E402  (REAL reference code)
    from flame_model.lbs import lbs  # noqa: E402

    rng = np.random.default_rng(20261015)
    A, P = assets(rng), params(rng)
    T = P["expr"].shape[0]
    dt = torch.float64
    ns = SimpleNamespace(dtype=dt, **{k: torch.tensor(v, dtype=dt if v.dtype == np.float32 else torch.long)
                                      for k, v in A.items()})
    C = rng.normal(size=(T, V, 3))
    out = {k: v for k, v in A.items()}
    out.update({f"param_{k}": v for k, v in P.items()})
    out["C"] = C
    verts_all, cano_all, joints_all = [], [], []
    grads = {k: [] for k in POSED}
    for t in range(T):
        fp = {k: torch.tensor(P[k], dtype=dt, requires_grad=k in POSED) for k in P}
        verts, cano = FlameHead.forward(ns, fp["shape"][None, ...], fp["expr"][[t]], fp["rotation"][[t]],
                                        fp["neck_pose"][[t]], fp["jaw_pose"][[t]], fp["eyes_pose"][[t]],
                                        fp["translation"][[t]], zero_centered_at_root_node=False, return_landmarks=False,
                                        return_verts_cano=True, static_offset=fp["static_offset"],
                                        dynamic_offset=torch.zeros(1, V, 3, dtype=dt))
        full_pose = torch.cat([fp["rotation"][[t]], fp["neck_pose"][[t]], fp["jaw_pose"][[t]], fp["eyes_pose"][[t]]], 1)
        _, joints, _ = lbs(full_pose, cano.detach(), ns.posedirs, ns.J_regressor, ns.parents, ns.lbs_weights, dtype=dt)
        (verts * torch.tensor(C[t][None], dtype=dt)).sum().backward()
        verts_all.append(verts[0].detach().numpy())
        cano_all.append(cano[0].detach().numpy())
        joints_all.append((joints + fp["translation"][[t]][:, None, :])[0].detach().numpy())
        for k in POSED:
            grads[k].append(fp[k].grad.numpy())
    out["verts"], out["verts_cano"], out["joints"] = np.stack(verts_all), np.stack(cano_all), np.stack(joints_all)
    for k in POSED:
        out[f"grad_{k}"] = np.stack(grads[k])   # (T timesteps, T rows, width)
    np.savez_compressed(os.path.join(HERE, "flame_vectors.npz"), **out)
    for k, v in out.items():
        print(k, v.shape, v.dtype)


if __name__ == "__main__":
    main()
