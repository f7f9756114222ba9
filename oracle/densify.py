"""CPU restatement (numpy, float32 arithmetic) of the reference's densify_and_prune as ONE gather plan.

TEST INFRASTRUCTURE (oracle).  Follows scene/gaussian_model.py:426-519 (densify_and_prune -> densify_and_clone,
densify_and_split, prune_points) with the optimizer-state surgery of :334-419, restated the way the CUDA op
(gaussianavatars_b200/csrc/densify.cu) computes it: every output row is either a kept original, a clone or a split
child of ONE input row, so the whole sequence -- append clones, append 2 children per split parent, prune the parents,
prune by opacity / world size, with the "every face keeps a splat" rule -- collapses to a source map.  Pinned against
the real reference run on CPU: tests/golden/make_golden_densify.py -> tests/test_oracle_densify.py.

Reference behaviours kept on purpose:
  * `densification_postfix` zeroes xyz_gradient_accum / denom / max_radii2D for ALL splats (:447-449), and it always
    runs before the final prune -- so `max_radii2D > max_screen_size` can never fire there; `max_screen_size` only
    switches the world-size criterion on (:510-513).
  * the face rule is all-or-nothing: if pruning would leave a face without splats, NONE of that face's candidates is
    pruned (:375-380).
  * split children add WORLD-scaled samples to the LOCAL position of a bound splat (:461-464) and take
    log(((exp(s) * fs) / fs) / 1.6) as their scale (:466-468).
"""
from __future__ import annotations

import numpy as np

NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
f32 = np.float32


def _sigmoid(x):
    return (f32(1.0) / (f32(1.0) + np.exp(-x.astype(f32)))).astype(f32)


def build_rotation(r):
    """utils/general_utils.py:78-99."""
    r = r.astype(f32)
    norm = np.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    R = np.zeros((q.shape[0], 3, 3), f32)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R[:, 0, 0] = 1 - 2 * (y * y + z * z)
    R[:, 0, 1] = 2 * (x * y - w * z)
    R[:, 0, 2] = 2 * (x * z + w * y)
    R[:, 1, 0] = 2 * (x * y + w * z)
    R[:, 1, 1] = 1 - 2 * (x * x + z * z)
    R[:, 1, 2] = 2 * (y * z - w * x)
    R[:, 2, 0] = 2 * (x * z - w * y)
    R[:, 2, 1] = 2 * (y * z + w * x)
    R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def plan(params, stats, hyper, binding=None, binding_counter=None, face_scaling=None):
    """hyper: (max_grad, min_opacity, extent, max_screen_size or -1 for None, percent_dense) as the caller holds them
    (Python floats).  Returns dict(clone, split, keep_orig, keep_clone, keep_child (bool [P]), child_scaling [P,3],
    std [P,3])."""
    max_grad, min_opacity = f32(hyper[0]), f32(hyper[1])
    extent, max_screen_size, percent_dense = float(hyper[2]), float(hyper[3]), float(hyper[4])
    accum, denom = stats["xyz_gradient_accum"].reshape(-1).astype(f32), stats["denom"].reshape(-1).astype(f32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        g = accum / denom
        g[np.isnan(g)] = 0
        e = np.exp(params["scaling"].astype(f32))
        if binding is not None:
            fs = face_scaling.reshape(-1).astype(f32)[binding][:, None]
            world = (e * fs).astype(f32)
        else:
            fs, world = None, e
        smax = world.max(axis=1)   # a NaN component makes the maximum NaN, as torch.max does; NaN compares false
        # the reference compares float32 with the Python products: formed in double, rounded to float32 once
        thr, big = f32(percent_dense * extent), f32(0.1 * extent)
        clone = (np.abs(g) >= max_grad) & (smax <= thr)
        split = (g >= max_grad) & (smax > thr)
        op = _sigmoid(params["opacity"].reshape(-1))
        ws_on = max_screen_size > 0
        crit_orig = (op < min_opacity) | (ws_on & (smax > big))
        base = (world / fs) if binding is not None else world
        child_scaling = np.log((base / f32(0.8 * 2)).astype(f32)).astype(f32)
        child_world = np.exp(child_scaling) * (fs if binding is not None else f32(1.0))
        crit_child = (op < min_opacity) | (ws_on & (child_world.max(axis=1) > big))
    if binding is not None:
        F = binding_counter.shape[0]
        delta = np.bincount(binding, weights=(clone | split).astype(np.int64), minlength=F).astype(np.int64)
        cand = ((~split) & crit_orig).astype(np.int64) + (clone & crit_orig).astype(np.int64) + 2 * (split & crit_child)
        pruned = np.bincount(binding, weights=cand, minlength=F).astype(np.int64)
        ok = ((binding_counter.astype(np.int64) + delta - pruned) > 0)[binding]
    else:
        ok = np.ones_like(clone)
    return dict(clone=clone, split=split, keep_orig=(~split) & ~(crit_orig & ok), keep_clone=clone & ~(crit_orig & ok),
                keep_child=split & ~(crit_child & ok), child_scaling=child_scaling, std=world)


def densify_and_prune(params, state, stats, hyper, noise, binding=None, binding_counter=None, face_scaling=None):
    """params / state: dicts name -> array (state: name -> (exp_avg, exp_avg_sq)); noise [2S,3] standard normal (rows
    [0,S): first child of the S split parents in index order, [S,2S): second).  Returns (params', state', binding',
    binding_counter', P')."""
    pl = plan(params, stats, hyper, binding, binding_counter, face_scaling)
    P = params["xyz"].shape[0]
    idx = np.arange(P)
    sel = idx[pl["split"]]
    S = sel.shape[0]
    rank = np.full(P, -1, np.int64)
    rank[sel] = np.arange(S)
    src_o, src_c, src_ch = idx[pl["keep_orig"]], idx[pl["keep_clone"]], idx[pl["keep_child"]]
    src = np.concatenate((src_o, src_c, src_ch, src_ch))
    n_o, n_c, n_ch = len(src_o), len(src_c), len(src_ch)
    out_p, out_s = {}, {}
    for n in NAMES:
        out_p[n] = params[n][src].copy()
        m, v = state[n]
        zeros = np.zeros((n_c + 2 * n_ch,) + m.shape[1:], m.dtype)
        out_s[n] = (np.concatenate((m[src_o], zeros)), np.concatenate((v[src_o], zeros)))
    if n_ch:
        R = build_rotation(params["rotation"][src_ch])
        for k in range(2):
            nz = noise[rank[src_ch] + k * S].astype(f32)
            samples = (nz * pl["std"][src_ch]).astype(f32)   # mean (zeros) + noise * std
            lo = n_o + n_c + k * n_ch
            out_p["xyz"][lo:lo + n_ch] = (np.einsum("nij,nj->ni", R, samples).astype(f32) + params["xyz"][src_ch]).astype(f32)
            out_p["scaling"][lo:lo + n_ch] = pl["child_scaling"][src_ch]
    b_out = c_out = None
    if binding is not None:
        b_out = binding[src].astype(np.int32)
        c_out = np.bincount(b_out, minlength=binding_counter.shape[0]).astype(np.int32)
    return out_p, out_s, b_out, c_out, len(src)
