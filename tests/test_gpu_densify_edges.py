"""-m gpu: densify_and_prune on the device (csrc/densify.cu) at its decision edges, against the REAL reference run on CPU
(tests/golden/densify_edges_vectors.npz, made by make_golden_densify_edges.py) fed the same split noise: thresholds
rounded as the reference rounds them, NaN and inf inputs, the face rule's boundaries, empty and degenerate models.
Also the C ABI on empty models: every output the plan and the apply promise is written, whatever the caller's buffers
held before."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import densify as od
from tests.test_gpu_densify import _to_dev
from tests.test_oracle_densify import EDGE_CASES, EDGES, check_edge_rows, load_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
JUNK = 0x5A5A5A5A


def _host(t):
    return None if t is None else t.detach().cpu().numpy()


def _want_info(case):
    params, state, stats, hyper, noise, extra, want, want_state, want_b, _ = load_case(case, EDGES)
    pl = od.plan(params, stats, hyper, **extra)
    info = dict(kept=int(pl["keep_orig"].sum()), cloned=int(pl["keep_clone"].sum()),
                split_children=2 * int(pl["keep_child"].sum()), split_parents=int(pl["split"].sum()),
                P_in=params["xyz"].shape[0], P_out=want["xyz"].shape[0])
    return info, (params, state, stats, hyper, noise, extra, want, want_state, want_b)


@pytest.mark.parametrize("case", EDGE_CASES)
def test_edge_case_matches_the_real_reference_run(case):
    import gaussianavatars_b200 as g

    want_info, (params, state, stats, hyper, noise, extra, want, want_state, want_b) = _want_info(case)
    p, s, accum, denom, b = _to_dev(params, state, stats, extra)
    screen = None if hyper[3] < 0 else float(hyper[3])         # 0 stays 0: the wrapper must read it as "off"
    out_p, out_s, b_out, c_out, info = g.densify_arrays(p, s, accum, denom, hyper[0], hyper[1], hyper[2], screen,
                                                        hyper[4], noise=torch.from_numpy(noise).to(DEV), **b)
    assert info == want_info
    check_edge_rows({n: _host(out_p[n]) for n in od.NAMES}, {n: (_host(m), _host(v)) for n, (m, v) in out_s.items()},
                    _host(b_out), _host(c_out), info["kept"] + info["cloned"], want, want_state, want_b)


def test_model_wrapper_at_the_threshold_with_a_python_float_extent():
    """The reference passes scene.cameras_extent (a Python float) and model.percent_dense: the wrapper hands both to
    gab200_densify_plan_f64 in double, which forms the thresholds exactly as the reference does, and clones the splats
    that sit on the threshold."""
    import gaussianavatars_b200 as g

    want_info, (params, state, stats, hyper, noise, extra, want, want_state, want_b) = _want_info("thr_gap_lo")
    extent = float(hyper[2])
    assert np.float32(np.float32(hyper[4]) * np.float32(extent)) != np.float32(hyper[4] * extent)
    t = lambda a, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dt)  # noqa: E731
    m = SimpleNamespace()
    groups = []
    for n in od.NAMES:
        prm = torch.nn.Parameter(t(params[n]))
        setattr(m, g.densify.ATTR[n], prm)
        groups.append({"params": [prm], "lr": 1e-3, "name": n})
    m.optimizer = g.Adam(groups, lr=0.0, eps=1e-15)
    for n in od.NAMES:
        prm = getattr(m, g.densify.ATTR[n])
        m.optimizer.state[prm] = {"step": torch.tensor(3.0), "exp_avg": t(state[n][0]), "exp_avg_sq": t(state[n][1])}
    m.xyz_gradient_accum, m.denom, m.max_radii2D = t(stats["xyz_gradient_accum"]), t(stats["denom"]), t(stats["max_radii2D"])
    m.percent_dense = float(hyper[4])
    m.binding, m.binding_counter = t(extra["binding"], torch.int64), t(extra["binding_counter"], torch.int32)
    m.face_scaling = t(extra["face_scaling"])
    info = g.densify_and_prune(m, float(hyper[0]), float(hyper[1]), extent, None, noise=t(noise))
    assert info == want_info and info["cloned"] > 0
    out_p = {n: _host(getattr(m, g.densify.ATTR[n])) for n in od.NAMES}
    out_s = {n: tuple(_host(m.optimizer.state[getattr(m, g.densify.ATTR[n])][k]) for k in ("exp_avg", "exp_avg_sq"))
             for n in od.NAMES}
    check_edge_rows(out_p, out_s, _host(m.binding), _host(m.binding_counter), info["kept"] + info["cloned"], want,
                    want_state, want_b)


def _empty_args(F, binding):
    """gab200_densify_args of a model without splats (P = 0), bound to F faces when F > 0."""
    from gaussianavatars_b200 import _native as N

    keep = []

    def dev(n, dtype, fill=0):
        x = torch.full((n,), fill, dtype=dtype, device=DEV)
        keep.append(x)
        return x.data_ptr()

    a = N.DensifyArgs()
    a.abi_version, a.P, a.sh_rest_width = N.ABI_VERSION, 0, 9
    a.grad_threshold, a.min_opacity, a.extent, a.percent_dense, a.max_screen_size = 2e-4, 5e-3, 1.0, 0.01, 20.0
    if F > 0:
        a.num_faces = F
        a.binding = dev(1, torch.int32) if binding else None   # an empty torch tensor's data_ptr() is 0
        a.binding_counter, a.face_scaling = dev(F, torch.int32), dev(F, torch.float32, 0.01)
    a.scratch = dev(int(N.lib().gab200_densify_scratch_bytes(0, F)) + 256, torch.uint8, 0xFF)
    totals = torch.full((4,), JUNK, dtype=torch.int32).pin_memory()
    keep.append(totals)
    a.totals_host = totals.data_ptr()
    return a, totals, keep


@pytest.mark.parametrize("entry", ["gab200_densify_plan", "gab200_densify_plan_f64"])
@pytest.mark.parametrize("F,binding", [(0, False), (7, False), (7, True)])
def test_plan_of_an_empty_model_writes_zero_totals(F, binding, entry):
    from gaussianavatars_b200 import _native as N

    a, totals, keep = _empty_args(F, binding)
    stream = C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    extra = (1.0, 0.01) if entry.endswith("_f64") else ()
    N.check(getattr(N.lib(), entry)(C.byref(a), *extra, stream), entry)
    assert totals.tolist() == [0, 0, 0, 0]


@pytest.mark.parametrize("binding", [False, True])
def test_apply_of_an_empty_bound_model_zeroes_the_counter(binding):
    from gaussianavatars_b200 import _native as N

    F = 7
    a, totals, keep = _empty_args(F, binding)
    stream = torch.cuda.current_stream(DEV).cuda_stream
    N.check(N.lib().gab200_densify_plan_f64(C.byref(a), 1.0, 0.01, C.c_void_p(stream)), "gab200_densify_plan_f64")
    counter = torch.full((F,), JUNK, dtype=torch.int32, device=DEV)
    o = N.DensifyOut()
    o.P_out, o.n_child_rows, o.binding_counter = 0, 0, counter.data_ptr()
    N.check(N.lib().gab200_densify_apply(C.byref(a), C.byref(o), C.c_void_p(stream)), "gab200_densify_apply")
    torch.cuda.synchronize(DEV)
    assert counter.tolist() == [0] * F
