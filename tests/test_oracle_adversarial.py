"""CPU: the adversarial scene builders reach the regimes they exist for (asserted on the oracle's own state), and the
oracle's hand-written backward equals float64 autograd of the dense model (oracle/dense64.py) on every one of them.

A builder that stops reaching its regime fails here rather than silently weakening tests/test_gpu_adversarial.py."""
import numpy as np
import pytest
import torch

from oracle import dense64
from tests import adversarial_scenes as A
from tests import helpers as h


def _oracle(sc):
    return h.oracle_forward(sc)


def _lens(st):
    return st.ranges[:, 1].astype(np.int64) - st.ranges[:, 0]


# ---- regimes --------------------------------------------------------------------------------------------------------
def test_needles_are_near_singular_and_mostly_culled_pairs():
    sc = A.build("needles")
    s = sc["scales"].numpy()
    assert (s.max(1) / s.min(1) >= 999.0).all()
    st = _oracle(sc)
    vis = st.radii > 0
    # 2-D covariance before the 0.3 dilation: inverse of the conic minus 0.3 I
    a, b, c = st.conic_opacity[vis, 0].astype(np.float64), st.conic_opacity[vis, 1], st.conic_opacity[vis, 2]
    det = a * c - b * b
    ca, cb, cc = c / det - 0.3, -b / det, a / det - 0.3
    ratio = (ca * cc - cb * cb) / (ca + cc) ** 2            # det / trace^2: 0 for a rank-1 footprint
    assert (ratio < 1e-3).mean() > 0.9, "needle footprints are not near-singular before the dilation"
    assert (st.radii[vis] > 0.3 * max(sc["W"], sc["H"])).sum() >= 10, "no needle reaches across the image"
    # pairs of the reference's bounding-square list that no pixel accepts: what the culled binning drops
    acc = A.accepted_instances(st)
    assert st.N - acc.size > 0.4 * st.N, f"only {st.N - acc.size}/{st.N} instances contribute nothing"


def test_near_plane_radii_beyond_the_image_and_culled_at_0_2():
    sc = A.build("near_plane")
    st = _oracle(sc)
    z = sc["means3D"][:, 2].numpy()
    assert (z <= np.float32(0.2)).sum() >= 8 and (st.radii[z <= np.float32(0.2)] == 0).all()
    just = z == np.nextafter(np.float32(0.2), np.float32(1))
    assert just.sum() >= 4 and (st.radii[just] > 0).all()
    big = st.radii > max(sc["W"], sc["H"])
    assert big.sum() >= 10, "no footprint larger than the image"
    gx, gy = (sc["W"] + 15) // 16, (sc["H"] + 15) // 16
    assert (st.tiles_touched[big] == gx * gy).all(), "a radius beyond the image must clamp to the whole grid"


def test_guard_band_splats_reach_the_image_through_the_clamped_jacobian():
    sc = A.build("guard_band")
    st = _oracle(sc)
    cam = sc["cam"]
    m = sc["means3D"].numpy()
    out = (np.abs(m[:, 0] / m[:, 2]) > 1.3 * cam.tanfovx) | (np.abs(m[:, 1] / m[:, 2]) > 1.3 * cam.tanfovy)
    assert out.all()
    gout = torch.randn(3, sc["H"], sc["W"], generator=torch.Generator().manual_seed(0))
    g = h.oracle_backward(sc, st, gout.numpy())
    contributes = np.abs(g["opacities"][:, 0]) > 0
    assert (contributes & out).sum() >= 20, "too few splats beyond the guard band reach a pixel"


@pytest.mark.parametrize("stacks", [(20, 400), (20, 400, 2100)])
def test_saturating_stack_stops_walks_partway_in_mixed_tiles(stacks):
    sc = A.saturating_stack(stacks=stacks)
    st = _oracle(sc)
    lens = _lens(st)
    gx = (sc["W"] + 15) // 16
    n_c = st.n_contrib
    stopped = np.zeros_like(st.final_T, bool)
    for tile in range(lens.size):
        ty, tx = divmod(tile, gx)
        blk = (slice(16 * ty, 16 * ty + 16), slice(16 * tx, 16 * tx + 16))
        stopped[blk] = (n_c[blk] < lens[tile]) & (st.final_T[blk] >= 1e-4) & (st.final_T[blk] < 1e-2)
    assert stopped.sum() >= 20, "no pixel ended its walk on the T < 1e-4 test partway through its list"
    # the stopped pixels share tiles with pixels that never saturated
    for tile in range(lens.size):
        ty, tx = divmod(tile, gx)
        blk = (slice(16 * ty, 16 * ty + 16), slice(16 * tx, 16 * tx + 16))
        if stopped[blk].any() and (st.final_T[blk] > 0.5).any():
            break
    else:
        raise AssertionError("no tile holds both saturated and unsaturated pixels")
    t = A.pair_table(st)
    on_clamp = t["alpha"] == np.float32(0.99)
    assert on_clamp.sum() >= 50 and (on_clamp & t["live"]).sum() >= 1, "alpha never sits on the 0.99 clamp"
    assert (lens > 0).any() and (lens[lens > 0] < 32).any() and ((lens >= 32) & (lens < 1984)).any()
    if max(stacks) > 2048:
        assert (lens >= 2048).any(), "no list beyond the default heavy-backward threshold"


def test_faint_splats_straddle_the_alpha_threshold():
    sc = A.build("faint")
    st = _oracle(sc)
    t = A.pair_table(st)
    near = (t["power"] <= 0) & (np.abs(t["alpha"].astype(np.float64) * 255.0 - 1.0) < 1e-3)
    acc = t["alpha"] >= A.ALPHA_MIN
    assert (near & acc).sum() >= 10 and (near & ~acc).sum() >= 10, \
        f"accepted {int((near & acc).sum())} / rejected {int((near & ~acc).sum())} pairs within 1e-3 of 1/255"
    # opacity a few ulp around float32(1/255) on an exact pixel centre: alpha == opacity on both sides of the test
    o = sc["opacities"][:, 0].numpy()
    thr = A.ALPHA_MIN
    ulp = np.abs(o - thr) <= 3 * np.spacing(thr)
    hit = ulp & (st.xy[:, 0] == np.round(st.xy[:, 0])) & (st.xy[:, 1] == np.round(st.xy[:, 1])) & (st.radii > 0)
    assert (hit & (o < thr)).sum() >= 2 and (hit & (o >= thr)).sum() >= 2, "no exact-centre ulp splats on both sides"
    below = o < np.float32(0.99) * thr
    assert below.sum() >= 10 and (st.radii[below] > 0).all(), "faint splats below the culling margin must stay listed"


def test_tile_borders_hit_the_borders_exactly():
    sc = A.build("tile_borders")
    st = _oracle(sc)
    vis = st.radii > 0
    assert vis.all() and set(np.unique(st.radii)) <= {2, 3, 4}
    for xy in (st.xy[:, 0], st.xy[:, 1]):
        for off in (-0.5, 0.0, 15.5):
            r = np.mod(xy - off, 16.0)
            assert (r == 0).sum() >= 3, f"no centre exactly on 16k {off:+}"
    # a splat on a border lands in the lists of both tiles it straddles
    assert (st.tiles_touched >= 2).mean() > 0.5


def test_ties_share_depth_keys_and_sort_by_id():
    sc = A.build("tile_borders+ties")
    st = _oracle(sc)
    d = st.depths[st.radii > 0]
    assert d.size - np.unique(d).size >= 20, "no equal depth keys"
    k, v = st.keys_sorted, st.vals_sorted
    same = k[1:] == k[:-1]
    assert same.sum() >= 20 and (v[1:][same] > v[:-1][same]).all()


def test_sh3_variant_clamps_colours():
    sc = A.build("needles+sh3")
    st = _oracle(sc)
    vis = st.radii > 0
    assert sc["sh_degree"] == 3 and sc["shs"].shape[1] == 16
    assert st.clamped[vis].sum() >= 20 and (st.clamped[vis] == 0).sum() >= 20


@pytest.mark.parametrize("W,H", A.RAGGED_SIZES)
def test_ragged_sizes_render_something(W, H):
    for name in A.BUILDERS:
        sc = A.build(name, W, H)
        st = _oracle(sc)
        assert st.out_color.shape == (3, H, W)
        assert np.isfinite(st.out_color).all()


# ---- oracle against float64 autograd of the dense model ----------------------------------------------------------------
# Needles run at 16x16 (long axes up to ~17 px): a 1e3 needle's covariance R diag(s^2) R^T has condition number ~1e6,
# so its float32 evaluation (the reference's, restated by the oracle and bit for bit by the CUDA preprocess) moves the
# conic by up to a few percent on the worst splat.  At 48x40 that reaches 1e-5 in the image against float64 (5e-6 gate),
# and at 24x20 the short axes' dL/dscale differ by 2e-4 of max|ref| (2e-5 gate): float32 rounding of an ill-conditioned
# input, not an error of either side.  The CUDA path is held to the oracle at 48x40 by tests/test_gpu_adversarial.py.
DENSE_CASES = [("needles", 16, 16), "near_plane", "guard_band", "saturating_stack", "faint", "tile_borders",
               "tile_borders+ties", ("needles+sh3", 16, 16), ("faint", 15, 17), ("near_plane", 1, 37), ("tile_borders", 33, 31), ("needles", 4, 20),
               ("guard_band", 37, 1), ("saturating_stack", 17, 15)]


def _case(c):
    return (c, None, None) if isinstance(c, str) else c


@pytest.mark.parametrize("case", DENSE_CASES, ids=lambda c: "-".join(map(str, c)) if not isinstance(c, str) else c)
def test_oracle_backward_equals_float64_autograd_on_adversarial_scenes(case):
    name, W, H = _case(case)
    sc = A.build(name, W, H)
    st = _oracle(sc)
    img, g64 = dense_image_and_grads(sc, st, seed=1)
    ke = A.knife_edges(st)
    print(f"[knife] {name} {sc['W']}x{sc['H']}: {ke['pairs']} pairs, {int(ke['pixels'].sum())} pixels, "
          f"{int(ke['splats'].sum())}/{st.P} splats")
    h.assert_image_explained(st.out_color, img, ke["pixels"], "oracle image vs float64", tol=5e-6, cap=5e-6)
    gout = torch.randn(3, sc["H"], sc["W"], generator=torch.Generator().manual_seed(1))
    g = h.oracle_backward(sc, st, gout.numpy())
    for k, ref in g64.items():
        h.assert_grad_explained(g[k], ref, A.affected(ke, k), f"oracle dL/d{k}", rtol=0.0, atol_frac=2e-5, knife_allowed=3)


def dense_image_and_grads(sc, st, seed=1):
    """float64 image and gradients of <image, gout> (gout ~ N(0,1), `seed`) from oracle/dense64.py with the oracle's
    radii and tile rectangles; the same method as test_oracle_grad.test_oracle_backward_equals_float64_autograd."""
    cam = sc["cam"]
    P = sc["means3D"].shape[0]
    t64 = {k: sc[k].double().clone().requires_grad_(True) for k in ("means3D", "opacities", "scales", "rotations", "shs")}
    m2 = torch.zeros(P, 3, dtype=torch.float64, requires_grad=True)
    img, _ = dense64.render(t64["means3D"], m2, t64["opacities"], cam.world_view_transform.double(),
                            cam.full_proj_transform.double(), cam.camera_center.double(), sc["W"], sc["H"],
                            cam.tanfovx, cam.tanfovy, sc["bg"].double(), shs=t64["shs"], sh_degree=sc["sh_degree"],
                            scales=t64["scales"], rotations=t64["rotations"], radii=torch.from_numpy(st.radii).long(),
                            rect_xy=torch.from_numpy(st.xy))
    gout = torch.randn(3, sc["H"], sc["W"], generator=torch.Generator().manual_seed(seed))
    img.backward(gout.double())
    grads = {k: t64[k].grad.numpy() for k in t64}
    grads["means2D"] = m2.grad.numpy()
    return img.detach().numpy(), grads
