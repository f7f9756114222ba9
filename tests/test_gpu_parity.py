"""-m gpu: the CUDA path (through the C ABI, via the reference-shaped Python surface) against the CPU oracle."""
import numpy as np
import pytest
import torch

from tests import adversarial_scenes as A
from tests import helpers as h

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=["counting-tile-sort", "cub-radix-tile-sort"])
def tile_sort_implementation(request):
    """Every test of this file runs on both implementations of the per-instance sort by tile
    (include/gab200_rasterizer.h GAB200_TUNE_TILE_SORT): the sorted stream, image and gradients must not depend on it."""
    from gaussianavatars_b200 import _native as N

    N.tune(N.TUNE_TILE_SORT, 1 if request.param.startswith("counting") else 0)
    yield
    N.tune(N.TUNE_TILE_SORT, 0)


def _dev():
    return torch.device("cuda:0")


def _run_cuda(scene, dev, need_grad=False, exact=True, **over):
    import gaussianavatars_b200 as g
    from gaussianavatars_b200 import rasterizer as R

    R.set_exact_binning(exact)
    R.keep_last_state(True)
    rs = h.cuda_settings(scene, dev, scale_modifier=over.pop("scale_modifier", 1.0))
    t = {k: scene[k].to(dev).clone().requires_grad_(need_grad) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    means2D = torch.zeros((scene["means3D"].shape[0], 3), device=dev, requires_grad=need_grad)
    kw = dict(means3D=t["means3D"], means2D=means2D, opacities=t["opacities"], shs=t["shs"], scales=t["scales"],
              rotations=t["rotations"])
    kw.update(over)
    img, radii = g.GaussianRasterizer(rs)(**kw)
    torch.cuda.synchronize()
    return img, radii, t, means2D


@pytest.mark.parametrize("P,W,H,deg,seed", [(10_000, 256, 256, 0, 0), (4_000, 333, 201, 3, 1), (2_000, 64, 48, 2, 2),
                                            (6_000, 200, 120, 1, 3)])
def test_forward_and_sorted_keys_bit_exact(P, W, H, deg, seed):
    """Config 1 (10k, 256^2, SH0) + ragged image sizes / SH degrees.  radii, the sorted (tile|depth key, splat id)
    stream and the tile ranges must be BIT-EXACT; the image within the 1e-4 budget."""
    from gaussianavatars_b200 import rasterizer as R

    dev = _dev()
    scene = h.random_scene(P, W, H, sh_degree=deg, seed=seed, scale_shift=0.6)
    st = h.oracle_forward(scene)
    img, radii, _, _ = _run_cuda(scene, dev, exact=True)
    assert np.array_equal(radii.cpu().numpy(), st.radii), "radii differ from the oracle"
    keys, vals, ranges, n = R.export_last_binning()
    assert n == st.N
    assert np.array_equal(keys.cpu().numpy().view(np.uint64), st.keys_sorted), "sorted tile|depth keys not bit-exact"
    assert np.array_equal(vals.cpu().numpy().view(np.uint32), st.vals_sorted), "sorted splat ids not bit-exact"
    assert np.array_equal(ranges.cpu().numpy().view(np.uint32), st.ranges), "tile ranges differ"
    h.assert_image_close(img.cpu().numpy(), st.out_color, "forward image")


def test_long_tile_lists_take_the_bitmap_sort_and_stay_bit_exact():
    """Every splat covers every tile: 5,000-entry lists, beyond the 2048 entries a CTA sorts in shared memory
    (tile_sort_long_kernel).  Sorted stream still bit-identical to the oracle's."""
    from gaussianavatars_b200 import rasterizer as R

    dev = _dev()
    scene = h.random_scene(5_000, 64, 48, sh_degree=0, seed=21, scale_shift=2.5)
    st = h.oracle_forward(scene)
    lens = st.ranges[:, 1].astype(np.int64) - st.ranges[:, 0]
    assert lens.max() > 2048, f"scene only reaches {lens.max()} entries per tile"
    img, radii, _, _ = _run_cuda(scene, dev, exact=True)
    keys, vals, ranges, n = R.export_last_binning()
    assert n == st.N
    assert np.array_equal(keys.cpu().numpy().view(np.uint64), st.keys_sorted)
    assert np.array_equal(vals.cpu().numpy().view(np.uint32), st.vals_sorted)
    assert np.array_equal(ranges.cpu().numpy().view(np.uint32), st.ranges)
    h.assert_image_close(img.cpu().numpy(), st.out_color, "long-list image")


def test_culled_binning_is_exact_subsequence_and_same_image():
    """Default binning drops (splat,tile) pairs that contribute nothing: the emitted stream must be a subsequence of the
    reference stream (same keys, same relative order) and the image must not change AT ALL."""
    from gaussianavatars_b200 import rasterizer as R

    dev = _dev()
    scene = h.random_scene(8_000, 320, 240, sh_degree=1, seed=7, scale_shift=0.9)
    img_e, radii_e, _, _ = _run_cuda(scene, dev, exact=True)
    keys_e, vals_e, _, n_e = R.export_last_binning()
    img_c, radii_c, _, _ = _run_cuda(scene, dev, exact=False)
    keys_c, vals_c, _, n_c = R.export_last_binning()
    assert torch.equal(radii_e, radii_c), "radii must not depend on the binning policy"
    assert n_c < n_e, "culling removed nothing on a scene where it must"
    ke = (keys_e.cpu().numpy().view(np.uint64), vals_e.cpu().numpy().view(np.uint32))
    kc = (keys_c.cpu().numpy().view(np.uint64), vals_c.cpu().numpy().view(np.uint32))
    # subsequence check: walk the exact stream once
    full = {(int(k), int(v)): i for i, (k, v) in enumerate(zip(*ke))}
    pos = np.array([full[(int(k), int(v))] for k, v in zip(*kc)])
    assert (np.diff(pos) > 0).all(), "culled stream is not an order-preserving subsequence"
    assert torch.equal(img_e, img_c), "culling changed the image"


def test_image_is_background_where_nothing_lands_and_weights_sum():
    dev = _dev()
    scene = h.random_scene(300, 128, 96, sh_degree=0, seed=11, scale_shift=-1.0)
    st = h.oracle_forward(scene)
    img, _, _, _ = _run_cuda(scene, dev)
    img = img.cpu().numpy()
    empty = st.n_contrib == 0
    assert empty.any()
    for ch in range(3):
        assert np.array_equal(img[ch][empty], np.full(empty.sum(), scene["bg"][ch].item(), np.float32))


def _explained_close(g, ref, affected, what):
    """helpers.assert_grad_close's tolerance (2e-3 max|ref|) for every entry outside the knife set of the oracle's
    state; its allowance (max(3, 1e-3 n) entries, no cap) for the entries inside it."""
    n = int(np.asarray(ref).size)
    h.assert_grad_explained(g, ref, affected, what, rtol=0.0, atol_frac=2e-3, cap=np.inf,
                            knife_allowed=max(3, int(1e-3 * n)))


@pytest.mark.parametrize("deg,seed,exact", [(3, 0, True), (3, 1, False), (0, 2, False), (2, 3, True)])
def test_backward_parity(deg, seed, exact):
    dev = _dev()
    scene = h.random_scene(3_000, 208, 160, sh_degree=deg, seed=seed, scale_shift=0.7)
    st = h.oracle_forward(scene)
    gout = torch.randn(3, scene["H"], scene["W"], generator=torch.Generator().manual_seed(1))
    ref = h.oracle_backward(scene, st, gout.numpy())
    img, radii, t, means2D = _run_cuda(scene, dev, need_grad=True, exact=exact)
    (img * gout.to(dev)).sum().backward()
    torch.cuda.synchronize()
    ke = A.knife_edges(st)
    for name in ("means3D", "opacities", "scales", "rotations", "shs"):
        _explained_close(t[name].grad.cpu().numpy(), ref[name], A.affected(ke, name), f"dL/d{name}")
    _explained_close(means2D.grad.cpu().numpy(), ref["means2D"], A.affected(ke, "means2D"), "dL/dmeans2D")
    # splats that never emitted an instance get exactly zero everywhere
    invis = torch.from_numpy(st.radii == 0).to(dev)
    assert float(t["means3D"].grad[invis].abs().sum()) == 0.0


def test_precomputed_colors_and_cov3d_route():
    """The other two input variants of the reference surface (colors_precomp / cov3D_precomp)."""
    dev = _dev()
    scene = h.random_scene(2_000, 160, 128, sh_degree=0, seed=5, scale_shift=0.8)
    st0 = h.oracle_forward(scene)
    colors = torch.rand(2_000, 3, generator=torch.Generator().manual_seed(3))
    cov = torch.from_numpy(st0.cov3D.copy())
    # cov3D of culled splats is zero in the oracle state; recompute for all through the scale/rotation route first
    st = h.oracle_forward(scene, shs=None, colors_precomp=colors.numpy(), scales=None, rotations=None,
                          cov3D_precomp=_all_cov(scene))
    cov = torch.from_numpy(_all_cov(scene))
    gout = torch.randn(3, scene["H"], scene["W"], generator=torch.Generator().manual_seed(2))
    ref = h.oracle_backward(scene, st, gout.numpy(), shs=None, scales=None, rotations=None)
    import gaussianavatars_b200 as g

    rs = h.cuda_settings(scene, dev)
    m3 = scene["means3D"].to(dev).requires_grad_(True)
    m2 = torch.zeros(2_000, 3, device=dev, requires_grad=True)
    op = scene["opacities"].to(dev).requires_grad_(True)
    col = colors.to(dev).requires_grad_(True)
    cv = cov.to(dev).requires_grad_(True)
    img, radii = g.GaussianRasterizer(rs)(means3D=m3, means2D=m2, opacities=op, colors_precomp=col, cov3D_precomp=cv)
    h.assert_image_close(img.detach().cpu().numpy(), st.out_color, "colors/cov3D route image")
    (img * gout.to(dev)).sum().backward()
    h.assert_grad_close(col.grad.cpu().numpy(), ref["colors_precomp"], "dL/dcolors_precomp")
    h.assert_grad_close(cv.grad.cpu().numpy(), ref["cov3D_precomp"], "dL/dcov3D_precomp")
    h.assert_grad_close(m3.grad.cpu().numpy(), ref["means3D"], "dL/dmeans3D (cov route)")


def _all_cov(scene):
    """cov3D for every splat via the Python twin (utils/general_utils.py:101-110 semantics)."""
    from oracle import dense64

    R = dense64.quat_to_R(scene["rotations"].double())
    s = scene["scales"].double()
    S = R @ torch.diag_embed(s * s) @ R.transpose(1, 2)
    c = torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], dim=1)
    return c.float().contiguous().numpy()


def test_scale_modifier_and_mark_visible():
    import gaussianavatars_b200 as g
    from oracle import rasterizer as orc

    dev = _dev()
    scene = h.random_scene(3_000, 160, 128, sh_degree=1, seed=9, scale_shift=0.5)
    cam = scene["cam"]
    st = orc.forward(scene["means3D"].numpy(), scene["opacities"].numpy(), cam.world_view_transform.numpy(),
                     cam.full_proj_transform.numpy(), cam.camera_center.numpy(), scene["W"], scene["H"], cam.tanfovx,
                     cam.tanfovy, scene["bg"].numpy(), shs=scene["shs"].numpy(), sh_degree=1,
                     scales=scene["scales"].numpy(), rotations=scene["rotations"].numpy(), scale_modifier=0.6)
    img, radii, _, _ = _run_cuda(scene, dev, scale_modifier=0.6)
    assert np.array_equal(radii.cpu().numpy(), st.radii)
    h.assert_image_close(img.cpu().numpy(), st.out_color, "scale_modifier image")
    # markVisible: put a third of the splats behind the camera
    pos = scene["means3D"].clone()
    pos[::3, 2] = -1.0
    vis = g.GaussianRasterizer(h.cuda_settings(scene, dev)).markVisible(pos.to(dev))
    assert np.array_equal(vis.cpu().numpy(), orc.mark_visible(pos.numpy(), cam.world_view_transform.numpy()))


def test_edge_cases_empty_and_all_culled():
    import gaussianavatars_b200 as g

    dev = _dev()
    scene = h.random_scene(64, 50, 34, sh_degree=0, seed=4)
    rs = h.cuda_settings(scene, dev)
    # (a) P = 0
    e = lambda *s: torch.zeros(*s, device=dev)  # noqa: E731
    img, radii = g.GaussianRasterizer(rs)(means3D=e(0, 3), means2D=e(0, 3), opacities=e(0, 1), shs=e(0, 1, 3),
                                          scales=e(0, 3), rotations=e(0, 4))
    assert radii.numel() == 0
    assert torch.allclose(img, scene["bg"].to(dev)[:, None, None].expand_as(img))
    # (b) everything behind the near plane -> radii 0, image = background, backward gives zeros
    m3 = scene["means3D"].clone()
    m3[:, 2] = 0.1
    m3 = m3.to(dev).requires_grad_(True)
    img, radii = g.GaussianRasterizer(rs)(means3D=m3, means2D=e(64, 3), opacities=scene["opacities"].to(dev),
                                          shs=scene["shs"].to(dev), scales=scene["scales"].to(dev),
                                          rotations=scene["rotations"].to(dev))
    assert int(radii.abs().sum()) == 0
    img.sum().backward()
    assert float(m3.grad.abs().sum()) == 0.0


def test_argument_validation_matches_reference_errors():
    import gaussianavatars_b200 as g

    dev = _dev()
    scene = h.random_scene(16, 32, 32, sh_degree=0, seed=4)
    rs = h.cuda_settings(scene, dev)
    t = {k: scene[k].to(dev) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    m2 = torch.zeros(16, 3, device=dev)
    r = g.GaussianRasterizer(rs)
    with pytest.raises(Exception, match="SHs or precomputed colors"):
        r(means3D=t["means3D"], means2D=m2, opacities=t["opacities"], scales=t["scales"], rotations=t["rotations"])
    with pytest.raises(Exception, match="SHs or precomputed colors"):
        r(means3D=t["means3D"], means2D=m2, opacities=t["opacities"], shs=t["shs"], colors_precomp=torch.rand(16, 3, device=dev),
          scales=t["scales"], rotations=t["rotations"])
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(means3D=t["means3D"], means2D=m2, opacities=t["opacities"], shs=t["shs"])
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(means3D=t["means3D"], means2D=m2, opacities=t["opacities"], shs=t["shs"], scales=t["scales"],
          rotations=t["rotations"], cov3D_precomp=torch.rand(16, 6, device=dev))
    with pytest.raises(RuntimeError):
        r(means3D=t["means3D"].cpu(), means2D=m2.cpu(), opacities=t["opacities"].cpu(), shs=t["shs"].cpu(),
          scales=t["scales"].cpu(), rotations=t["rotations"].cpu())


# ------------------------------------------------------------------------------------------------------------
# fused FLAME binding
# ------------------------------------------------------------------------------------------------------------
def _fused_cuda(sc, dev, need_grad=True, exact=False):
    import gaussianavatars_b200 as g
    from gaussianavatars_b200 import rasterizer as R
    from gaussianavatars_b200.model import face_frame

    R.set_exact_binning(exact)
    R.keep_last_state(True)
    p = sc["params"]
    leaves = {k: p[k].to(dev).clone().requires_grad_(need_grad)
              for k in ("_xyz", "_rotation", "_scaling", "_opacity", "_features_dc", "_features_rest")}
    verts = sc["verts"].to(dev).clone().requires_grad_(need_grad)
    fc, fR, fs = face_frame(verts, sc["faces"].to(dev))
    cam = sc["cam"]
    rs = g.GaussianRasterizationSettings(sc["H"], sc["W"], cam.tanfovx, cam.tanfovy, sc["bg"].to(dev), 1.0,
                                         cam.world_view_transform.to(dev), cam.full_proj_transform.to(dev),
                                         sc["sh_degree"], cam.camera_center.to(dev), False, True)
    m2 = torch.zeros(p["_xyz"].shape[0], 3, device=dev, requires_grad=need_grad)
    img, radii = g.rasterize_bound(rs, leaves["_xyz"], leaves["_rotation"], leaves["_scaling"], leaves["_opacity"],
                                   leaves["_features_dc"], leaves["_features_rest"], p["binding"].to(dev), fc, fR, fs,
                                   means2D=m2)
    return img, radii, leaves, verts, m2, rs, (fc, fR, fs)


def test_fused_binding_forward_keys_bit_exact_on_exported_activation():
    """Fused surface contract (SURVEY.md 7.4-2): (i) the exported world-space activation is within a few ulp of the
    eager getters; (ii) the tile|depth key stream of the fused forward is BIT-IDENTICAL to the oracle evaluated on
    that exported activation; (iii) the image matches the eager-getter oracle within budget."""
    import gaussianavatars_b200 as g
    from gaussianavatars_b200 import rasterizer as R
    from oracle import rasterizer as orc

    dev = _dev()
    sc = h.avatar_scene(P=12_000, W=400, H=304, seed=1)
    img, radii, leaves, verts, m2, rs, (fc, fR, fs) = _fused_cuda(sc, dev, need_grad=False, exact=True)
    keys, vals, ranges, n = R.export_last_binning()
    means3D, opac, scales, cov = g.bind_activate(rs, leaves["_xyz"], leaves["_rotation"], leaves["_scaling"],
                                                 leaves["_opacity"], sc["params"]["binding"].to(dev), fc, fR, fs)
    act, _, _, _ = h.avatar_activated(sc)
    rel = lambda a, b: float((a - b).abs().max() / b.abs().max())  # noqa: E731
    assert rel(means3D.cpu(), act["means3D"]) < 2e-6
    assert rel(scales.cpu(), act["scales"]) < 2e-6
    assert rel(opac.cpu(), act["opacities"]) < 2e-6
    cam = sc["cam"]
    shs = torch.cat((sc["params"]["_features_dc"], sc["params"]["_features_rest"]), dim=1).contiguous()
    st = orc.forward(means3D.cpu().numpy(), opac.cpu().numpy(), cam.world_view_transform.numpy(),
                     cam.full_proj_transform.numpy(), cam.camera_center.numpy(), sc["W"], sc["H"], cam.tanfovx,
                     cam.tanfovy, sc["bg"].numpy(), shs=shs.numpy(), sh_degree=3, cov3D_precomp=cov.cpu().numpy())
    assert np.array_equal(radii.cpu().numpy(), st.radii)
    assert n == st.N
    assert np.array_equal(keys.cpu().numpy().view(np.uint64), st.keys_sorted)
    assert np.array_equal(vals.cpu().numpy().view(np.uint32), st.vals_sorted)
    h.assert_image_close(img.cpu().numpy(), st.out_color, "fused image vs oracle(exported activation)")
    # (iii) against the eager getters (quaternion product route of the reference)
    st2 = orc.forward(act["means3D"].numpy(), act["opacities"].numpy(), cam.world_view_transform.numpy(),
                      cam.full_proj_transform.numpy(), cam.camera_center.numpy(), sc["W"], sc["H"], cam.tanfovx,
                      cam.tanfovy, sc["bg"].numpy(), shs=act["shs"].contiguous().numpy(), sh_degree=3,
                      scales=act["scales"].numpy(), rotations=act["rotations"].numpy())
    assert (radii.cpu().numpy() != st2.radii).mean() < 1e-3  # ceil() knife edges only
    # R_face * R(q) (fused) vs R(q_face (x) q) (eager) round differently -> a handful of radius/threshold flips
    h.assert_image_close(img.cpu().numpy(), st2.out_color, "fused image vs eager-getter oracle", frac=2e-4)


def test_fused_binding_backward_matches_eager_autograd_through_oracle():
    """Gradients of the fused op w.r.t. the RAW parameters and the mesh VERTICES equal autograd through the eager
    getters (quaternion detour included) chained into the oracle rasterizer (SURVEY.md 7.4-5)."""
    dev = _dev()
    sc = h.avatar_scene(P=6_000, W=320, H=240, seed=2, n_lat=14, n_lon=24)
    gout = torch.randn(3, sc["H"], sc["W"], generator=torch.Generator().manual_seed(4))
    # reference chain on CPU
    from oracle import rasterizer as orc
    from gaussianavatars_b200 import GaussianRasterizationSettings

    act, leaves_ref, verts_ref, _ = h.avatar_activated(sc, requires_grad=True)
    cam = sc["cam"]
    rs_cpu = GaussianRasterizationSettings(sc["H"], sc["W"], cam.tanfovx, cam.tanfovy, sc["bg"], 1.0,
                                           cam.world_view_transform, cam.full_proj_transform, 3, cam.camera_center,
                                           False, False)
    Fn = orc.make_autograd_function()
    m2_ref = torch.zeros(sc["params"]["_xyz"].shape[0], 3, requires_grad=True)
    img_ref, _ = Fn.apply(act["means3D"], m2_ref, act["shs"].contiguous(), None, act["opacities"], act["scales"],
                          act["rotations"], None, rs_cpu)
    (img_ref * gout).sum().backward()
    # fused CUDA
    img, radii, leaves, verts, m2, _, _ = _fused_cuda(sc, dev, need_grad=True, exact=False)
    (img * gout.to(dev)).sum().backward()
    torch.cuda.synchronize()
    h.assert_image_close(img.detach().cpu().numpy(), img_ref.detach().numpy(), "fused image", frac=2e-4)
    for k in leaves:
        h.assert_grad_close(leaves[k].grad.cpu().numpy(), leaves_ref[k].grad.numpy(), f"dL/d{k}", rtol=3e-3)
    h.assert_grad_close(m2.grad.cpu().numpy(), m2_ref.grad.numpy(), "dL/dmeans2D", rtol=3e-3)
    h.assert_grad_close(verts.grad.cpu().numpy(), verts_ref.grad.numpy(), "dL/dverts (through the face frame)", rtol=5e-3,
                        frac=5e-3)


def test_fused_identity_binding_equals_plain_model():
    """binding=None: plain GaussianModel semantics (exp / sigmoid / normalize only)."""
    import gaussianavatars_b200 as g

    dev = _dev()
    scene = h.random_scene(3_000, 192, 144, sh_degree=2, seed=6, scale_shift=0.6)
    st = h.oracle_forward(scene)
    raw = scene["raw"]
    rs = h.cuda_settings(scene, dev)
    img, radii = g.rasterize_bound(rs, raw["_xyz"].to(dev), raw["_rotation"].to(dev), (raw["_scaling"] + 0.6).to(dev),
                                   raw["_opacity"].to(dev), raw["_features_dc"].to(dev), raw["_features_rest"].to(dev))
    assert (radii.cpu().numpy() != st.radii).mean() < 2e-3
    h.assert_image_close(img.cpu().numpy(), st.out_color, "identity-binding fused image", frac=2e-4)


def test_render_dropin_dict_and_routes_agree():
    """render() returns the reference's dict; fused route == reference route (eager getters on the GPU)."""
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.model import MeshBoundGaussians
    from gaussianavatars_b200.renderer import render

    dev = _dev()
    sc = h.avatar_scene(P=8_000, W=352, H=256, seed=3, n_lat=14, n_lon=24)

    class Pipe:
        debug = False
        compute_cov3D_python = False
        convert_SHs_python = False

    outs = []
    for fused in (True, False):
        pc = MeshBoundGaussians(sc["params"], 3, sc["verts"], sc["faces"], device=dev, requires_grad=True)
        pc.select_mesh_by_timestep(0)
        out = render(sc["cam"], pc, Pipe, sc["bg"].to(dev), fused=fused)
        assert set(out) == {"render", "viewspace_points", "visibility_filter", "radii"}
        assert out["render"].shape == (3, sc["H"], sc["W"]) and out["radii"].dtype == torch.int32
        out["render"].square().sum().backward()
        outs.append((out, pc))
    (o1, p1), (o2, p2) = outs
    h.assert_image_close(o1["render"].detach().cpu().numpy(), o2["render"].detach().cpu().numpy(), "fused vs eager route",
                         frac=2e-4)
    assert (o1["visibility_filter"] != o2["visibility_filter"]).float().mean() < 1e-3
    h.assert_grad_close(p1._xyz.grad.cpu().numpy(), p2._xyz.grad.cpu().numpy(), "route dL/d_xyz", rtol=3e-3)
    h.assert_grad_close(o1["viewspace_points"].grad.cpu().numpy(), o2["viewspace_points"].grad.cpu().numpy(),
                        "route viewspace grad", rtol=3e-3)


def test_full_size_properties_1080p():
    """BASELINE config-2 size (100k splats, 1920x1080, SH3) through size-independent properties: permutation
    invariance (distinct depths), sortedness of the key stream, blend weights + final T = 1 via a white-colour
    render, determinism of the forward."""
    import gaussianavatars_b200 as g
    from gaussianavatars_b200 import rasterizer as R
    from gaussianavatars_b200 import synthetic as syn
    from gaussianavatars_b200.model import MeshBoundGaussians
    from gaussianavatars_b200.renderer import render

    dev = _dev()
    verts, faces = syn.head_mesh()
    params = syn.avatar_splats(100_000, n_faces=faces.shape[0], seed=0, sh_degree=3)
    cam = syn.orbit_camera(1920, 1080)

    class Pipe:
        debug = False
        compute_cov3D_python = False
        convert_SHs_python = False

    bg = torch.zeros(3, device=dev)
    R.set_exact_binning(False)
    R.keep_last_state(True)
    pc = MeshBoundGaussians(params, 3, verts, faces, device=dev)
    pc.select_mesh_by_timestep(0)
    with torch.no_grad():
        o1 = render(cam, pc, Pipe, bg)
        keys, vals, ranges, n = R.export_last_binning()
        k = keys.cpu().numpy().view(np.uint64)
        assert n > 100_000 and (np.diff(k.astype(np.float64)) >= 0).all() and (k[1:] >= k[:-1]).all(), "key stream not sorted"
        r = ranges.cpu().numpy().view(np.uint32)
        assert int((r[:, 1] - r[:, 0]).sum()) == n, "tile ranges do not partition the stream"
        o1b = render(cam, pc, Pipe, bg)
        assert torch.equal(o1["render"], o1b["render"]), "forward is not deterministic"
        # permutation invariance
        perm = torch.randperm(100_000, generator=torch.Generator().manual_seed(0))
        params_p = {k_: v[perm] for k_, v in params.items()}
        pc2 = MeshBoundGaussians(params_p, 3, verts, faces, device=dev)
        pc2.select_mesh_by_timestep(0)
        o2 = render(cam, pc2, Pipe, bg)
        assert torch.equal(o2["radii"], o1["radii"][perm.to(dev)])
        d = (o2["render"] - o1["render"]).abs()
        assert float(d.max()) < 0.1 and float((d > 1e-4).float().mean()) < 3e-3  # ~1500 equal-depth pairs (birthday) reorder
        # weights + T_final = 1: white splats over black bg, then over white bg
        white = torch.ones(100_000, 3, device=dev)
        a = render(cam, pc, Pipe, torch.zeros(3, device=dev), override_color=white)["render"]
        b = render(cam, pc, Pipe, torch.ones(3, device=dev), override_color=white)["render"]
        assert float((b - 1.0).abs().max()) < 2e-5, "sum of blend weights + final transmittance != 1"
        assert float(a.max()) <= 1.0 + 1e-5


def test_face_frame_kernel_matches_reference_math_and_autograd():
    """gab200_face_frame_{forward,backward} vs the torch restatement of compute_face_orientation
    (utils/graphics_utils.py:116-135) and its autograd."""
    import gaussianavatars_b200 as g
    from gaussianavatars_b200 import synthetic as syn
    from oracle import binding as ob

    dev = _dev()
    verts, faces = syn.head_mesh(n_lat=20, n_lon=36, seed=3)
    verts = syn.pose_mesh(verts, 5)
    v_ref = verts.double().clone().requires_grad_(True)
    fr = ob.update_mesh_properties(v_ref, faces)
    gen = torch.Generator().manual_seed(0)
    F = faces.shape[0]
    g_c, g_R, g_s = torch.randn(F, 3, generator=gen), torch.randn(F, 3, 3, generator=gen), torch.randn(F, 1, generator=gen)
    ((fr["face_center"] * g_c.double()).sum() + (fr["face_orien_mat"] * g_R.double()).sum()
     + (fr["face_scaling"] * g_s.double()).sum()).backward()
    v = verts.to(dev).requires_grad_(True)
    fc, fR, fs = g.face_frame(v, faces.to(dev))
    assert torch.allclose(fc.cpu().double(), fr["face_center"].detach(), atol=1e-7, rtol=1e-5)
    assert torch.allclose(fR.cpu().double(), fr["face_orien_mat"].detach(), atol=2e-6, rtol=1e-5)
    assert torch.allclose(fs.cpu().double(), fr["face_scaling"].detach(), atol=1e-8, rtol=1e-5)
    ((fc * g_c.to(dev)).sum() + (fR * g_R.to(dev)).sum() + (fs * g_s.to(dev)).sum()).backward()
    h.assert_grad_close(v.grad.cpu().numpy(), v_ref.grad.numpy(), "dL/dverts of the face frame", rtol=1e-4, frac=0.0)


def test_l1_loss_u8_kernel():
    import gaussianavatars_b200 as g

    dev = _dev()
    gen = torch.Generator().manual_seed(0)
    for shape in ((3, 1080, 1920), (3, 33, 17), (5,)):
        img = torch.rand(shape, generator=gen).to(dev).requires_grad_(True)
        gt = torch.randint(0, 256, shape, generator=gen, dtype=torch.uint8).to(dev)
        loss = g.l1_loss_u8(img, gt)
        (loss * 2.0).backward()
        ref_in = img.detach().clone().requires_grad_(True)
        ref = (ref_in - gt.float() / 255.0).abs().mean()
        (ref * 2.0).backward()
        assert abs(float(loss) - float(ref)) < 1e-5
        assert torch.allclose(img.grad, ref_in.grad, atol=1e-9)


@pytest.mark.parametrize("active_deg,mod", [(1, 1.0), (2, 0.8), (0, 1.0)])
def test_active_degree_below_max_and_scale_modifier_backward(active_deg, mod):
    """train.py raises active_sh_degree every 1000 its while 16 coefficients are stored (M=16, D<3): unused
    coefficients must get zero gradient; scale_modifier != 1 keeps the reference's dL/dscale convention."""
    import gaussianavatars_b200 as g
    from oracle import rasterizer as orc

    dev = _dev()
    scene = h.random_scene(2_500, 550 // 2, 802 // 4, sh_degree=active_deg, seed=13, scale_shift=0.8, max_sh_degree=3)
    cam = scene["cam"]
    kw = dict(shs=scene["shs"].numpy(), sh_degree=active_deg, scales=scene["scales"].numpy(),
              rotations=scene["rotations"].numpy(), scale_modifier=mod)
    args = (cam.world_view_transform.numpy(), cam.full_proj_transform.numpy(), cam.camera_center.numpy())
    st = orc.forward(scene["means3D"].numpy(), scene["opacities"].numpy(), *args, scene["W"], scene["H"], cam.tanfovx,
                     cam.tanfovy, scene["bg"].numpy(), **kw)
    gout = torch.randn(3, scene["H"], scene["W"], generator=torch.Generator().manual_seed(1))
    ref = orc.backward(st, gout.numpy(), scene["means3D"].numpy(), *args, cam.tanfovx, cam.tanfovy, scene["bg"].numpy(), **kw)
    img, radii, t, m2 = _run_cuda(scene, dev, need_grad=True, exact=False, scale_modifier=mod)
    assert scene["shs"].shape[1] == 16
    h.assert_image_close(img.detach().cpu().numpy(), st.out_color, "image (D < max degree)")
    (img * gout.to(dev)).sum().backward()
    ke = A.knife_edges(st)
    for name in ("means3D", "scales", "rotations", "opacities", "shs"):
        _explained_close(t[name].grad.cpu().numpy(), ref[name], A.affected(ke, name), f"dL/d{name}")
    nb = (active_deg + 1) ** 2
    assert float(t["shs"].grad[:, nb:].abs().sum()) == 0.0


def test_fused_route_with_override_color_and_benchmark_resolution():
    """render(..., override_color=...) on the fused route at the reference's default benchmark size 550x802
    (fps_benchmark_demo.py:78-80; 550 is not a multiple of 16)."""
    from gaussianavatars_b200.model import MeshBoundGaussians
    from gaussianavatars_b200.renderer import render

    dev = _dev()
    sc = h.avatar_scene(P=9_000, W=550, H=802, seed=4, n_lat=14, n_lon=24, scale_gain=1.5)

    class Pipe:
        debug = False
        compute_cov3D_python = False
        convert_SHs_python = False

    outs = []
    for fused in (True, False):
        pc = MeshBoundGaussians(sc["params"], 3, sc["verts"], sc["faces"], device=dev, requires_grad=True)
        pc.select_mesh_by_timestep(0)
        col = torch.rand(9_000, 3, generator=torch.Generator().manual_seed(5)).to(dev).requires_grad_(True)
        out = render(sc["cam"], pc, Pipe, sc["bg"].to(dev), override_color=col, fused=fused)
        out["render"].square().sum().backward()
        outs.append((out, pc, col))
    (o1, p1, c1), (o2, p2, c2) = outs
    assert o1["render"].shape == (3, 802, 550)
    h.assert_image_close(o1["render"].detach().cpu().numpy(), o2["render"].detach().cpu().numpy(), "override_color routes",
                         frac=2e-4)
    h.assert_grad_close(c1.grad.cpu().numpy(), c2.grad.cpu().numpy(), "dL/doverride_color", rtol=3e-3)
    h.assert_grad_close(p1._xyz.grad.cpu().numpy(), p2._xyz.grad.cpu().numpy(), "dL/d_xyz", rtol=3e-3)
    assert p1._features_dc.grad is None or float(p1._features_dc.grad.abs().sum()) == 0.0
