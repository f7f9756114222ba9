"""ctypes front-end of the C oracle (oracle/splat_oracle.c).

TEST INFRASTRUCTURE -- parity unpinned for the rasterizer proper (see the header of
splat_oracle.c).  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs may import this module; gaussianavatars_b200 never does.

The Python surface mirrors the stage boundaries of the reference module
(SURVEY.md Appendix B.1-B.5) so that tests can compare stage by stage, and
`OracleRasterizer` mirrors `_RasterizeGaussians` (Appendix B.6) as a CPU
torch.autograd.Function so that the reference's render() data flow
(gaussian_renderer/__init__.py:19-101) can be replayed on CPU tensors.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libsplat_oracle.so")
_lib = None


def build(force: bool = False) -> str:
    """Compile the oracle with gcc (seconds).  Called by __graft_entry__.build() and lazily by load()."""
    src = os.path.join(_HERE, "splat_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.run(["make", "-C", _HERE, "-B", "libsplat_oracle.so"], check=True, capture_output=True)
    return _LIB_PATH


def load():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.oracle_preprocess.restype = C.c_int64
        _lib.oracle_tile_bits.restype = C.c_uint32
        _lib.oracle_tile_bits.argtypes = [C.c_uint32]
    return _lib


def set_threads(n: int) -> int:
    """OpenMP threads of the C oracle (returns the count in effect)."""
    lib = load()
    lib.oracle_set_threads.restype = C.c_int
    return int(lib.oracle_set_threads(C.c_int(int(n))))


def _p(a: Optional[np.ndarray]):
    if a is None:
        return C.c_void_p(0)
    assert a.flags["C_CONTIGUOUS"], "oracle needs contiguous arrays"
    return C.c_void_p(a.ctypes.data)


def _f32(a) -> Optional[np.ndarray]:
    if a is None:
        return None
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32))


def tile_bits(n_tiles: int) -> int:
    return int(load().oracle_tile_bits(n_tiles))


@dataclass
class OracleState:
    """Everything the reference module keeps between forward and backward (its three byte buffers)."""
    P: int
    W: int
    H: int
    N: int
    depths: np.ndarray
    radii: np.ndarray
    xy: np.ndarray
    conic_opacity: np.ndarray
    rgb: np.ndarray
    cov3D: np.ndarray
    clamped: np.ndarray
    tiles_touched: np.ndarray
    offsets: np.ndarray
    keys_unsorted: np.ndarray
    vals_unsorted: np.ndarray
    keys_sorted: np.ndarray
    vals_sorted: np.ndarray
    ranges: np.ndarray
    out_color: np.ndarray
    final_T: np.ndarray
    n_contrib: np.ndarray


def forward(means3D, opacities, viewmatrix, projmatrix, campos, W, H, tanfovx, tanfovy, bg, *, shs=None,
            sh_degree=0, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None,
            scale_modifier=1.0) -> OracleState:
    lib = load()
    means3D = _f32(means3D)
    P = means3D.shape[0]
    opacities = _f32(opacities).reshape(-1)
    shs, colors_precomp = _f32(shs), _f32(colors_precomp)
    scales, rotations, cov3D_precomp = _f32(scales), _f32(rotations), _f32(cov3D_precomp)
    V, Pm, cam, bg = _f32(viewmatrix).reshape(16), _f32(projmatrix).reshape(16), _f32(campos).reshape(3), _f32(bg).reshape(3)
    M = 0 if shs is None else shs.shape[1]
    assert (shs is None) != (colors_precomp is None)
    assert (cov3D_precomp is None) != (scales is None or rotations is None)
    depths = np.zeros(P, np.float32)
    radii = np.zeros(P, np.int32)
    xy = np.zeros((P, 2), np.float32)
    conic_opacity = np.zeros((P, 4), np.float32)
    rgb = np.zeros((P, 3), np.float32)
    cov3D = np.zeros((P, 6), np.float32)
    clamped = np.zeros((P, 3), np.uint8)
    tiles = np.zeros(P, np.uint32)
    N = lib.oracle_preprocess(C.c_int(P), C.c_int(sh_degree), C.c_int(M), _p(means3D), _p(scales),
                              C.c_float(scale_modifier), _p(rotations), _p(opacities), _p(shs), _p(colors_precomp),
                              _p(cov3D_precomp), _p(V), _p(Pm), _p(cam), C.c_int(W), C.c_int(H),
                              C.c_float(tanfovx), C.c_float(tanfovy), _p(depths), _p(radii), _p(xy),
                              _p(conic_opacity), _p(rgb), _p(cov3D), _p(clamped), _p(tiles))
    N = int(N)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    offsets = np.zeros(P, np.uint32)
    ku = np.zeros(max(N, 1), np.uint64)
    vu = np.zeros(max(N, 1), np.uint32)
    ks = np.zeros(max(N, 1), np.uint64)
    vs = np.zeros(max(N, 1), np.uint32)
    ranges = np.zeros((gx * gy, 2), np.uint32)
    lib.oracle_bin_sort(C.c_int(P), C.c_int(W), C.c_int(H), _p(depths), _p(radii), _p(xy), _p(tiles), _p(offsets),
                        C.c_int64(N), _p(ku), _p(vu), _p(ks), _p(vs), _p(ranges))
    out = np.zeros((3, H, W), np.float32)
    final_T = np.zeros((H, W), np.float32)
    n_contrib = np.zeros((H, W), np.uint32)
    lib.oracle_blend_forward(C.c_int(W), C.c_int(H), _p(ranges), _p(vs), _p(xy), _p(conic_opacity), _p(rgb), _p(bg),
                             _p(out), _p(final_T), _p(n_contrib))
    return OracleState(P, W, H, N, depths, radii, xy, conic_opacity, rgb, cov3D, clamped, tiles, offsets, ku[:N],
                       vu[:N], ks[:N], vs[:N], ranges, out, final_T, n_contrib)


def backward(st: OracleState, dL_dpix, means3D, viewmatrix, projmatrix, campos, tanfovx, tanfovy, bg, *, shs=None,
             sh_degree=0, scales=None, rotations=None, scale_modifier=1.0):
    """Returns dict with the 8 gradients of Appendix B.6 (numpy float32) plus the 2-D intermediates."""
    lib = load()
    P, W, H = st.P, st.W, st.H
    means3D = _f32(means3D)
    shs, scales, rotations = _f32(shs), _f32(scales), _f32(rotations)
    V, Pm, cam, bg = _f32(viewmatrix).reshape(16), _f32(projmatrix).reshape(16), _f32(campos).reshape(3), _f32(bg).reshape(3)
    dL_dpix = _f32(dL_dpix)
    M = 0 if shs is None else shs.shape[1]
    g_mean2D = np.zeros((P, 2), np.float32)
    g_conic = np.zeros((P, 3), np.float32)
    g_opac = np.zeros((P, 1), np.float32)
    g_color = np.zeros((P, 3), np.float32)
    vs = np.ascontiguousarray(st.vals_sorted) if st.N > 0 else np.zeros(1, np.uint32)
    lib.oracle_blend_backward(C.c_int(P), C.c_int(W), C.c_int(H), _p(st.ranges), _p(vs), _p(st.xy),
                              _p(st.conic_opacity), _p(st.rgb), _p(bg), _p(st.final_T), _p(st.n_contrib),
                              _p(dL_dpix), _p(g_mean2D), _p(g_conic), _p(g_opac), _p(g_color))
    g = preprocess_backward(st, g_mean2D, g_conic, g_color, means3D, viewmatrix, projmatrix, campos, tanfovx, tanfovy,
                            shs=shs, sh_degree=sh_degree, scales=scales, rotations=rotations,
                            scale_modifier=scale_modifier)
    g_means2D = np.zeros((P, 3), np.float32)
    g_means2D[:, :2] = g_mean2D
    return dict(g, means2D=g_means2D, colors_precomp=g_color, opacities=g_opac, conic=g_conic)


def preprocess_backward(st: OracleState, dL_dmean2D, dL_dconic, dL_dcolor, means3D, viewmatrix, projmatrix, campos,
                        tanfovx, tanfovy, *, shs=None, sh_degree=0, scales=None, rotations=None, scale_modifier=1.0,
                        radii=None, clamped=None):
    """Stage 5 alone: the per-splat upstream dL/dmean2D (P,2, NDC units), dL/dconic (P,3, the off-diagonal entry
    stored once) and dL/dcolor (P,3) -> dict of means3D, cov3D_precomp, shs, scales and rotations gradients (numpy
    float32; None where the input is absent).  `radii` / `clamped` replace the state's visibility and colour clamp
    bits (another forward's decisions)."""
    lib = load()
    P, W, H = st.P, st.W, st.H
    means3D = _f32(means3D)
    shs, scales, rotations = _f32(shs), _f32(scales), _f32(rotations)
    V, Pm, cam = _f32(viewmatrix).reshape(16), _f32(projmatrix).reshape(16), _f32(campos).reshape(3)
    radii = st.radii if radii is None else np.ascontiguousarray(radii, np.int32)
    clamped = st.clamped if clamped is None else np.ascontiguousarray(clamped, np.uint8)
    g_mean2D, g_conic, g_color = _f32(dL_dmean2D), _f32(dL_dconic), _f32(dL_dcolor)
    M = 0 if shs is None else shs.shape[1]
    g_means3D = np.zeros((P, 3), np.float32)
    g_cov3D = np.zeros((P, 6), np.float32)
    g_sh = np.zeros((P, M, 3), np.float32) if shs is not None else None
    g_scales = np.zeros((P, 3), np.float32) if scales is not None else None
    g_rots = np.zeros((P, 4), np.float32) if scales is not None else None
    lib.oracle_preprocess_backward(C.c_int(P), C.c_int(sh_degree), C.c_int(M), _p(means3D), _p(radii), _p(shs),
                                   _p(clamped), _p(scales), _p(rotations), C.c_float(scale_modifier),
                                   _p(st.cov3D), _p(V), _p(Pm), _p(cam), C.c_int(W), C.c_int(H), C.c_float(tanfovx),
                                   C.c_float(tanfovy), _p(g_mean2D), _p(g_conic), _p(g_color), _p(g_means3D),
                                   _p(g_cov3D), _p(g_sh), _p(g_scales), _p(g_rots))
    return dict(means3D=g_means3D, shs=g_sh, scales=g_scales, rotations=g_rots, cov3D_precomp=g_cov3D)


def mark_visible(means3D, viewmatrix):
    lib = load()
    means3D = _f32(means3D)
    out = np.zeros(means3D.shape[0], np.uint8)
    lib.oracle_mark_visible(C.c_int(means3D.shape[0]), _p(means3D), _p(_f32(viewmatrix).reshape(16)), _p(out))
    return out.astype(bool)


# --------------------------------------------------------------------------- #
# CPU autograd.Function with the surface of the reference module's wrapper
# --------------------------------------------------------------------------- #
def make_autograd_function():
    import torch

    class OracleRasterize(torch.autograd.Function):
        @staticmethod
        def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, rs):
            def n(t):
                return None if t is None or t.numel() == 0 else t.detach().cpu().numpy()

            st = forward(n(means3D), n(opacities), n(rs.viewmatrix), n(rs.projmatrix), n(rs.campos), rs.image_width,
                         rs.image_height, rs.tanfovx, rs.tanfovy, n(rs.bg), shs=n(sh), sh_degree=rs.sh_degree,
                         colors_precomp=n(colors_precomp), scales=n(scales), rotations=n(rotations),
                         cov3D_precomp=n(cov3Ds_precomp), scale_modifier=rs.scale_modifier)
            ctx.st, ctx.rs = st, rs
            ctx.save_for_backward(means3D, sh, scales, rotations)
            ctx.has = (colors_precomp is not None and colors_precomp.numel() > 0,
                       cov3Ds_precomp is not None and cov3Ds_precomp.numel() > 0)
            color = torch.from_numpy(st.out_color.copy())
            radii = torch.from_numpy(st.radii.copy())
            ctx.mark_non_differentiable(radii)
            return color, radii

        @staticmethod
        def backward(ctx, grad_color, _):
            means3D, sh, scales, rotations = ctx.saved_tensors
            rs, st = ctx.rs, ctx.st

            def n(t):
                return None if t is None or t.numel() == 0 else t.detach().cpu().numpy()

            g = backward(st, n(grad_color.contiguous()), n(means3D), n(rs.viewmatrix), n(rs.projmatrix), n(rs.campos),
                         rs.tanfovx, rs.tanfovy, n(rs.bg), shs=n(sh), sh_degree=rs.sh_degree, scales=n(scales),
                         rotations=n(rotations), scale_modifier=rs.scale_modifier)

            def t(a):
                return None if a is None else torch.from_numpy(a)

            has_colors, has_cov = ctx.has
            return (t(g["means3D"]), t(g["means2D"]), t(g["shs"]), t(g["colors_precomp"]) if has_colors else None,
                    t(g["opacities"]), t(g["scales"]), t(g["rotations"]), t(g["cov3D_precomp"]) if has_cov else None,
                    None)

    return OracleRasterize
