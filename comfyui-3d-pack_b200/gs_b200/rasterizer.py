"""Host-side mirror of the `diff_gaussian_rasterization` Python interface.

Same names, argument meaning and error behaviour as the package the reference
imports at MVs_Algorithms/GaussianSplatting/main_3DGS_renderer.py:840-843 and
calls at :849-864 / :927-936 (also LGM/core/gs.py:57-84,
TriplaneGaussian/models/renderer.py:209-304, TRELLIS gaussian_render.py:62-137):

    GaussianRasterizationSettings(image_height, image_width, tanfovx, tanfovy, bg,
        scale_modifier, viewmatrix, projmatrix, sh_degree, campos, prefiltered, debug)
    GaussianRasterizer(raster_settings)(means3D, means2D, opacities, shs=None,
        colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None)
        -> (color[3,H,W], radii[N] int32, depth[1,H,W], alpha[1,H,W])

PyTorch is plumbing only (device memory, streams, autograd glue); all compute is
the sm_90a library behind include/gs_b200.h.  No CPU path exists.
"""
from typing import NamedTuple, Optional
import ctypes as C

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from ._lib import stream as _stream


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


def _dev_f32(t: torch.Tensor, what: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{what} must be a torch.Tensor")
    if not t.is_cuda:
        raise RuntimeError(f"{what} must be a CUDA tensor (gs_b200 has no CPU path)")
    t = t.detach()
    if t.dtype != torch.float32:
        t = t.float()
    if not t.is_contiguous():
        t = t.contiguous()
    if t.data_ptr() % 16 != 0:
        t = t.clone()
    return t


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


class _Buffers:
    """Allocator callback target: torch owns every buffer (SURVEY §8b ownership).

    The callback closes over the two lists only (never over `self`), so there is no
    reference cycle and the buffers are released by refcount the moment the autograd
    node / caller drops them — a cycle here would park ~120 MB per view until the GC runs.
    """

    def __init__(self, device):
        saved, scratch = [], []       # saved: geom/binning/image (live until backward); scratch: per call

        def _alloc(user, tag, nbytes):
            try:
                t = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
            except Exception:  # noqa: BLE001  (reported by the C side as an allocation failure)
                return None
            (scratch if tag == _lib.BUF_SCRATCH else saved).append(t)
            return t.data_ptr()

        self.saved, self.scratch = saved, scratch
        self.cb = _lib.ALLOC_FN(_alloc)


def _make_view(rs: GaussianRasterizationSettings, keep: list) -> _lib.View:
    bg = _dev_f32(rs.bg, "bg"); vm = _dev_f32(rs.viewmatrix, "viewmatrix")
    pm = _dev_f32(rs.projmatrix, "projmatrix"); cp = _dev_f32(rs.campos, "campos")
    if bg.numel() != 3 or vm.numel() != 16 or pm.numel() != 16 or cp.numel() != 3:
        raise ValueError("bg[3], viewmatrix[4,4], projmatrix[4,4], campos[3] expected")
    keep += [bg, vm, pm, cp]
    return _lib.View(int(rs.image_height), int(rs.image_width), float(rs.tanfovx), float(rs.tanfovy),
                     bg.data_ptr(), float(rs.scale_modifier), vm.data_ptr(), pm.data_ptr(), int(rs.sh_degree),
                     cp.data_ptr(), int(bool(rs.prefiltered)), int(bool(rs.debug)))


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings):
        rs = raster_settings
        dev = means3D.device
        if dev.type != "cuda":
            raise RuntimeError("means3D must be a CUDA tensor (gs_b200 has no CPU path)")
        with torch.cuda.device(dev):
            m3 = _dev_f32(means3D, "means3D")
            N = m3.shape[0]
            sh_ = None if sh is None else _dev_f32(sh, "shs")
            cp_ = None if colors_precomp is None else _dev_f32(colors_precomp, "colors_precomp")
            op_ = _dev_f32(opacities, "opacities")
            sc_ = None if scales is None else _dev_f32(scales, "scales")
            ro_ = None if rotations is None else _dev_f32(rotations, "rotations")
            cv_ = None if cov3Ds_precomp is None else _dev_f32(cov3Ds_precomp, "cov3D_precomp")
            M = 0 if sh_ is None else int(sh_.shape[1])
            H, W = int(rs.image_height), int(rs.image_width)
            color = torch.empty(3, H, W, dtype=torch.float32, device=dev)
            depth = torch.empty(1, H, W, dtype=torch.float32, device=dev)
            alpha = torch.empty(1, H, W, dtype=torch.float32, device=dev)
            radii = torch.empty(N, dtype=torch.int32, device=dev)
            keep = []
            view = _make_view(rs, keep)
            bufs = _Buffers(dev)
            state = _lib.State()
            rc = _lib.lib.gs_b200_rasterize_forward(
                C.byref(view), N, M, _ptr(m3), _ptr(sh_), _ptr(cp_), _ptr(op_), _ptr(sc_), _ptr(ro_), _ptr(cv_),
                _ptr(color), _ptr(depth), _ptr(alpha), _ptr(radii), bufs.cb, None, C.byref(state), _stream())
            bufs.scratch.clear()
            _lib.check(rc)
        ctx.rs = rs
        ctx.state = state
        ctx.bufs = bufs
        ctx.view_keep = keep
        # save_for_backward (not plain attributes): an in-place update of a parameter between forward and backward then
        # trips autograd's version check instead of silently pairing new parameters with the saved binning state
        ctx.save_for_backward(m3, sh_, cp_, op_, sc_, ro_, cv_, radii)
        ctx.M = M
        ctx.mark_non_differentiable(radii)
        return color, radii, depth, alpha

    @staticmethod
    def backward(ctx, g_color, g_radii, g_depth, g_alpha):
        rs = ctx.rs
        m3, sh_, cp_, op_, sc_, ro_, cv_, radii = ctx.saved_tensors
        dev = m3.device
        N = m3.shape[0]
        H, W = int(rs.image_height), int(rs.image_width)
        with torch.cuda.device(dev):
            def up(g, shape):
                return torch.zeros(shape, dtype=torch.float32, device=dev) if g is None else _dev_f32(g, "grad")
            gc, gd, ga = up(g_color, (3, H, W)), up(g_depth, (1, H, W)), up(g_alpha, (1, H, W))
            d_m3 = torch.empty_like(m3)
            d_m2 = torch.empty(N, 3, dtype=torch.float32, device=dev)
            d_sh = None if sh_ is None else torch.empty_like(sh_)
            d_cp = None if cp_ is None else torch.empty_like(cp_)
            d_op = torch.empty_like(op_)
            d_sc = None if sc_ is None else torch.empty_like(sc_)
            d_ro = None if ro_ is None else torch.empty_like(ro_)
            d_cv = None if cv_ is None else torch.empty_like(cv_)
            keep = []
            view = _make_view(rs, keep)
            bufs = _Buffers(dev)
            rc = _lib.lib.gs_b200_rasterize_backward(
                C.byref(view), N, ctx.M, _ptr(m3), _ptr(sh_), _ptr(cp_), _ptr(op_), _ptr(sc_), _ptr(ro_), _ptr(cv_),
                _ptr(radii), C.byref(ctx.state), _ptr(gc), _ptr(gd), _ptr(ga),
                _ptr(d_m3), _ptr(d_m2), _ptr(d_sh), _ptr(d_cp), _ptr(d_op), _ptr(d_sc), _ptr(d_ro), _ptr(d_cv),
                0, bufs.cb, None, _stream())
            bufs.scratch.clear()
            _lib.check(rc)
        return d_m3, d_m2, d_sh, d_cp, d_op, d_sc, d_ro, d_cv, None


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings)


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        """Frustum test of the package (z > 0.2 in view space); bool [N]."""
        with torch.no_grad():
            vm = self.raster_settings.viewmatrix.float()
            z = positions.float() @ vm[:3, 2] + vm[3, 2]
            return z > 0.2

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        raster_settings = self.raster_settings
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                   cov3D_precomp, raster_settings)


def _view_of(bufs: _Buffers, ptr: int, count: int, dtype: torch.dtype) -> torch.Tensor:
    esz = torch.empty(0, dtype=dtype).element_size()
    for b in bufs.saved:
        off = ptr - b.data_ptr()
        if 0 <= off and off + count * esz <= b.numel():
            return b[off:off + count * esz].view(dtype)
    raise RuntimeError("state pointer not inside a saved buffer")


def forward_with_state(raster_settings, means3D, opacities, shs=None, colors_precomp=None, scales=None,
                       rotations=None, cov3D_precomp=None):
    """Forward only, plus the binning/image state as torch tensors (parity tests, benchmarks).

    Returns dict(color, radii, depth, alpha, recs[N,12] float32 (the 48-byte splat records: px, py, depth, radius bits |
    log2-scaled conic a', b', c', opacity | r, g, b, tiles_touched bits), point_list[P] int32, tile_keys[P] int32,
    sorted_keys[P] int64 (tile<<32 | float_bits(depth)), ranges[tiles,2] int32, n_contrib[H,W] int32, final_T[H,W],
    num_rendered).
    """
    class _Ctx:
        def mark_non_differentiable(self, *a):
            pass

        def save_for_backward(self, *a):
            self.saved_tensors = a
    ctx = _Ctx()
    color, radii, depth, alpha = _RasterizeGaussians.forward(
        ctx, means3D, None, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, raster_settings)
    st, bufs = ctx.state, ctx.bufs
    P = int(st.num_rendered)
    H, W = int(raster_settings.image_height), int(raster_settings.image_width)
    ntiles = st.tiles_x * st.tiles_y
    out = dict(color=color, radii=radii, depth=depth, alpha=alpha, num_rendered=P,
               ranges=_view_of(bufs, st.ranges, ntiles * 2, torch.int32).view(ntiles, 2),
               n_contrib=_view_of(bufs, st.n_contrib, H * W, torch.int32).view(H, W),
               final_T=_view_of(bufs, st.final_T, H * W, torch.float32).view(H, W))
    N = int(st.num_gaussians)
    out["recs"] = (_view_of(bufs, st.geom, N * 12, torch.float32).view(N, 12) if N > 0 else
                   torch.empty(0, 12, dtype=torch.float32, device=color.device))
    if P > 0:
        out["point_list"] = _view_of(bufs, st.point_list, P, torch.int32)
        out["tile_keys"] = _view_of(bufs, st.tile_keys, P, torch.int32)
        keys = torch.empty(P, dtype=torch.int64, device=color.device)
        _lib.check(_lib.lib.gs_b200_debug_sorted_keys(C.byref(st), C.c_void_p(keys.data_ptr()), _stream()))
        out["sorted_keys"] = keys
    else:
        z = torch.empty(0, dtype=torch.int32, device=color.device)
        out.update(point_list=z, tile_keys=z, sorted_keys=torch.empty(0, dtype=torch.int64, device=color.device))
    out["_keepalive"] = (ctx, bufs)
    return out


def set_tile_culling(mode: int) -> None:
    """0: the package's tile lists everywhere; 1 (default): culled lists in the multi-view step entries only;
    2: culled lists in `GaussianRasterizer` too.  Images are bit-identical in all modes (include/gs_b200.h)."""
    if _lib.lib.gs_b200_set_tile_culling(int(mode)) != 0:
        raise ValueError(_lib.last_error())


def get_tile_culling() -> int:
    return int(_lib.lib.gs_b200_get_tile_culling())


def sort_pairs_u32(keys: torch.Tensor, vals: Optional[torch.Tensor], begin_bit: int = 0, end_bit: int = 32):
    """CUB-free onesweep radix sort of int32-viewed u32 keys (+values); returns sorted (keys, vals)."""
    assert keys.is_cuda and keys.dtype == torch.int32 and keys.is_contiguous()
    n = keys.numel()
    k0 = keys.clone(); k1 = torch.empty_like(k0)
    v0 = None if vals is None else vals.clone(); v1 = None if vals is None else torch.empty_like(v0)
    scratch = torch.empty(max(int(_lib.lib.gs_b200_sort_scratch_bytes(n)), 256), dtype=torch.uint8, device=keys.device)
    alt = C.c_int32(0)
    with torch.cuda.device(keys.device):
        _lib.check(_lib.lib.gs_b200_sort_pairs_u32(_ptr(k0), _ptr(k1), _ptr(v0), _ptr(v1), n, begin_bit, end_bit,
                                                   _ptr(scratch), C.byref(alt), _stream()))
    return (k1, v1) if alt.value else (k0, v0)


def sort_pairs_segmented(keys: torch.Tensor, vals: torch.Tensor, seg_off, begin_bit: int = 0, end_bit: int = 32,
                         key_bias: Optional[torch.Tensor] = None, bias_stride: int = 0):
    """The binning's segmented sort (tests): segments [seg_off[i], seg_off[i+1]) of int32-viewed u32 keys + values,
    each sorted on its own by (key - key_bias[i * bias_stride]) mod 2^32; returns sorted (keys, vals)."""
    assert keys.is_cuda and keys.dtype == torch.int32 and keys.is_contiguous() and vals.shape == keys.shape
    k0, v0 = keys.clone(), vals.clone()
    k1, v1 = torch.empty_like(k0), torch.empty_like(v0)
    off = (C.c_int64 * len(seg_off))(*[int(x) for x in seg_off])
    alt = C.c_int32(0)
    with torch.cuda.device(keys.device):
        _lib.check(_lib.lib.gs_b200_debug_sort_segmented(_ptr(k0), _ptr(k1), _ptr(v0), _ptr(v1), off, len(seg_off) - 1,
                                                         begin_bit, end_bit, _ptr(key_bias), bias_stride, C.byref(alt),
                                                         _stream()))
    return (k1, v1) if alt.value else (k0, v0)


def bin_views(views: torch.Tensor, H: int, W: int, sh_degree: int, scale_modifier: float, means3D, shs, opacities,
              scales, rotations, tight: bool, lists: bool = True) -> dict:
    """The multi-view step's projection and binning (tests): views [V, 40] as the step entries take them.  Returns
    per view [V, N] radii, tiles_touched, spans [V, N, 4] (tight only), sorted_dkeys, sorted_ids, offsets and
    totals [V] (int64, host); with `lists` also ranges [V, tiles, 2] and point_list / tile_keys, each a list of V
    tensors.  u32 values are returned as int64."""
    V, N, M = views.shape[0], means3D.shape[0], shs.shape[1]
    dev = means3D.device
    ntiles = ((W + 15) // 16) * ((H + 15) // 16)
    ins = [_dev_f32(t, "input") for t in (views, means3D, shs, opacities, scales, rotations)]
    i32 = lambda *sh: torch.empty(*sh, dtype=torch.int32, device=dev)        # noqa: E731
    out = dict(radii=i32(V, N), tiles_touched=i32(V, N), spans=i32(V, N, 4) if tight else None, sorted_dkeys=i32(V, N),
               sorted_ids=i32(V, N), offsets=i32(V, N))
    totals = (C.c_int64 * V)()

    def call(pl, tk, rg):
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.gs_b200_debug_bin_views(
                V, H, W, sh_degree, scale_modifier, _ptr(ins[0]), N, M, *(_ptr(t) for t in ins[1:]), int(bool(tight)),
                *(_ptr(out[k]) for k in ("radii", "tiles_touched", "spans", "sorted_dkeys", "sorted_ids", "offsets")),
                totals, _ptr(rg), _ptr(pl), _ptr(tk), _stream()))
        torch.cuda.synchronize(dev)
    call(None, None, None)
    tot = [int(t) for t in totals]
    res = {}
    if lists:
        P = sum(tot)
        pl, tk, rg = i32(max(P, 1)), i32(max(P, 1)), i32(V, ntiles, 2)
        call(pl, tk, rg)
        if [int(t) for t in totals] != tot:
            raise RuntimeError("bin_views: pair totals changed between the two calls")
        cut = np.cumsum([0] + tot)
        res["point_list"] = [pl[cut[v]:cut[v + 1]].long() & 0xFFFFFFFF for v in range(V)]
        res["tile_keys"] = [tk[cut[v]:cut[v + 1]].long() & 0xFFFFFFFF for v in range(V)]
        res["ranges"] = rg.long() & 0xFFFFFFFF
    res.update({k: None if v is None else v.long() & 0xFFFFFFFF for k, v in out.items()})
    res["radii"], res["totals"] = out["radii"], tot
    return res


def knn_mean_dist2(points: torch.Tensor) -> torch.Tensor:
    """distCUDA2 replacement (simple_knn._C.distCUDA2, main_3DGS_renderer.py:408,419)."""
    pts = _dev_f32(points, "points")
    out = torch.empty(pts.shape[0], dtype=torch.float32, device=pts.device)
    with torch.cuda.device(pts.device):
        _lib.check(_lib.lib.gs_b200_knn_mean_dist2(_ptr(pts), pts.shape[0], _ptr(out), _stream()))
    return out
