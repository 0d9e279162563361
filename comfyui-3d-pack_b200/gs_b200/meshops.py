"""Host-side mirror of the `nvdiffrast.torch` surface the reference uses (SURVEY §8b):

    RasterizeCudaContext / RasterizeGLContext, rasterize, interpolate, texture, antialias

Call sites: MVs_Algorithms/DiffRastMesh/diff_mesh_renderer.py:45-138, FlexiCubes/flexicubes_renderer.py:46-66,
FlexiCubes/util.py:90-93, mesh_processer/mesh_utils.py:522-541.  All compute is the sm_90a library behind
include/dr_b200.h; PyTorch is device memory + autograd glue.  No CPU path.
"""
import ctypes as C
import weakref

import torch

from . import _lib

_P = lambda t: None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _f32(t, what):
    if not t.is_cuda:
        raise RuntimeError(f"{what} must be a CUDA tensor (gs_b200 mesh ops have no CPU path)")
    t = t.detach()
    if t.dtype != torch.float32:
        t = t.float()
    if not t.is_contiguous():
        t = t.contiguous()
    if t.data_ptr() % 16:
        t = t.clone()
    return t


def _i32(t, what):
    if not t.is_cuda:
        raise RuntimeError(f"{what} must be a CUDA tensor")
    if t.dtype != torch.int32:
        raise TypeError(f"{what} must be int32 (nvdiffrast contract)")
    return t.contiguous()


class RasterizeCudaContext:
    """Stateless here (scratch comes from torch's caching allocator per call), so creating one per call, as
    FlexiCubesRenderer.render_mesh does (flexicubes_renderer.py:46), costs nothing."""

    def __init__(self, device=None):
        self.device = device


class RasterizeGLContext(RasterizeCudaContext):
    def __init__(self, output_db=True, mode="automatic", device=None):
        super().__init__(device)


# ------------------------------------------------------------------------------------------------ rasterize
class _Rasterize(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos, tri, H, W):
        p = _f32(pos, "pos"); t = _i32(tri, "tri")
        B, V, _ = p.shape
        F = t.shape[0]
        dev = p.device
        with torch.cuda.device(dev):
            rast = torch.empty(B, H, W, 4, device=dev); db = torch.empty(B, H, W, 4, device=dev)
            scratch = torch.empty(int(_lib.lib.dr_b200_rasterize_scratch_bytes(B, F, H, W)), dtype=torch.uint8, device=dev)
            _lib.check(_lib.lib.dr_b200_rasterize_fwd(_P(p), _P(t), B, V, F, H, W, _P(rast), _P(db), _P(scratch), _stream()))
        ctx.save_for_backward(p, t, rast)
        ctx.dims = (B, V, F, H, W)
        ctx.mark_non_differentiable(db)
        return rast, db

    @staticmethod
    def backward(ctx, g_rast, g_db):
        p, t, rast = ctx.saved_tensors
        B, V, F, H, W = ctx.dims
        d_pos = torch.zeros_like(p)
        if g_rast is not None and F > 0:
            g = _f32(g_rast, "grad")
            with torch.cuda.device(p.device):
                _lib.check(_lib.lib.dr_b200_rasterize_bwd(_P(p), _P(t), B, V, F, H, W, _P(rast), _P(g), _P(d_pos), _stream()))
        return d_pos, None, None, None


def rasterize(glctx, pos, tri, resolution, ranges=None, grad_db=True):
    """(rast[B,H,W,4] = (u, v, z/w, id+1), rast_db[B,H,W,4]); gradients flow to pos through u,v."""
    if ranges is not None or pos.dim() != 3:
        raise NotImplementedError("range mode (2-D pos + ranges) is not used by the reference and not implemented")
    if pos.shape[-1] != 4 or tri.dim() != 2 or tri.shape[1] != 3:
        raise ValueError("pos must be [B,V,4], tri must be [F,3]")
    H, W = int(resolution[0]), int(resolution[1])
    return _Rasterize.apply(pos, tri, H, W)


# ------------------------------------------------------------------------------------------------ interpolate
class _Interpolate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, attr, rast, tri, rast_db, want_da):
        a = _f32(attr, "attr"); r = _f32(rast, "rast"); t = _i32(tri, "tri")
        db = _f32(rast_db, "rast_db") if want_da else None
        B, H, W, _ = r.shape
        aB, V, A = a.shape
        F = t.shape[0]
        dev = r.device
        with torch.cuda.device(dev):
            out = torch.empty(B, H, W, A, device=dev)
            out_da = torch.empty(B, H, W, 2 * A, device=dev) if want_da else None
            _lib.check(_lib.lib.dr_b200_interpolate_fwd(_P(a), aB, _P(r), _P(t), _P(db), B, V, F, H, W, A, _P(out), _P(out_da), _stream()))
        ctx.save_for_backward(a, r, t, db)
        ctx.dims = (aB, B, V, F, H, W, A, want_da)
        if want_da:
            return out, out_da
        return out, torch.empty(0, device=dev)

    @staticmethod
    def backward(ctx, g_out, g_da):
        a, r, t, db = ctx.saved_tensors
        aB, B, V, F, H, W, A, want_da = ctx.dims
        dev = r.device
        g = _f32(g_out, "grad") if g_out is not None else torch.zeros(B, H, W, A, device=dev)
        gda = _f32(g_da, "grad") if (want_da and g_da is not None and g_da.numel()) else None
        d_attr = torch.zeros_like(a)
        d_rast = torch.empty_like(r)
        d_db = torch.empty_like(r) if gda is not None else None
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.dr_b200_interpolate_bwd(_P(a), aB, _P(r), _P(t), _P(db if gda is not None else None), B, V, F, H, W, A,
                                                        _P(g), _P(gda), _P(d_attr), _P(d_rast), _P(d_db), _stream()))
        return d_attr, d_rast, None, d_db, None


def interpolate(attr, rast, tri, rast_db=None, diff_attrs=None):
    """out = u a0 + v a1 + (1-u-v) a2 per pixel; with rast_db and diff_attrs='all' also (da/dX, da/dY)."""
    if attr.dim() == 2:
        attr = attr[None]
    want_da = rast_db is not None and diff_attrs is not None
    if want_da and diff_attrs != "all":
        sel = list(diff_attrs)
        if sel != list(range(attr.shape[-1])):
            raise NotImplementedError("diff_attrs must be None or 'all' (the reference uses only those)")
    out, da = _Interpolate.apply(attr, rast, tri, rast_db if want_da else None, want_da)
    return out, (da if want_da else None)


# ------------------------------------------------------------------------------------------------ texture
class _Texture(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tex, uv, boundary):
        t = _f32(tex, "tex"); u = _f32(uv, "uv")
        tB, Ht, Wt, Cc = t.shape
        B, H, W, _ = u.shape
        dev = u.device
        with torch.cuda.device(dev):
            out = torch.empty(B, H, W, Cc, device=dev)
            _lib.check(_lib.lib.dr_b200_texture_fwd(_P(t), tB, Ht, Wt, Cc, _P(u), B, H, W, boundary, _P(out), _stream()))
        ctx.save_for_backward(t, u)
        ctx.boundary = boundary
        return out

    @staticmethod
    def backward(ctx, g_out):
        t, u = ctx.saved_tensors
        tB, Ht, Wt, Cc = t.shape
        B, H, W, _ = u.shape
        g = _f32(g_out, "grad")
        d_tex = torch.zeros_like(t); d_uv = torch.empty_like(u)
        with torch.cuda.device(u.device):
            _lib.check(_lib.lib.dr_b200_texture_bwd(_P(t), tB, Ht, Wt, Cc, _P(u), B, H, W, ctx.boundary, _P(g), _P(d_tex), _P(d_uv), _stream()))
        return d_tex, d_uv, None


def _mip_pyramid(tex, max_mip_level=None):
    """2x2 box-filtered levels while both sides are even (1 texel for power-of-two textures), at most max_mip_level."""
    levels = [tex]
    while levels[-1].shape[1] % 2 == 0 and levels[-1].shape[2] % 2 == 0 and (max_mip_level is None or len(levels) <= max_mip_level):
        t = levels[-1]
        levels.append((0.25 * (t[:, 0::2, 0::2] + t[:, 1::2, 0::2] + t[:, 0::2, 1::2] + t[:, 1::2, 1::2])).contiguous())
    return levels


def _mip_level(uv_da, Ht, Wt, n_levels, mip_level_bias=None):
    """half log2 of the squared major axis of the pixel footprint in texel units (nvdiffrast calculateMipLevel, restated)."""
    dsdx, dsdy, dtdx, dtdy = uv_da[..., 0] * Wt, uv_da[..., 1] * Wt, uv_da[..., 2] * Ht, uv_da[..., 3] * Ht
    A = dsdx * dsdx + dtdx * dtdx
    Bq = dsdy * dsdy + dtdy * dtdy
    Cq = dsdx * dsdy + dtdx * dtdy
    major2 = 0.5 * (A + Bq) + torch.sqrt(0.25 * (A - Bq) * (A - Bq) + Cq * Cq)
    level = 0.5 * torch.log2(torch.clamp_min(major2, 1e-30))
    if mip_level_bias is not None:
        level = level + mip_level_bias
    return torch.clamp(level, 0.0, float(n_levels - 1))


def texture(tex, uv, uv_da=None, mip_level_bias=None, mip=None, filter_mode="auto", boundary_mode="wrap", max_mip_level=None):
    """filter_mode 'linear': one bilinear lookup (CUDA kernel) — what DiffRastRenderer passes (diff_mesh_renderer.py:72,105).
    'auto' = 'linear-mipmap-linear' when uv_da or mip_level_bias is given (LGM's texture fit,
    Gen_3D_Modules/LGM/nerf_marching_cubes_converter.py:229-230), else 'linear'.  The mip-mapped mode runs the same
    bilinear kernel on every level of a box-filtered pyramid and blends the two levels around the per-pixel level of detail
    with tent weights; gradients reach the texture (through the pyramid), uv and uv_da."""
    if filter_mode == "auto":
        filter_mode = "linear-mipmap-linear" if (uv_da is not None or mip_level_bias is not None) else "linear"
    if filter_mode not in ("linear", "linear-mipmap-linear"):
        raise NotImplementedError(f"filter_mode={filter_mode!r}: 'linear' and 'linear-mipmap-linear' (and 'auto') are implemented")
    if boundary_mode not in ("wrap", "clamp"):
        raise NotImplementedError(f"boundary_mode={boundary_mode!r}")
    if tex.dim() != 4 or uv.dim() != 4 or uv.shape[-1] != 2:
        raise ValueError("tex must be [T,Ht,Wt,C], uv must be [B,H,W,2]")
    bmode = 0 if boundary_mode == "wrap" else 1
    if filter_mode == "linear":
        return _Texture.apply(tex, uv, bmode)
    if mip is not None:
        raise NotImplementedError("pre-built mip stacks (texture_construct_mip) are not implemented")
    if uv_da is None:
        uv_da = torch.zeros(*uv.shape[:-1], 4, device=uv.device, dtype=torch.float32)
    levels = _mip_pyramid(tex.float(), max_mip_level)
    lod = _mip_level(uv_da.float(), tex.shape[1], tex.shape[2], len(levels), mip_level_bias)
    out = None
    for l, t in enumerate(levels):
        w = torch.clamp(1.0 - (lod - float(l)).abs(), min=0.0)
        if not bool((w > 0).any()):          # no pixel of this call uses the level
            continue
        term = w[..., None] * _Texture.apply(t, uv, bmode)
        out = term if out is None else out + term
    return out


# ------------------------------------------------------------------------------------------------ antialias
_TOPO_CACHE = {}        # id(tri tensor) -> (weakref, meta, opp); tensors cannot be dict keys (elementwise __eq__)


def get_topology(tri, n_vertices):
    """opp[F,3] (the package's topology hash): cached per tri tensor object/version; rebuilt on the GPU otherwise
    (FlexiCubes changes topology every step, flexicubes_trainer.py:134)."""
    key = (tri.data_ptr(), tri._version, tuple(tri.shape), int(n_vertices))
    ent = _TOPO_CACHE.get(id(tri))
    if ent is not None and ent[0]() is tri and ent[1] == key:
        return ent[2]
    t = _i32(tri, "tri")
    F = t.shape[0]
    opp = torch.empty(F, 3, dtype=torch.int32, device=t.device)
    if F > 0:
        with torch.cuda.device(t.device):
            scratch = torch.empty(int(_lib.lib.dr_b200_topology_scratch_bytes(F)), dtype=torch.uint8, device=t.device)
            _lib.check(_lib.lib.dr_b200_edge_opposites(_P(t), F, int(n_vertices), _P(opp), _P(scratch), _stream()))
    tid = id(tri)
    try:
        _TOPO_CACHE[tid] = (weakref.ref(tri, lambda _r, tid=tid: _TOPO_CACHE.pop(tid, None)), key, opp)
    except TypeError:
        pass
    return opp


class _Antialias(torch.autograd.Function):
    @staticmethod
    def forward(ctx, color, rast, pos, tri, opp):
        c = _f32(color, "color"); r = _f32(rast, "rast"); p = _f32(pos, "pos"); t = _i32(tri, "tri")
        B, H, W, Cc = c.shape
        V = p.shape[1]; F = t.shape[0]
        with torch.cuda.device(c.device):
            out = torch.empty_like(c)
            _lib.check(_lib.lib.dr_b200_antialias_fwd(_P(c), _P(r), _P(p), _P(t), _P(opp), B, V, F, H, W, Cc, _P(out), _stream()))
        ctx.save_for_backward(c, r, p, t, opp)
        return out

    @staticmethod
    def backward(ctx, g_out):
        c, r, p, t, opp = ctx.saved_tensors
        B, H, W, Cc = c.shape
        V = p.shape[1]; F = t.shape[0]
        g = _f32(g_out, "grad")
        d_color = torch.empty_like(c); d_pos = torch.zeros_like(p)
        with torch.cuda.device(c.device):
            _lib.check(_lib.lib.dr_b200_antialias_bwd(_P(c), _P(r), _P(p), _P(t), _P(opp), B, V, F, H, W, Cc, _P(g), _P(d_color), _P(d_pos), _stream()))
        return d_color, None, d_pos, None, None


def antialias(color, rast, pos, tri, topology_hash=None, pos_gradient_boost=1.0):
    """Analytic silhouette antialiasing; gradients to color and pos."""
    if pos.dim() != 3:
        raise NotImplementedError("range mode is not implemented")
    opp = topology_hash if topology_hash is not None else get_topology(tri, pos.shape[1])
    out = _Antialias.apply(color, rast, pos, tri, opp)
    if pos_gradient_boost != 1.0:
        raise NotImplementedError("pos_gradient_boost != 1 is not used by the reference")
    return out


def antialias_construct_topology_hash(tri):
    return get_topology(tri, int(tri.max().item()) + 1 if tri.numel() else 0)
