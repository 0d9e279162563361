"""Hunyuan3D's texture-bake rasterizer on the GPU: the surface of the `custom_rasterizer` package (render.py's
rasterize / interpolate) and of its kernel module (`custom_rasterizer_kernel.rasterize_image`), over the sm_90a kernels
of csrc/cr_raster.cu (include/dr_b200.h, dr_b200_cr_*).

Call sites: Hunyuan3D 2.0 texgen/differentiable_renderer/mesh_render.py:145,165-189 and Hunyuan3D 2.1
hy3dpaint/DifferentiableRenderer/MeshRender.py:373 (normal / position renders, back_project, uv_feature_map,
render_uvpos).  The import names `custom_rasterizer` and `custom_rasterizer_kernel` (comfyui-3d-pack_b200/) re-export
this module.

- findices and barycentric are bit-identical to the reference's CPU path; the arithmetic is stated in
  csrc/cr_raster.cu.  Faces the reference's loop is undefined on (a vertex id out of range, a non-finite screen
  coordinate, an x or y screen coordinate outside the int range) are skipped.
- interpolate computes ((+0 + b0 c0) + b1 c1) + b2 c2 in fp32, the order of torch's CPU sum, and is differentiable
  in col and barycentric.  The col gradient goes through the deterministic scatter sum (gs_b200.scatter), so gradients have the same bits on every
  run; that scatter makes its one host read per backward, nothing else reads the device.
- Deviations from the reference: inputs are made contiguous (the reference reads raw pointers, so a strided view is
  misread there); all work goes on the current stream (the reference runs its resolve pass on the legacy default
  stream); CPU tensors raise RuntimeError and other dtypes TypeError (no CPU path).
"""
import ctypes as C

import torch

from . import _lib
from . import scatter as _scatter

OCCLUSION_TRUNCATION = 1e-6


def _P(t):
    return C.c_void_p(t.data_ptr() if t is not None and t.numel() else None)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _cuda(t, what, dtypes):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{what} must be a tensor, got {type(t).__name__}")
    if not t.is_cuda:
        raise RuntimeError(f"{what} must be a CUDA tensor (gs_b200's custom_rasterizer has no CPU path)")
    if t.dtype not in dtypes:
        raise TypeError(f"{what} must be {' or '.join(str(d) for d in dtypes)}, got {t.dtype}")
    return t.detach().contiguous()


def rasterize_image(V, F, D, width, height, occlusion_truncation, use_depth_prior):
    """custom_rasterizer_kernel.rasterize_image: V[N,4] fp32 clip space, F[M,3] int32, D[height,width] fp32 depth prior
    (read only when use_depth_prior) -> (findices int32 [height,width], barycentric fp32 [height,width,3])."""
    v = _cuda(V, "V", (torch.float32,))
    f = _cuda(F, "F", (torch.int32,))
    if v.dim() != 2 or v.shape[1] != 4:
        raise ValueError(f"V must be [N, 4], got {tuple(v.shape)}")
    if f.dim() != 2 or f.shape[1] != 3:
        raise ValueError(f"F must be [M, 3], got {tuple(f.shape)}")
    if f.device != v.device:
        raise RuntimeError(f"V and F must be on one device, got {v.device} and {f.device}")
    W, H = int(width), int(height)
    if W <= 0 or H <= 0:
        raise ValueError(f"width and height must be positive, got {W} x {H}")
    d = None
    if use_depth_prior:
        d = _cuda(D, "D", (torch.float32,))
        if d.numel() < H * W or d.device != v.device:
            raise ValueError(f"the depth prior D must hold height*width = {H * W} values on {v.device}, "
                             f"got {tuple(d.shape)} on {d.device}")
    if v.data_ptr() % 16:
        v = v.clone()
    dev = v.device
    with torch.cuda.device(dev):
        nbytes = int(_lib.lib.dr_b200_cr_scratch_bytes(f.shape[0], H, W))
        if nbytes == 0:
            raise ValueError(f"rasterize_image: bad sizes {H} x {W}")
        findices = torch.empty(H, W, dtype=torch.int32, device=dev)
        bary = torch.empty(H, W, 3, dtype=torch.float32, device=dev)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _lib.check(_lib.lib.dr_b200_cr_rasterize(_P(v), v.shape[0], _P(f), f.shape[0], _P(d), H, W,
                                                 float(occlusion_truncation), _P(findices), _P(bary), _P(scratch),
                                                 _stream()))
    return [findices, bary]


def rasterize(pos, tri, resolution, clamp_depth=torch.zeros(0), use_depth_prior=0):
    """custom_rasterizer.rasterize: reads pos[0] ([B,N,4]); resolution is (H, W).  Returns (findices, barycentric)."""
    findices, barycentric = rasterize_image(pos[0], tri, clamp_depth, resolution[1], resolution[0],
                                            OCCLUSION_TRUNCATION, use_depth_prior)
    return findices, barycentric


class _InterpolateFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, col, barycentric, findices, tri):
        c0 = col[0]
        NV, Cn = c0.shape
        c0 = c0.contiguous()
        npix = findices.numel()
        out = torch.empty(*findices.shape, Cn, dtype=torch.float32, device=col.device)
        args = (_P(c0), NV, Cn, _P(findices), int(findices.dtype == torch.float32), _P(barycentric), _P(tri),
                int(tri.dtype == torch.int64), tri.shape[0], npix)
        with torch.cuda.device(col.device):
            _lib.check(_lib.lib.dr_b200_cr_interpolate_fwd(*args, _P(out), _stream()))
        ctx.save_for_backward(c0, barycentric, findices, tri)
        ctx.col_shape = tuple(col.shape)
        return out.view(1, *out.shape)

    @staticmethod
    def backward(ctx, grad):
        c0, barycentric, findices, tri = ctx.saved_tensors
        want_col, want_bary = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        NV, Cn = c0.shape
        npix = findices.numel()
        dev = c0.device
        g = grad.detach().float().contiguous()
        gb = torch.empty(*barycentric.shape, dtype=torch.float32, device=dev) if want_bary else None
        contrib = torch.empty(3 * npix, Cn, dtype=torch.float32, device=dev) if want_col else None
        cidx = torch.empty(3 * npix, dtype=torch.int64, device=dev) if want_col else None
        gcol = None
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.dr_b200_cr_interpolate_bwd(
                _P(c0), NV, Cn, _P(findices), int(findices.dtype == torch.float32), _P(barycentric), _P(tri),
                int(tri.dtype == torch.int64), tri.shape[0], npix, _P(g), _P(gb), _P(contrib), _P(cidx), _stream()))
            if want_col:
                gcol = torch.zeros(ctx.col_shape, dtype=torch.float32, device=dev)
                if npix:
                    _scatter.scatter_sum(contrib, cidx, dim=0, out=gcol[0])
        return gcol, gb, None, None


def interpolate(col, findices, barycentric, tri):
    """custom_rasterizer.interpolate: col[B,V,C] (only col[0] is read), findices [H,W] int32 or fp32, barycentric
    [H,W,3], tri [F,3] int32 or int64 -> [1,H,W,C].  An empty pixel reads face 0 with weight 0."""
    if not isinstance(col, torch.Tensor) or not col.is_cuda:
        raise RuntimeError("col must be a CUDA tensor (gs_b200's custom_rasterizer has no CPU path)")
    if col.dtype != torch.float32:
        raise TypeError(f"col must be torch.float32, got {col.dtype}")
    if col.dim() != 3 or col.shape[0] < 1:
        raise ValueError(f"col must be [B, V, C] with B >= 1, got {tuple(col.shape)}")
    fid = _cuda(findices, "findices", (torch.int32, torch.float32))
    t = _cuda(tri, "tri", (torch.int32, torch.int64))
    if barycentric.dtype != torch.float32:
        raise TypeError(f"barycentric must be torch.float32, got {barycentric.dtype}")
    if not barycentric.is_cuda:
        raise RuntimeError("barycentric must be a CUDA tensor")
    if tuple(barycentric.shape) != (*fid.shape, 3):
        raise ValueError(f"barycentric {tuple(barycentric.shape)} does not match findices {tuple(fid.shape)} + (3,)")
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f"tri must be [F, 3], got {tuple(t.shape)}")
    if col.shape[2] < 1:
        raise ValueError("col must have at least one channel")
    if any(x.device != col.device for x in (fid, t, barycentric)):
        raise RuntimeError("col, findices, barycentric and tri must be on one device")
    return _InterpolateFn.apply(col, barycentric.contiguous(), fid, t)


def build_hierarchy(*args, **kwargs):
    raise NotImplementedError("custom_rasterizer_kernel.build_hierarchy is not implemented by gs_b200 (no pack call site)")


def build_hierarchy_with_feat(*args, **kwargs):
    raise NotImplementedError("custom_rasterizer_kernel.build_hierarchy_with_feat is not implemented by gs_b200 "
                              "(no pack call site)")
