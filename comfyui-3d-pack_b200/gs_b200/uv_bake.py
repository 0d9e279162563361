"""StableFast3D's UV texture baker on the GPU: bake_uv and interpolate of sf3d/texture_baker.slang, bit-identical to the
reference's own kernels, over the sm_90a kernels of csrc/uv_bake.cu (include/dr_b200.h, dr_b200_uvbake_*).

Call site: sf3d/system.py (TextureBaker.rasterize, get_mask, then interpolate of positions, normals and tangents).  The
import name `slangtorch` (comfyui-3d-pack_b200/slangtorch) serves texture_baker.slang's module from these functions.

- rasterize(uv, faces, res) -> [res, res, 4]: per texel (u, v, w, face) of the lowest-index face whose barycentric test
  accepts it, or (0, 0, 0, -1).  interpolate(attr, rast, faces) -> [H, W, 3].
- rasterize_into / interpolate_into write only the launched region, rows x cols texels from the origin, of an output
  tensor the caller owns: the rest keeps what it held, as the reference's launches leave it.
- Inputs: CUDA fp32 uv [V,2] and attr [V,3], int32 or int64 faces [F,3] (int64 is narrowed to int32, as TextureBaker
  itself does).  Read-only inputs are made contiguous; outputs must be contiguous fp32.  CPU tensors raise
  RuntimeError.  Everything runs on the current stream with no host read.
- Deviations, where the reference is undefined: a face with a vertex id out of range is skipped; interpolate of a face
  or vertex id out of range gives 0; a region larger than the texture is clipped.
"""

import torch

from . import _lib
from ._lib import ptr, stream


def _cuda(t, what, dtypes):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{what} must be a tensor, got {type(t).__name__}")
    if not t.is_cuda:
        raise RuntimeError(f"{what} must be a CUDA tensor (gs_b200's uv_bake has no CPU path)")
    if t.dtype not in dtypes:
        raise TypeError(f"{what} must be {' or '.join(str(d) for d in dtypes)}, got {t.dtype}")
    return t.detach().contiguous()


def _faces(faces):
    f = _cuda(faces, "faces", (torch.int32, torch.int64))
    if f.dim() != 2 or f.shape[1] != 3:
        raise ValueError(f"faces must be [F, 3], got {tuple(f.shape)}")
    return f.to(torch.int32)


def _aligned(t, n):
    return t if t.data_ptr() % n == 0 else t.clone()


def _out(out, what, channels):
    if not isinstance(out, torch.Tensor):
        raise TypeError(f"{what} must be a tensor, got {type(out).__name__}")
    if not out.is_cuda:
        raise RuntimeError(f"{what} must be a CUDA tensor (gs_b200's uv_bake has no CPU path)")
    if out.dtype != torch.float32:
        raise TypeError(f"{what} must be torch.float32, got {out.dtype}")
    if out.dim() != 3 or out.shape[2] != channels:
        raise ValueError(f"{what} must be [H, W, {channels}], got {tuple(out.shape)}")
    if out.shape[0] != out.shape[1]:
        raise NotImplementedError(f"{what}: only square textures are baked (TextureBaker makes no other), got "
                                  f"{tuple(out.shape[:2])}")
    if not out.is_contiguous():
        raise ValueError(f"{what} must be contiguous (it is written in place)")
    return int(out.shape[0])


def rasterize_into(uv, faces, out, rows, cols, counts=False):
    """Bake texels [0, rows) x [0, cols) of out[res,res,4] in place; returns out.  With counts=True returns
    (out, (warp, cta, whole)): the faces the warp and CTA queues got, and those of the CTA queue no candidate box bounds
    (a host read, for tests and benchmarks)."""
    u = _cuda(uv, "uv", (torch.float32,))
    if u.dim() != 2 or u.shape[1] != 2:
        raise ValueError(f"uv must be [V, 2], got {tuple(u.shape)}")
    f = _faces(faces)
    res = _out(out, "output", 4)
    if any(x.device != out.device for x in (u, f)):
        raise RuntimeError("uv, faces and output must be on one device")
    if out.data_ptr() % 16:
        raise ValueError("output must be 16-byte aligned")
    u = _aligned(u, 8)
    with torch.cuda.device(out.device):
        nbytes = int(_lib.lib.dr_b200_uvbake_scratch_bytes(f.shape[0], res))
        if nbytes == 0:
            raise ValueError(f"uv_bake: bad sizes (F = {f.shape[0]}, res = {res})")
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=out.device)
        _lib.check(_lib.lib.dr_b200_uvbake_rasterize(ptr(u), u.shape[0], ptr(f), f.shape[0], ptr(out), res,
                                                     max(0, int(rows)), max(0, int(cols)), ptr(scratch), stream()))
    if counts:
        return out, tuple(int(x) for x in scratch[:12].view(torch.int32).cpu())
    return out


def rasterize(uv, faces, res):
    """TextureBaker.rasterize: [res, res, 4] fp32 over the whole texture."""
    res = int(res)
    if res <= 0:
        raise ValueError(f"res must be positive, got {res}")
    out = torch.empty(res, res, 4, dtype=torch.float32, device=uv.device if isinstance(uv, torch.Tensor) else None)
    return rasterize_into(uv, faces, out, res, res)


def interpolate_into(attr, rast, faces, out, rows, cols):
    """Interpolate texels [0, rows) x [0, cols) of out[H,W,3] in place (rast[H,W,4]); returns out."""
    a = _cuda(attr, "attr", (torch.float32,))
    if a.dim() != 2 or a.shape[1] != 3:
        raise ValueError(f"attr must be [V, 3], got {tuple(a.shape)}")
    r = _cuda(rast, "rast", (torch.float32,))
    f = _faces(faces)
    res = _out(out, "output", 3)
    if tuple(r.shape) != (res, res, 4):
        raise ValueError(f"rast {tuple(r.shape)} does not match output {tuple(out.shape)}")
    if any(x.device != out.device for x in (a, r, f)):
        raise RuntimeError("attr, rast, faces and output must be on one device")
    r = _aligned(r, 16)
    with torch.cuda.device(out.device):
        _lib.check(_lib.lib.dr_b200_uvbake_interpolate(ptr(a), a.shape[0], ptr(f), f.shape[0], ptr(r), ptr(out), res,
                                                       max(0, int(rows)), max(0, int(cols)), stream()))
    return out


def interpolate(attr, rast, faces):
    """TextureBaker.interpolate: [H, W, 3] fp32 over the whole texture."""
    if not isinstance(rast, torch.Tensor) or rast.dim() != 3:
        raise ValueError("rast must be an [H, W, 4] tensor")
    out = torch.zeros(rast.shape[0], rast.shape[1], 3, dtype=torch.float32, device=rast.device)
    return interpolate_into(attr, rast, faces, out, rast.shape[0], rast.shape[1])
