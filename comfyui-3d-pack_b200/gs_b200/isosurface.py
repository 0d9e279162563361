"""Marching cubes on the GPU: the sm_90a kernels behind ngp_b200_mcubes_* (include/ngp_b200.h).

Replaces PyMCubes' `marching_cubes(volume, iso)` in the density-to-mesh step of the Instant-NGP node
(mesh_processer/mesh_utils.py:509) and LGM's converter (nerf_marching_cubes_converter.py:245).  The case table is
csrc/mc_table.cuh, written by scripts/gen_mc_table.py.  No CPU path."""
import ctypes as C

import torch

from . import _lib

_P = lambda t: C.c_void_p(t.data_ptr())


@torch.no_grad()
def marching_cubes(volume, iso):
    """Iso-surface of a CUDA volume[X,Y,Z]: (verts fp32 [V,3], tris int32 [F,3]) on the volume's device, computed on
    the current stream.  A corner is above iff value > iso, with value and iso both in fp32; vertex column c is the
    coordinate along array axis c in index units; triangles are counter-clockwise seen from the below-iso side (their
    normals point from above to below, outward for a density blob).  A non-finite sample raises RuntimeError."""
    if not isinstance(volume, torch.Tensor) or not volume.is_cuda:
        raise TypeError("marching_cubes: volume must be a CUDA tensor (gs_b200 has no CPU path)")
    if volume.dim() != 3:
        raise ValueError(f"marching_cubes: volume must be 3-D [X,Y,Z], got shape {tuple(volume.shape)}")
    if volume.dtype.is_complex or volume.dtype == torch.bool:
        raise TypeError(f"marching_cubes: volume must be real, got {volume.dtype}")
    dev = volume.device
    vol = volume.to(torch.float32).contiguous()
    X, Y, Z = vol.shape
    with torch.cuda.device(dev):
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        scratch = torch.empty(int(_lib.lib.ngp_b200_mcubes_scratch_bytes(X, Y, Z)), dtype=torch.uint8, device=dev)
        totals = torch.empty(3, dtype=torch.int64, device=dev)
        _lib.check(_lib.lib.ngp_b200_mcubes_count(_P(vol), X, Y, Z, float(iso), _P(totals), _P(scratch), stream))
        nv, nf, nonfinite = totals.tolist()
        host = (C.c_ulonglong * 3)(nv, nf, nonfinite)
        ok = nonfinite == 0 and max(nv, nf) < 2 ** 31       # otherwise the write call fails with the library's message
        verts = torch.empty((nv if ok else 0, 3), dtype=torch.float32, device=dev)
        tris = torch.empty((nf if ok else 0, 3), dtype=torch.int32, device=dev)
        _lib.check(_lib.lib.ngp_b200_mcubes_write(_P(vol), X, Y, Z, float(iso), host, _P(verts), _P(tris), _P(scratch),
                                                  stream))
    return verts, tris
