"""Import-name shim for PyMCubes' `marching_cubes(volume, isovalue)` (mesh_processer/mesh_utils.py:489,509; LGM
nerf_marching_cubes_converter.py:245; InstantMesh models/lrm.py:178; TripoSR models/isosurface.py:45).

The numpy volume is cast to fp32, uploaded to the current CUDA device and meshed by gs_b200.isosurface; the result
comes back as numpy arrays.  Differences from PyMCubes' own C++ extractor:
- the comparison `value > iso` is made in fp32;
- the case table resolves every ambiguous face by cutting off its above corners, so the mesh is always watertight;
- triangles are counter-clockwise seen from the below-iso side.
"""
import numpy as np
import torch

from gs_b200.isosurface import marching_cubes as _marching_cubes_cuda

__version__ = "0.1.2+b200"

# PyMCubes 0.1.x returns float64 vertices and uint64 triangles (recalled, not pinned against the package); every
# known caller casts both, so only these two names would change if that recollection were wrong.
VERTEX_DTYPE = np.float64
TRIANGLE_DTYPE = np.uint64


def marching_cubes(volume, isovalue):
    """(vertices VERTEX_DTYPE [V,3], triangles TRIANGLE_DTYPE [F,3]) of the iso-surface of a real numpy volume[X,Y,Z].
    Vertex column c is the coordinate along array axis c, in index units."""
    vol = np.asarray(volume)
    if vol.dtype == np.bool_ or not (np.issubdtype(vol.dtype, np.integer) or np.issubdtype(vol.dtype, np.floating)):
        raise TypeError(f"marching_cubes: volume must have a real dtype, got {vol.dtype}")
    if vol.ndim != 3:
        raise ValueError(f"marching_cubes: volume must be 3-D, got shape {vol.shape}")
    if not torch.cuda.is_available():
        raise RuntimeError("marching_cubes: needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", torch.cuda.current_device())
    v = torch.from_numpy(np.ascontiguousarray(vol, dtype=np.float32)).to(dev)
    verts, tris = _marching_cubes_cuda(v, isovalue)
    return verts.cpu().numpy().astype(VERTEX_DTYPE), tris.cpu().numpy().astype(TRIANGLE_DTYPE)


def _not_provided(name):
    def fn(*a, **k):
        raise NotImplementedError(f"mcubes.{name} is not provided: only marching_cubes(volume, isovalue) runs on the GPU, "
                                  f"and no caller in the pack uses {name}")
    fn.__name__ = name
    return fn


smooth = _not_provided("smooth")
export_obj = _not_provided("export_obj")
marching_cubes_func = _not_provided("marching_cubes_func")
