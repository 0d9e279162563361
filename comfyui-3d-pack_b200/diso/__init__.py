"""Import-name shim for diso's `DiffDMC`, the differentiable dual marching cubes that TripoSG
(Gen_3D_Modules/TripoSG/inference_utils.py:7,466-472) and Hunyuan3D 2.0 / 2.1's DMCSurfaceExtractor call as their
final mesh-extraction step.  It runs on the GPU through gs_b200.isosurface.DiffDMC, whose contract is stated in
include/ngp_b200.h.  Differences from the package: no CPU path and fp32 only; vertices and faces come in a fixed
order (diso's order comes from atomics); the empty result has (0, 3) faces.  Parity with diso's own binaries is
unpinned.  With this directory on sys.path, `import diso` resolves here for the whole process, shadowing an
installed diso.
"""
from gs_b200.isosurface import DiffDMC


class DiffMC:
    """Not provided: no caller in the pack uses diso's DiffMC."""

    def __init__(self, *a, **k):
        raise NotImplementedError("diso.DiffMC is not provided: only DiffDMC runs on the GPU here, and no caller in "
                                  "the pack uses DiffMC")


__all__ = ["DiffDMC", "DiffMC"]
