"""Iso-surfaces on the GPU: the sm_90a kernels behind ngp_b200_mcubes_* and ngp_b200_flexicubes_* (include/ngp_b200.h).

`marching_cubes` replaces PyMCubes' `marching_cubes(volume, iso)` in the density-to-mesh step of the Instant-NGP node
(mesh_processer/mesh_utils.py:509) and LGM's converter (nerf_marching_cubes_converter.py:245); its case table is
csrc/mc_table.cuh, written by scripts/gen_mc_table.py.  `FlexiCubes` replaces the FlexiCubes class of the FlexiCubes
node, CRM and InstantMesh; its case table is csrc/fc_table.cuh, written by scripts/gen_fc_table.py.  No CPU path."""
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


# ---- FlexiCubes ------------------------------------------------------------------------------------------------
def _res3(res):
    if isinstance(res, int):
        return (res, res, res)
    r = tuple(int(v) for v in res)
    if len(r) != 3:
        raise ValueError(f"FlexiCubes: res must be an int or 3 ints, got {res!r}")
    return r


def voxel_grid(res, device):
    """FlexiCubes.construct_voxel_grid in closed form: point (i,j,k) has id (i*Sy + j)*Sz + k (S = R + 1) and
    coordinate round(fp32(i / R) * 1e5) / 1e5 - 0.5 per axis; cube (i,j,k) = (i*Ry + j)*Rz + k lists its corners
    c = 0..7 at offset (c & 1, (c >> 1) & 1, c >> 2).  Fresh tensors on every call."""
    R = _res3(res)
    axes = []
    for r in R:
        t = torch.arange(r + 1, device=device, dtype=torch.float32) / torch.tensor(float(r), device=device)
        axes.append(torch.round(t * 10 ** 5) / (10 ** 5) - 0.5)
    verts = torch.stack(torch.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3)
    Sy, Sz = R[1] + 1, R[2] + 1
    ijk = torch.stack(torch.meshgrid(*[torch.arange(r, device=device) for r in R], indexing="ij"), -1).reshape(-1, 3)
    c = torch.arange(8, device=device)
    p = ijk[:, None, :] + torch.stack([c & 1, (c >> 1) & 1, c >> 2], -1)[None]
    return verts, (p[..., 0] * Sy + p[..., 1]) * Sz + p[..., 2]


def _weight_arg(w, cols, F, name):
    """(tensor with unit column stride, row stride) of a raw weight view such as weight[:, :12]; None stays None."""
    if w is None:
        return None, 0
    shape = (F, cols) if cols else (F,)
    if tuple(w.shape) != shape:
        raise ValueError(f"FlexiCubes: {name} must have shape {shape}, got {tuple(w.shape)}")
    if w.dtype != torch.float32 or (cols and w.stride(1) != 1):
        w = w.float().contiguous()
    return w, w.stride(0)


class _FlexiCubesFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, s, beta, alpha, gamma, R, ws, training):
        dev = x.device
        F = R[0] * R[1] * R[2]
        (beta, sb), (alpha, sa), (gamma, sg) = (_weight_arg(beta, 12, F, "beta_fx12"),
                                                _weight_arg(alpha, 8, F, "alpha_fx8"),
                                                _weight_arg(gamma, 0, F, "gamma_f"))
        opt = lambda t: _P(t) if t is not None else None
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            scratch = torch.empty(int(_lib.lib.ngp_b200_flexicubes_scratch_bytes(*R)), dtype=torch.uint8, device=dev)
            totals = torch.empty(4, dtype=torch.int64, device=dev)
            _lib.check(_lib.lib.ngp_b200_flexicubes_count(_P(s), *R, _P(totals), _P(scratch), stream))
            nvd, nl, nq, ns = totals.tolist()                   # the one host read
            host = (C.c_ulonglong * 4)(nvd, nl, nq, ns)
            nv = nvd + (nq if training else 0) if nvd else 0
            verts = torch.empty((nv, 3), dtype=torch.float32, device=dev)
            faces = torch.empty(((4 if training else 2) * nq if nvd else 0, 3), dtype=torch.int64, device=dev)
            ldev = torch.empty((nl if nvd else 0,), dtype=torch.float32, device=dev)
            _lib.check(_lib.lib.ngp_b200_flexicubes_write(
                _P(x), _P(s), opt(beta), sb, opt(alpha), sa, opt(gamma), sg, *R, float(ws), int(training), host,
                _P(verts), _P(faces), _P(ldev), _P(scratch), stream))
        ctx.mark_non_differentiable(faces)
        ctx.save_for_backward(x, s, beta, alpha, gamma, verts, scratch)
        ctx.meta = (R, ws, training, (nvd, nl, nq, ns), (sb, sa, sg))
        return verts, faces, ldev

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gverts, _gfaces, gldev):
        x, s, beta, alpha, gamma, verts, scratch = ctx.saved_tensors
        R, ws, training, totals, (sb, sa, sg) = ctx.meta
        need = ctx.needs_input_grad
        dev = x.device
        F = R[0] * R[1] * R[2]
        host = (C.c_ulonglong * 4)(*totals)
        gverts = torch.zeros_like(verts) if gverts is None else gverts.float().contiguous()
        gldev = torch.zeros((totals[1] if totals[0] else 0,), dtype=torch.float32, device=dev) if gldev is None \
            else gldev.float().contiguous()
        new = lambda want, shape: torch.empty(shape, dtype=torch.float32, device=dev) if want else None
        gx, gs = new(need[0], x.shape), new(need[1], s.shape)
        gb, ga, gg = new(need[2], (F, 12)), new(need[3], (F, 8)), new(need[4], (F,))
        opt = lambda t: _P(t) if t is not None else None
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            ws_bytes = int(_lib.lib.ngp_b200_flexicubes_backward_workspace_bytes(host, int(training)))
            work = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
            _lib.check(_lib.lib.ngp_b200_flexicubes_backward(
                _P(x), _P(s), opt(beta), sb, opt(alpha), sa, opt(gamma), sg, *R, float(ws), int(training), host,
                _P(verts), _P(gverts), _P(gldev), opt(gx), opt(gs), opt(gb), opt(ga), opt(gg), _P(scratch), _P(work),
                stream))
        return gx, gs, gb, ga, gg, None, None, None


class FlexiCubes:
    """FlexiCubes mesh extraction on the GPU (the sm_90a kernels behind ngp_b200_flexicubes_*): a drop-in for
    MVs_Algorithms/FlexiCubes/flexicubes.py's FlexiCubes in the FlexiCubes node's trainer and in the CRM and
    InstantMesh geometry modules.  The triangle-mesh path only: tetrahedral output and the QEF path (grad_func) raise
    NotImplementedError.  No CPU path."""
    CUBE_EDGES = [0, 1, 1, 5, 4, 5, 0, 4, 2, 3, 3, 7, 6, 7, 2, 6, 2, 0, 3, 1, 7, 5, 6, 4]

    def __init__(self, device="cuda", qef_reg_scale=1e-3, weight_scale=0.99):
        self.device = torch.device(device)
        self.qef_reg_scale = qef_reg_scale
        self.weight_scale = weight_scale
        self.cube_edges = torch.tensor(self.CUBE_EDGES, dtype=torch.long, device=self.device)
        self._known_cubes = {}

    def construct_voxel_grid(self, res):
        """(verts fp32 [N,3], cubes int64 [F,8]): the same bytes as the reference's grid, built in closed form."""
        return voxel_grid(res, self.device)

    def _check_cubes(self, cube_fx8, R):
        key = id(cube_fx8)
        sig = (cube_fx8._version, cube_fx8.data_ptr(), tuple(cube_fx8.shape), cube_fx8.device, R)
        if self._known_cubes.get(key) == sig:
            return
        _, ref = voxel_grid(R, cube_fx8.device)
        if tuple(cube_fx8.shape) != tuple(ref.shape) or not bool((cube_fx8.long() == ref).all()):
            raise ValueError(f"FlexiCubes: cube_fx8 is not the regular grid of res {R} "
                             "(the one construct_voxel_grid returns); no other topology is supported")
        if len(self._known_cubes) > 16:
            self._known_cubes.clear()
        self._known_cubes[key] = sig

    def __call__(self, x_nx3, s_n, cube_fx8, res, beta_fx12=None, alpha_fx8=None, gamma_f=None, training=False,
                 output_tetmesh=False, grad_func=None):
        """(vertices fp32 [V,3], faces int64 [T,3], L_dev fp32 [E]) of the triangle mesh, on the current stream with
        one host read; differentiable in x_nx3, s_n and the three raw weights."""
        if output_tetmesh:
            raise NotImplementedError("FlexiCubes: tetrahedral output is not implemented on the GPU path")
        if grad_func is not None:
            raise NotImplementedError("FlexiCubes: the QEF path (grad_func) is not implemented on the GPU path")
        for name, t in (("x_nx3", x_nx3), ("s_n", s_n), ("cube_fx8", cube_fx8), ("beta_fx12", beta_fx12),
                        ("alpha_fx8", alpha_fx8), ("gamma_f", gamma_f)):
            if t is not None and (not isinstance(t, torch.Tensor) or not t.is_cuda):
                raise TypeError(f"FlexiCubes: {name} must be a CUDA tensor (gs_b200 has no CPU path)")
        R = _res3(res)
        P = (R[0] + 1) * (R[1] + 1) * (R[2] + 1)
        if tuple(x_nx3.shape) != (P, 3) or tuple(s_n.reshape(-1).shape) != (P,):
            raise ValueError(f"FlexiCubes: x_nx3 must be [{P},3] and s_n [{P}] for res {R}, got "
                             f"{tuple(x_nx3.shape)} and {tuple(s_n.shape)}")
        self._check_cubes(cube_fx8, R)
        x = x_nx3.float().contiguous()
        s = s_n.reshape(-1).float().contiguous()
        return _FlexiCubesFn.apply(x, s, beta_fx12, alpha_fx8, gamma_f, R, float(self.weight_scale), bool(training))
