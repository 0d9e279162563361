"""Iso-surfaces on the GPU: the sm_90a kernels behind ngp_b200_mcubes_* and ngp_b200_flexicubes_* (include/ngp_b200.h).

`marching_cubes` replaces PyMCubes' `marching_cubes(volume, iso)` in the density-to-mesh step of the Instant-NGP node
(mesh_processer/mesh_utils.py:509) and LGM's converter (nerf_marching_cubes_converter.py:245); its case table is
csrc/mc_table.cuh, written by scripts/gen_mc_table.py.  `FlexiCubes` replaces the FlexiCubes class of the FlexiCubes
node, CRM and InstantMesh; its case table is csrc/fc_table.cuh, written by scripts/gen_fc_table.py.
`TrellisFlexiCubes` replaces the FlexiCubes of TRELLIS and Stable3DGen's mesh decoders (cube2mesh.py), the same
extraction with per-vertex colours.  `DiffDMC` replaces diso's differentiable dual marching cubes, the mesh
extraction of TripoSG and Hunyuan3D (FlashVDM); it shares FlexiCubes' case table.  No CPU path."""
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


def _attr_arg(a, P):
    """(tensor with unit column stride, row stride, C) of raw vertex attributes [P,C] such as v_attrs_d[..., 4:]."""
    if a is None:
        return None, 0, 0
    if a.dim() != 2 or a.shape[0] != P or a.shape[1] < 1:
        raise AssertionError("'voxelgrid_colors' should be a tensor of shape (num_vertices, C)")
    if a.dtype != torch.float32 or a.stride(1) != 1 or a.stride(0) < a.shape[1]:
        a = a.float().contiguous()
    return a, a.stride(0), a.shape[1]


class _FlexiCubesFn(torch.autograd.Function):
    """Both extractions: without attributes (attrs None) through ngp_b200_flexicubes_{write,backward}, with them
    through the *_attrs entries.  Returns (verts, faces, L_dev, vertex attributes or None)."""
    @staticmethod
    def forward(ctx, x, s, beta, alpha, gamma, attrs, R, ws, training):
        dev = x.device
        F = R[0] * R[1] * R[2]
        (beta, sb), (alpha, sa), (gamma, sg) = (_weight_arg(beta, 12, F, "beta_fx12"),
                                                _weight_arg(alpha, 8, F, "alpha_fx8"),
                                                _weight_arg(gamma, 0, F, "gamma_f"))
        attrs, sc, nc = _attr_arg(attrs, x.shape[0])
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
            args = (_P(x), _P(s), opt(beta), sb, opt(alpha), sa, opt(gamma), sg, *R, float(ws), int(training), host,
                    _P(verts), _P(faces), _P(ldev))
            if attrs is None:
                vattrs = None
                _lib.check(_lib.lib.ngp_b200_flexicubes_write(*args, _P(scratch), stream))
            else:
                vattrs = torch.empty((nv, nc), dtype=torch.float32, device=dev)
                _lib.check(_lib.lib.ngp_b200_flexicubes_write_attrs(*args, _P(attrs), sc, nc, _P(vattrs),
                                                                     _P(scratch), stream))
        ctx.mark_non_differentiable(faces)
        ctx.save_for_backward(x, s, beta, alpha, gamma, attrs, verts, vattrs, scratch)
        ctx.meta = (R, ws, training, (nvd, nl, nq, ns), (sb, sa, sg, sc, nc))
        return verts, faces, ldev, vattrs

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gverts, _gfaces, gldev, gvattrs):
        x, s, beta, alpha, gamma, attrs, verts, vattrs, scratch = ctx.saved_tensors
        R, ws, training, totals, (sb, sa, sg, sc, nc) = ctx.meta
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
        gat = new(attrs is not None and need[5], (x.shape[0], nc))
        opt = lambda t: _P(t) if t is not None else None
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            args = (_P(x), _P(s), opt(beta), sb, opt(alpha), sa, opt(gamma), sg, *R, float(ws), int(training), host,
                    _P(verts), _P(gverts), _P(gldev), opt(gx), opt(gs), opt(gb), opt(ga), opt(gg))
            if attrs is None:
                ws_bytes = int(_lib.lib.ngp_b200_flexicubes_backward_workspace_bytes(host, int(training)))
                work = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
                _lib.check(_lib.lib.ngp_b200_flexicubes_backward(*args, _P(scratch), _P(work), stream))
            else:
                gvattrs = torch.zeros_like(vattrs) if gvattrs is None else gvattrs.float().contiguous()
                ws_bytes = int(_lib.lib.ngp_b200_flexicubes_backward_attrs_workspace_bytes(host, int(training), nc))
                work = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
                _lib.check(_lib.lib.ngp_b200_flexicubes_backward_attrs(
                    *args, _P(attrs), sc, nc, _P(vattrs), _P(gvattrs), opt(gat), _P(scratch), _P(work), stream))
        return gx, gs, gb, ga, gg, gat, None, None, None


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
        return _FlexiCubesFn.apply(x, s, beta_fx12, alpha_fx8, gamma_f, None, R, float(self.weight_scale),
                                   bool(training))[:3]


class TrellisFlexiCubes:
    """FlexiCubes mesh extraction with vertex attributes on the GPU: a drop-in for the FlexiCubes of TRELLIS and
    Stable3DGen (trellis/representations/mesh/flexicubes), which SparseFeatures2Mesh calls once per shape.  The
    geometry is FlexiCubes' (same kernels, same bits); voxelgrid_colors [P,C] go through a sigmoid and are
    interpolated to each dual vertex with the same weights as its position, and in training to each quad centre with
    the same gamma-weighted means.  qef_reg_scale is accepted and unused, as in the reference.  No CPU path."""

    def __init__(self, device="cuda"):
        self.device = torch.device(device)
        self._fc = FlexiCubes(device=device)

    def __call__(self, voxelgrid_vertices, scalar_field, cube_idx, resolution, qef_reg_scale=1e-3,
                 weight_scale=0.99, beta=None, alpha=None, gamma_f=None, voxelgrid_colors=None, training=False):
        """(vertices fp32 [V,3], faces int64 [T,3], L_dev fp32 [E], vertices_color fp32 [V,C] or None), on the current
        stream with one host read; differentiable in the vertices, the scalar field, the three raw weights and the
        raw colours."""
        def shaped(t, shape):
            return torch.is_tensor(t) and t.dim() == len(shape) and all(
                d is None or t.shape[i] == d for i, d in enumerate(shape))

        if not shaped(voxelgrid_vertices, (None, 3)):
            raise AssertionError("'voxelgrid_vertices' should be a tensor of shape (num_vertices, 3)")
        P = voxelgrid_vertices.shape[0]
        if not shaped(scalar_field, (P,)):
            raise AssertionError("'scalar_field' should be a tensor of shape (num_vertices,)")
        if not shaped(cube_idx, (None, 8)):
            raise AssertionError("'cube_idx' should be a tensor of shape (num_cubes, 8)")
        F = cube_idx.shape[0]
        for name, t, shape, text in (("beta", beta, (F, 12), "(num_cubes, 12)"),
                                     ("alpha", alpha, (F, 8), "(num_cubes, 8)"),
                                     ("gamma_f", gamma_f, (F,), "(num_cubes,)")):
            if t is not None and not shaped(t, shape):
                raise AssertionError(f"'{name}' should be a tensor of shape {text}")
        if voxelgrid_colors is not None and not shaped(voxelgrid_colors, (P, None)):
            raise AssertionError("'voxelgrid_colors' should be a tensor of shape (num_vertices, C)")
        for name, t in (("voxelgrid_vertices", voxelgrid_vertices), ("scalar_field", scalar_field),
                        ("cube_idx", cube_idx), ("beta", beta), ("alpha", alpha), ("gamma_f", gamma_f),
                        ("voxelgrid_colors", voxelgrid_colors)):
            if t is not None and not t.is_cuda:
                raise TypeError(f"TrellisFlexiCubes: {name} must be a CUDA tensor (gs_b200 has no CPU path)")
        R = _res3(resolution)
        if P != (R[0] + 1) * (R[1] + 1) * (R[2] + 1):
            raise ValueError(f"TrellisFlexiCubes: {P} grid points do not make the grid of resolution {R}")
        self._fc._check_cubes(cube_idx, R)
        x = voxelgrid_vertices.float().contiguous()
        s = scalar_field.float().contiguous()
        return _FlexiCubesFn.apply(x, s, beta, alpha, gamma_f, voxelgrid_colors, R, float(weight_scale),
                                   bool(training))


# ---- dual marching cubes (diso.DiffDMC) ----------------------------------------------------------------------------
class _DiffDMCFn(torch.autograd.Function):
    """Dual marching cubes through ngp_b200_dmc_{count,write,backward}; returns (verts, faces)."""
    @staticmethod
    def forward(ctx, grid, deform, iso, return_quads, normalize):
        dev = grid.device
        X, Y, Z = grid.shape
        opt = lambda t: _P(t) if t is not None else None
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            scratch = torch.empty(int(_lib.lib.ngp_b200_dmc_scratch_bytes(X, Y, Z)), dtype=torch.uint8, device=dev)
            totals = torch.empty(3, dtype=torch.int64, device=dev)
            _lib.check(_lib.lib.ngp_b200_dmc_count(_P(grid), X, Y, Z, iso, _P(totals), _P(scratch), stream))
            nv, nq, flags = totals.tolist()                     # the one host read
            host = (C.c_ulonglong * 3)(nv, nq, flags)
            ok = max(nv, nq) < 2 ** 31                          # otherwise the write call fails with the library's message
            verts = torch.empty((nv if ok else 0, 3), dtype=torch.float32, device=dev)
            shape = (nq, 4) if return_quads else (2 * nq, 3)
            faces = torch.empty(shape if ok else (0, shape[1]), dtype=torch.int32, device=dev)
            _lib.check(_lib.lib.ngp_b200_dmc_write(_P(grid), opt(deform), X, Y, Z, iso, int(return_quads),
                                                   int(normalize), host, _P(verts), _P(faces), _P(scratch), stream))
        ctx.mark_non_differentiable(faces)
        ctx.save_for_backward(grid, deform, scratch)
        ctx.meta = (iso, normalize, (nv, nq, flags))
        return verts, faces

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gverts, _gfaces):
        grid, deform, scratch = ctx.saved_tensors
        iso, normalize, totals = ctx.meta
        need = ctx.needs_input_grad
        dev = grid.device
        X, Y, Z = grid.shape
        gverts = torch.zeros((totals[0], 3), dtype=torch.float32, device=dev) if gverts is None \
            else gverts.float().contiguous()
        gg = torch.empty_like(grid) if need[0] else None
        gd = torch.empty_like(deform) if deform is not None and need[1] else None
        opt = lambda t: _P(t) if t is not None else None
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            work = torch.empty(max(int(_lib.lib.ngp_b200_dmc_backward_workspace_bytes(X, Y, Z)), 1), dtype=torch.uint8,
                               device=dev)
            _lib.check(_lib.lib.ngp_b200_dmc_backward(_P(grid), opt(deform), X, Y, Z, iso, int(normalize),
                                                      (C.c_ulonglong * 3)(*totals), _P(gverts), opt(gg), opt(gd),
                                                      _P(scratch), _P(work), stream))
        return gg, gd, None, None, None


class DiffDMC(torch.nn.Module):
    """Differentiable dual marching cubes on the GPU (the sm_90a kernels behind ngp_b200_dmc_*): a drop-in for
    diso.DiffDMC as TripoSG (inference_utils.py:466-472) and Hunyuan3D's DMCSurfaceExtractor call it.  The contract
    is include/ngp_b200.h's: the grid is closed by a virtual ring of samples isovalue + 1, cubes with a non-finite
    corner are masked, vertices and faces come in a fixed order, and gradients are bit-identical from run to run.
    Parity with diso's own binaries is unpinned.  fp32 only; no parameters, so .to(device) is a no-op.  No CPU path."""

    def __init__(self, dtype=torch.float32):
        super().__init__()
        if dtype != torch.float32:
            raise NotImplementedError(f"DiffDMC: only dtype=torch.float32 is implemented on the GPU path, got {dtype}")
        self.dtype = dtype

    def forward(self, grid, deform=None, isovalue=0.0, return_quads=False, normalize=True):
        """(vertices fp32 [V,3], faces int32 [2Q,3], or quads int32 [Q,4] with return_quads) on the grid's device,
        computed on the current stream with one host read; differentiable in grid and deform."""
        if not isinstance(grid, torch.Tensor) or not grid.is_cuda or grid.dtype != torch.float32:
            raise TypeError("DiffDMC: grid must be a CUDA float32 tensor (gs_b200 has no CPU path), got "
                            f"{getattr(grid, 'dtype', type(grid))} on {getattr(grid, 'device', None)}")
        if grid.dim() != 3 or grid.numel() == 0:
            raise ValueError(f"DiffDMC: grid must be a non-empty 3-D [X,Y,Z] tensor, got shape {tuple(grid.shape)}")
        if normalize and min(grid.shape) < 2:
            raise ValueError(f"DiffDMC: normalize divides by (dim - 1), so every dimension must be >= 2, got "
                             f"{tuple(grid.shape)}")
        if deform is not None:
            if not isinstance(deform, torch.Tensor) or deform.device != grid.device or deform.dtype != torch.float32:
                raise TypeError("DiffDMC: deform must be a float32 tensor on the grid's device")
            if tuple(deform.shape) != (*grid.shape, 3):
                raise ValueError(f"DiffDMC: deform must have shape {(*grid.shape, 3)}, got {tuple(deform.shape)}")
            deform = deform.contiguous()
        return _DiffDMCFn.apply(grid.contiguous(), deform, float(isovalue), bool(return_quads), bool(normalize))
