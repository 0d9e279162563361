"""Writes tests/golden/ref_sf3d_baker.npz: StableFast3D texture bakes by the reference's own code.

Two stages:
  1. CPU, needs a ComfyUI-3D-Pack checkout (COMFYUI_3D_PACK, or one next to this repository):
         python tests/golden/make_golden_sf3d_baker.py uv  OUT_DIR
     runs SF3D's own box_projection_uv_unwrap (sf3d/box_uv_unwrap.py) on seeded meshes and lays the result out as
     Mesh.unwrap_uv does (a triangle soup: V = 3F, faces = arange(3F)); writes OUT_DIR/sf3d_uv_stage1.npz.
  2. GPU, needs the oracle/_ref build of the reference's generated CUDA (oracle/build_ref_sf3d.py):
         python tests/golden/make_golden_sf3d_baker.py bake OUT_DIR/sf3d_uv_stage1.npz OUT_DIR
     replays TextureBaker.rasterize and interpolate (positions, normals) with its exact launches (res // 16 blocks of
     16, outputs from torch.empty / torch.zeros; the texels a launch leaves are pinned to a sentinel first) at 256^2,
     1000^2 (not a multiple of 16) and 1024^2; writes OUT_DIR/ref_sf3d_baker.npz.
Inputs are stored as fp32 bits: SF3D's unwrapped uvs of both meshes and blob15k's vertices and normals, which soup()
gathers into the soup over grid_faces' triangles (integers, rebuilt rather than stored).  Outputs are stored as the
SHA-256 digests of their bytes: the bake of both meshes, and interpolate of blob15k's positions and normals.
"""
import hashlib
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

MESHES = {"blob15k": (15000, 11), "blob60k": (60000, 12)}       # approximate face counts, seeds
WITH_ATTRS = ("blob15k",)       # meshes whose positions and normals are stored and interpolated (the others: uv only)
RESOLUTIONS = (256, 1000, 1024)
SENTINEL = np.float32(-7.25)                                     # what unlaunched texels hold in the fixture


def grid_faces(faces_target):
    """(nlat, nlon, f int64 [F,3]): the triangles of blob_mesh's nlat x nlon grid with two poles, from integers only."""
    nlon = int(round((faces_target / 2) ** 0.5 * 1.4))
    nlat = max(3, int(round(faces_target / (2 * nlon))))
    idx = lambda i, j: i * nlon + (j % nlon)  # noqa: E731
    tris = []
    for i in range(nlat - 1):
        for j in range(nlon):
            tris += [(idx(i, j), idx(i + 1, j), idx(i + 1, j + 1)), (idx(i, j), idx(i + 1, j + 1), idx(i, j + 1))]
    top, bot = nlat * nlon, nlat * nlon + 1
    for j in range(nlon):
        tris += [(top, idx(0, j + 1), idx(0, j)), (bot, idx(nlat - 1, j), idx(nlat - 1, j + 1))]
    return nlat, nlon, np.array(tris, np.int64)


def blob_mesh(faces_target, seed):
    """A seeded bumpy sphere: grid_faces' triangles, positions pushed along a low-frequency random field."""
    import torch
    g = torch.Generator().manual_seed(seed)
    nlat, nlon, f = grid_faces(faces_target)
    th = torch.linspace(0, np.pi, nlat + 2, dtype=torch.float64)[1:-1]
    ph = torch.linspace(0, 2 * np.pi, nlon + 1, dtype=torch.float64)[:-1]
    T, P = torch.meshgrid(th, ph, indexing="ij")
    d = torch.stack([T.sin() * P.cos(), T.sin() * P.sin(), T.cos()], -1).reshape(-1, 3)
    d = torch.cat([d, torch.tensor([[0, 0, 1.0], [0, 0, -1.0]], dtype=torch.float64)])
    k = torch.randn(6, 3, generator=g, dtype=torch.float64) * 2.5
    a = torch.rand(6, generator=g, dtype=torch.float64) * 0.12
    r = 1 + (a[None] * torch.sin(d @ k.T)).sum(-1)
    v = (d * r[:, None]).float()
    f = torch.from_numpy(f)
    fn = torch.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]], dim=-1)
    vn = torch.zeros_like(v).index_add_(0, f.reshape(-1), fn.repeat_interleave(3, 0))
    vn = torch.nn.functional.normalize(vn, dim=-1)
    return v, vn, f


def stage_uv(out_dir):
    from oracle import build_ref_sf3d
    src = build_ref_sf3d.source()
    if src is None:
        raise SystemExit("no ComfyUI-3D-Pack checkout found (set COMFYUI_3D_PACK)")
    gen3d = src.split("/StableFast3D/")[0]
    sys.path.insert(0, gen3d)
    om = types.ModuleType("omegaconf")          # sf3d.models.utils imports it at module level; the unwrap never uses it
    om.DictConfig, om.OmegaConf = dict, object
    sys.modules.setdefault("omegaconf", om)
    import PIL.Image  # noqa: F401  (sf3d.models.utils reads PIL.Image at import)
    import torch
    from StableFast3D.sf3d.box_uv_unwrap import box_projection_uv_unwrap
    out = {}
    for name, (nf, seed) in MESHES.items():
        v, vn, f = blob_mesh(nf, seed)
        uv, indices = box_projection_uv_unwrap(v, vn, f, 0.02)
        # stored per mesh vertex / per unwrapped uv (the triangles are grid_faces'); soup() lays them out as
        # Mesh.unwrap_uv does
        if name in WITH_ATTRS:
            out[f"{name}/v"] = v.float().numpy().view(np.uint32)
            out[f"{name}/vn"] = vn.float().numpy().view(np.uint32)
        out[f"{name}/uv_unique"] = uv.float().numpy().view(np.uint32)
        out[f"{name}/uv_index"] = indices.int().numpy()
        print(name, "faces", f.shape[0], "uvs", uv.shape[0])
    os.makedirs(out_dir, exist_ok=True)
    np.savez_compressed(os.path.join(out_dir, "sf3d_uv_stage1.npz"), **out)


def soup(z, name):
    """(uv [3F,2], faces [F,3] = arange, pos [3F,3], nrm [3F,3]) of a fixture mesh, in Mesh.unwrap_uv's soup layout:
    pure gathers of the stored fp32 bits, so the same on every machine.  pos and nrm are None for a mesh stored with
    its uvs only."""
    f = grid_faces(MESHES[name][0])[2]
    uv = z[f"{name}/uv_unique"].view(np.float32)[z[f"{name}/uv_index"].astype(np.int64)].reshape(-1, 2)
    pos = z[f"{name}/v"].view(np.float32)[f].reshape(-1, 3) if f"{name}/v" in z else None
    nrm = z[f"{name}/vn"].view(np.float32)[f].reshape(-1, 3) if f"{name}/vn" in z else None
    faces = np.arange(3 * f.shape[0], dtype=np.int32).reshape(-1, 3)
    return uv, faces, pos, nrm


def ref_bake(lib, uv, faces, res):
    """TextureBaker.rasterize with the reference kernel; unlaunched texels hold SENTINEL."""
    import torch
    out = torch.full((res, res, 4), float(SENTINEL), device="cuda")
    g = res // 16
    rc = lib.sf3d_ref_bake_uv(uv.data_ptr(), uv.shape[0], faces.data_ptr(), faces.shape[0], out.data_ptr(), res, res,
                              16, 16, g, g, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rc
    return out


def ref_interp(lib, attr, faces, rast):
    import torch
    res = rast.shape[0]
    out = torch.full((res, res, 3), float(SENTINEL), device="cuda")
    g = res // 16
    rc = lib.sf3d_ref_interpolate(attr.data_ptr(), attr.shape[0], faces.data_ptr(), faces.shape[0], rast.data_ptr(),
                                  out.data_ptr(), res, res, 16, 16, g, g, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rc
    return out


def digest(t):
    return np.frombuffer(hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).digest(), np.uint8)


def stage_bake(stage1, out_dir):
    import torch
    from oracle import build_ref_sf3d
    lib = build_ref_sf3d.load()
    if lib is None:
        raise SystemExit("oracle/_ref has no SF3D reference build: run oracle/build_ref_sf3d.py first")
    src = dict(np.load(stage1))
    out = dict(src)
    out["sentinel"] = np.array([SENTINEL], np.float32).view(np.uint32)
    for name in MESHES:
        uv, faces, pos, nrm = (None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()
                               for a in soup(src, name))
        for res in RESOLUTIONS:
            rast = ref_bake(lib, uv, faces, res)
            key = f"{name}/{res}"
            out[f"{key}/rast_sha256"] = digest(rast)
            if pos is not None:
                out[f"{key}/pos_bake_sha256"] = digest(ref_interp(lib, pos, faces, rast))
                out[f"{key}/nrm_bake_sha256"] = digest(ref_interp(lib, nrm, faces, rast))
            print(key, "covered", float((rast[..., 3] >= 0).float().mean()))
    os.makedirs(out_dir, exist_ok=True)
    np.savez_compressed(os.path.join(out_dir, "ref_sf3d_baker.npz"), **out)


if __name__ == "__main__":
    if sys.argv[1] == "uv":
        stage_uv(sys.argv[2])
    else:
        stage_bake(sys.argv[2], sys.argv[3])
