"""Generates tests/golden/ref_custom_rasterizer.npz by running the REFERENCE's own custom_rasterizer code on the CPU:
render.py's rasterize / interpolate over the reference's compiled custom_rasterizer_kernel (oracle/_ref, built by
oracle/build_ref.py without FMA contraction), with camera matrices from the reference's own camera_utils.py.

    COMFYUI_3D_PACK=/path/to/ComfyUI-3D-Pack python tests/golden/make_golden_custom_rasterizer.py

Inputs are stored exactly: the mesh as integer codes (vertex = code / 4096, uv = code / 4096, colour = code / 256,
faces as ints), with each view's model-view-projection matrix (from the reference's camera_utils, multiplied in
float64): a view's clip positions are mesh_pos(codes, mvp), rounded once to float32. The UV bake's positions are
(2u - 1, 2v - 1, 0, 1). Small cases store clip-space positions and depth maps as their float32 bits.
Outputs are stored as bits: findices and barycentric in full for the small cases, and as SHA-256 digests (with the
covered-pixel count) for the 512^2 and 383x257 mesh views and the UV-space bake.
Each case `k` has k/hw = (H, W); k/pos (uint32 bits of pos[0], [N,4]) and k/tri, or k/mvp / k/uv_pos for the mesh
cases; optionally k/depth (uint32 bits); and either k/findices + k/bary (uint32 bits) or k/digest
("findices:bary" hex) + k/covered. Interpolate cases have k/col (uint32 bits, [1,N,C]; the mesh cases use
mesh/col_codes), k/interp_src naming the raster case, k/fp32_ids, k/tri_i64 (tri's dtype), and k/out (uint32 bits) or k/out_digest.
oracle/cr_oracle.golden_cases rebuilds the inputs.
Nothing from the reference is copied into the repo: only inputs and the numeric outputs are stored."""
import hashlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import build_ref  # noqa: E402

REF = os.environ["COMFYUI_3D_PACK"]
PAINT = os.path.join(REF, "Gen_3D_Modules/Hunyuan3D_2_1/hy3dpaint")
OUT = os.path.join(HERE, "ref_custom_rasterizer.npz")


def load_reference():
    kern = build_ref.load("nofma")
    if kern is None:
        raise SystemExit("oracle/_ref has no nofma build: run oracle/build_ref.py first")
    sys.modules["custom_rasterizer_kernel"] = kern
    render = {}
    src = open(os.path.join(PAINT, "custom_rasterizer/custom_rasterizer/render.py")).read()
    exec(compile(src, "ref_custom_rasterizer_render", "exec"), render)
    cam = {}
    src = open(os.path.join(PAINT, "DifferentiableRenderer/camera_utils.py")).read()
    exec(compile(src, "ref_camera_utils", "exec"), cam)
    return types.SimpleNamespace(**render), types.SimpleNamespace(**cam)


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32)).view(np.uint32)


def sphere_mesh(nu=100, nv=101, seed=0):
    """A seeded bumpy closed-ish UV sphere: vertex codes (x = code / 4096), faces [F,3] (2*(nu-1)*(nv-1) faces)."""
    rng = np.random.default_rng(seed)
    th = np.linspace(0.05, np.pi - 0.05, nu)[:, None]
    ph = np.linspace(0, 2 * np.pi, nv)[None, :]
    r = 0.45 * (1 + 0.15 * rng.standard_normal((nu, nv)).clip(-2, 2))
    xyz = np.stack([r * np.sin(th) * np.cos(ph), r * np.cos(th), r * np.sin(th) * np.sin(ph)], -1).reshape(-1, 3)
    codes = np.round(xyz * 4096).astype(np.int32)
    i, j = np.meshgrid(np.arange(nu - 1), np.arange(nv - 1), indexing="ij")
    a = (i * nv + j).reshape(-1)
    b, c, d = a + 1, a + nv, a + nv + 1
    tri = np.concatenate([np.stack([a, c, b], 1), np.stack([b, c, d], 1)]).astype(np.int32)
    uv = np.stack([np.broadcast_to(ph / (2 * np.pi), (nu, nv)), np.broadcast_to(th / np.pi, (nu, nv))], -1).reshape(-1, 2)
    uv_codes = np.round(uv * 4096).astype(np.int32)
    return codes, tri, uv_codes


def mesh_pos(codes, mvp):
    """Clip-space positions of the mesh under a 4x4 float64 matrix, rounded once to float32 (the test repeats this)."""
    v = np.concatenate([codes.astype(np.float64) / 4096, np.ones((codes.shape[0], 1))], 1)
    return (v @ np.asarray(mvp, np.float64).T).astype(np.float32)


def main():
    render, cam = load_reference()
    store = {}

    def raster(key, pos, tri, hw, depth=None, full=True, mesh_mvp=None):
        pos = torch.from_numpy(np.asarray(pos, dtype=np.float32))
        tri_t = torch.from_numpy(np.asarray(tri, dtype=np.int32).reshape(-1, 3))
        args = (pos[None], tri_t, hw) if depth is None else \
            (pos[None], tri_t, hw, torch.from_numpy(np.asarray(depth, dtype=np.float32)), 1)
        fi, b = render.rasterize(*args)
        if mesh_mvp is None:
            store[f"{key}/pos"] = bits(pos)
            store[f"{key}/tri"] = tri_t.numpy()
        else:                # the test rebuilds pos from the mesh codes: mesh_pos(codes, mvp)
            store[f"{key}/mvp"] = mesh_mvp
        store[f"{key}/hw"] = np.array(hw, dtype=np.int64)
        if depth is not None:
            store[f"{key}/depth"] = bits(depth)
        if full:
            store[f"{key}/findices"] = fi.numpy()
            store[f"{key}/bary"] = bits(b)
        else:
            store[f"{key}/digest"] = np.array(hashlib.sha256(fi.numpy().tobytes()).hexdigest() + ":" +
                                              hashlib.sha256(bits(b).tobytes()).hexdigest())
            store[f"{key}/covered"] = np.array(int((fi != 0).sum()))
        print(key, hw, "faces", tri_t.shape[0], "covered", int((fi != 0).sum()))
        return fi, b

    def interp(key, src, col, fi, b, tri, fp32_ids, full=True, col_codes=False):
        col_t = torch.from_numpy(np.asarray(col, dtype=np.float32))
        if fp32_ids:       # MeshRender: ids concatenated into a float rast_out and sliced back out
            rast_out = torch.cat((b, fi.unsqueeze(-1)), dim=-1).unsqueeze(0)
            out = render.interpolate(col_t, rast_out[0, ..., -1], rast_out[0, ..., :-1], torch.from_numpy(tri))
        else:
            out = render.interpolate(col_t, fi, b, torch.from_numpy(tri))
        if not col_codes:
            store[f"{key}/col"] = bits(col_t)
        store[f"{key}/interp_src"] = np.array(src)
        store[f"{key}/fp32_ids"] = np.array(int(fp32_ids))
        store[f"{key}/tri_i64"] = np.array(int(np.asarray(tri).dtype == np.int64))
        if full:
            store[f"{key}/out"] = bits(out)
        else:
            store[f"{key}/out_digest"] = np.array(hashlib.sha256(bits(out).tobytes()).hexdigest())

    # ---- MeshRender views of a ~20k-face mesh ----------------------------------------------------------------------
    codes, tri, uv_codes = sphere_mesh()
    store["mesh/codes"] = codes
    store["mesh/uv_codes"] = uv_codes
    store["mesh/tri"] = tri
    rng = np.random.default_rng(1)
    vcol_codes = rng.integers(-512, 512, (1, codes.shape[0], 3)).astype(np.int16)
    store["mesh/col_codes"] = vcol_codes
    vcol = vcol_codes.astype(np.float32) / 256
    for hw in ((512, 512), (383, 257)):
        projs = {"persp": cam.get_perspective_projection_matrix(49.13, hw[1] / hw[0], 0.01, 100.0),
                 "ortho": cam.get_orthographic_projection_matrix(-0.6, 0.6, -0.6, 0.6, 0.1, 100)}
        for name, proj in projs.items():
            mv = cam.get_mv_matrix(elev=20, azim=35, camera_distance=1.45)
            mvp = np.asarray(proj, np.float64) @ np.asarray(mv, np.float64)
            key = f"view_{name}_{hw[0]}x{hw[1]}"
            fi, b = raster(key, mesh_pos(codes, mvp), tri, hw, full=False, mesh_mvp=mvp)
            interp(f"{key}_interp", key, vcol, fi, b, tri, fp32_ids=True, full=False, col_codes=True)

    # ---- UV-space rasterization, as uv_feature_map builds it -------------------------------------------------------
    uv = torch.from_numpy(uv_codes.astype(np.float32) / 4096)
    vtx_uv = torch.cat([uv * 2 - 1.0, torch.zeros_like(uv)], dim=1)
    vtx_uv[..., -1] = 1
    store["uv_256/uv_pos"] = np.array(1)       # the test rebuilds pos from mesh/uv_codes
    fi, b = raster("uv_256", vtx_uv, tri, (256, 256), full=False, mesh_mvp=np.zeros((4, 4)))
    del store["uv_256/mvp"]
    interp("uv_256_interp", "uv_256", vcol, fi, b, tri.astype(np.int64), fp32_ids=True, full=False, col_codes=True)

    # ---- small edge cases, stored in full --------------------------------------------------------------------------
    def clip(xs, ys, zs, ws, W, H):
        """clip-space x, y that land exactly on screen coordinate xs, ys (k + 0.5 is a pixel centre)."""
        x = ((np.asarray(xs, np.float64) - 0.5) / (W - 1) * 2 - 1) * np.asarray(ws)
        y = ((np.asarray(ys, np.float64) - 0.5) / (H - 1) * 2 - 1) * np.asarray(ws)
        return np.stack([x, y, np.asarray(zs) * np.asarray(ws), np.asarray(ws) + 0 * x], 1).astype(np.float32)

    # a fan around a vertex on a pixel centre, every vertex on a pixel centre: shared edges through centres
    W = H = 9
    ring = [(1.5, 1.5), (4.5, 0.5), (7.5, 1.5), (8.5, 4.5), (7.5, 7.5), (4.5, 8.5), (1.5, 7.5), (0.5, 4.5)]
    P = clip([4.5] + [p[0] for p in ring], [4.5] + [p[1] for p in ring], [0.3] * 9, [1.0] * 9, W, H)
    fan = np.array([[0, 1 + k, 1 + (k + 1) % 8] for k in range(8)], np.int32)
    fi, b = raster("fan_centres", P, fan, (H, W))
    interp("fan_centres_interp", "fan_centres", rng.standard_normal((1, 9, 4)), fi, b, fan, fp32_ids=False)
    interp("fan_centres_interp_f32", "fan_centres", rng.standard_normal((1, 9, 2)), fi, b, fan.astype(np.int64),
           fp32_ids=True)

    # zero-area faces (collinear and repeated vertices) over a real one
    P = clip([1.5, 6.5, 3.5, 1.5, 4.5, 7.5], [1.5, 1.5, 6.5, 4.5, 4.5, 4.5], [0.4, 0.4, 0.4, 0.2, 0.2, 0.2], [1.0] * 6, W, H)
    raster("zero_area", P, np.array([[3, 4, 5], [0, 0, 1], [0, 1, 2], [2, 2, 2], [3, 5, 4]], np.int32), (H, W))

    # equal-depth overlaps: the lower id wins a tie, whatever the face order
    P = clip([0.5, 8.5, 4.5, 0.5, 8.5, 4.5, 2.5], [0.5, 0.5, 8.5, 8.5, 8.5, 0.5, 2.5], [0.5] * 7, [1.0] * 7, W, H)
    raster("equal_depth", P, np.array([[0, 1, 2], [3, 5, 4], [0, 1, 2], [6, 1, 2]], np.int32), (H, W))

    # a vertex with w < 0, off-screen vertices, negative depth, in one random case and alone
    rng2 = np.random.default_rng(7)
    N = 60
    P = np.concatenate([rng2.uniform(-1.4, 1.4, (N, 3)), rng2.uniform(0.4, 1.6, (N, 1))], 1).astype(np.float32)
    P[:4, 3] = -0.8                               # w < 0
    P[4:8, :2] *= 6                               # off screen
    P[8:14, 2] = -3.0 * P[8:14, 3]                # z/w = -3: negative screen depth
    T = rng2.integers(0, N, (150, 3)).astype(np.int32)
    raster("mixed_40x31", P, T, (40, 31))
    Pbig = np.array([[-0.9, -0.9, 0.1, 1.0], [0.95, -0.2, 0.3, 1.0], [-0.1, 0.9, 0.2, 1.0], [0.8, 0.9, 0.05, 1.0]], np.float32)
    Tbig = np.array([[0, 1, 2], [1, 3, 2], [0, 3, 2]], np.int32)
    # H or W = 1 makes (H - 1) or (W - 1) zero in the screen transform, so every projected face has zero area and the
    # reference covers nothing: these cases pin that empty result, not thin-image coverage
    for hw in ((1, 37), (29, 1), (1, 1)):
        raster(f"line_{hw[0]}x{hw[1]}", Pbig, Tbig, hw)
    fi, b = raster("mixed_40x31_again", P, T, (40, 31))
    interp("mixed_interp", "mixed_40x31_again", rng2.standard_normal((1, N, 3)), fi, b, T, fp32_ids=True)
    P1 = np.array([[-0.8, -0.7, 0.2, 1.0], [0.9, -0.5, 0.1, 1.0], [0.1, 0.8, 0.3, -1.2]], np.float32)
    raster("w_negative", P1, np.array([[0, 1, 2]], np.int32), (16, 16))
    P2 = np.array([[-0.8, -0.7, -1.5, 1.0], [0.9, -0.5, -1.2, 1.0], [0.1, 0.8, -1.1, 1.0]], np.float32)
    raster("negative_depth", P2, np.array([[0, 1, 2]], np.int32), (16, 16))

    # depth prior
    depth = rng2.uniform(-1, 1, (40, 31)).astype(np.float32)
    raster("depth_prior", P, T, (40, 31), depth=depth)

    # F = 0
    raster("no_faces", P, np.zeros((0, 3), np.int32), (12, 10))

    np.savez_compressed(OUT, **store)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
