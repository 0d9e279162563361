"""Generates tests/golden/ref_trellis_flexicubes.npz from the REFERENCE's own TRELLIS FlexiCubes code
(trellis/representations/mesh/flexicubes/{flexicubes,tables}.py and mesh/utils_cube.py), run on the CPU.

    COMFYUI_3D_PACK=/path/to/ComfyUI-3D-Pack python tests/golden/make_golden_trellis_flexicubes.py

Stores:
  * SHA-256 digests of construct_dense_grid's (verts, cubes) bytes for res 64 and 256;
  * seeded cases, each run with weight_scale 0.99 (and 0.5 for "random"), weights given and None, colours given and
    None, training on and off: the outputs with an order-free identity per vertex and L_dev entry (ref_keys of
    make_golden_flexicubes.py), the vertex colours, and the gradients of
        sum_v sin(a . v) + (b . v)^2 + lam * mean(L_dev) + sum_{v,c} k_c sin(2 colour_vc)
    with respect to x, s and the raw colours (rows of the surface cubes' corners, the rest must be zero) and the
    [F,21] weight (surface cube rows).
Cases:
  * "trellis": SparseFeatures2Mesh's layout at res 32 with C = 6, built by the reference's own sparse_cube2verts,
    get_dense_attrs and get_defomed_verts from seeded sparse cubes in a band around a sphere (sdf bias -1/res, dense
    default sdf 1, no s == 0).  Its dense inputs are the reference's fp32 outputs, so they are stored as fp32 arrays,
    and only at the rows the sparse cubes touch: trellis/prows for x, s and the colours, trellis/wrows for the
    weights.  Every other row holds the dense defaults: s = 1, zero colours and weights, and x = get_defomed_verts
    at zero deform, i.e. point / res - 0.5 + (1 - 1e-8) / (2 res) * tanh(0) in fp32 (the generator checks the
    rebuild bit for bit).
  * "random" (res 5, C = 6), "c1" (a noisy sphere at res 8, C = 1, no s == 0), "inside" and "outside" (res 6,
    C = 3): inputs stored as small integer codes with power-of-two scales: x = grid * 2 + xq / 4096, s = sq / 1024,
    weight = wq / 32, colours = cq / 16.
Vertices, faces, L_dev and keys are stored under the colours-given tag only (case/ws/given/1/training): the
generator checks that the call without colours gives the same bits.  The gradient rows (grows: the surface cubes'
corners; gw_rows: the surface cubes) are stored once per case.  Indices are stored as int32 and cube edges as int8.
For every variant the generator asserts that the TRELLIS class's vertices, faces and L_dev equal, bit for bit, those
of the FlexiCubes node's class (MVs_Algorithms/FlexiCubes) on the same inputs.  Only numbers are stored."""
import hashlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_flexicubes as MG  # noqa: E402  (reads COMFYUI_3D_PACK)

MESH = os.path.join(MG.REF, "Gen_3D_Modules/TRELLIS/trellis/representations/mesh")
A_VEC, B_VEC, LAM = MG.A_VEC, MG.B_VEC, MG.LAM
K_VEC = [0.9, -0.6, 0.5, -1.1, 0.7, 0.3]


def load_trellis():
    tables = types.ModuleType("trellis_fc_tables")
    exec(compile(open(os.path.join(MESH, "flexicubes/tables.py")).read(), "ref_trellis_tables", "exec"),
         tables.__dict__)
    sys.modules["trellis_fc_tables"] = tables
    src = open(os.path.join(MESH, "flexicubes/flexicubes.py")).read().replace(
        "from .tables import *", "from trellis_fc_tables import *")
    fns, cube = {}, {}
    exec(compile(src, "ref_trellis_flexicubes", "exec"), fns)
    exec(compile(open(os.path.join(MESH, "utils_cube.py")).read(), "ref_trellis_utils_cube", "exec"), cube)
    return fns["FlexiCubes"], cube


def loss_of(v, L, vc):
    out = (torch.sin(v @ torch.tensor(A_VEC)) + (v @ torch.tensor(B_VEC)) ** 2).sum() + LAM * L.mean()
    if vc is not None:
        out = out + (torch.sin(2 * vc) * torch.tensor(K_VEC[:vc.shape[1]])).sum()
    return out


def run_case(TFC, NodeFC, name, res, x0, s0, w0, c0, cubes, out, wss=(0.99,)):
    fc = TFC(device="cpu")
    out[f"{name}/res"] = np.array([res] * 3)
    sc_all = None
    for ws in wss:
        node = NodeFC(device="cpu", weight_scale=ws)
        for given in (1, 0):
            for colours in (1, 0):
                for training in (0, 1):
                    x = x0.clone().requires_grad_(True)
                    s = s0.clone().requires_grad_(True)
                    w = w0.clone().requires_grad_(True)
                    c = c0.clone().requires_grad_(True)
                    kw = dict(beta=w[:, :12], alpha=w[:, 12:20], gamma_f=w[:, 20]) if given else {}
                    v, f, L, vc = fc(voxelgrid_vertices=x, scalar_field=s, cube_idx=cubes, resolution=res,
                                     weight_scale=ws, voxelgrid_colors=c if colours else None,
                                     training=bool(training), **kw)
                    assert (vc is None) == (not colours)
                    nkw = dict(beta_fx12=w[:, :12], alpha_fx8=w[:, 12:20], gamma_f=w[:, 20]) if given else {}
                    with torch.no_grad():
                        nv, nf, nL = node(x, s, cubes, res, training=bool(training), **nkw)
                    assert torch.equal(v.detach().view(torch.int32), nv.view(torch.int32)), (name, "verts")
                    assert torch.equal(f, nf) and torch.equal(L.detach().view(torch.int32), nL.view(torch.int32))
                    tag = f"{name}/{ws}/{given}/{colours}/{training}"
                    geo = f"{name}/{ws}/{given}/1/{training}"       # the geometry is stored with colours only
                    with torch.no_grad():
                        vk, lvk, le, sc = MG.ref_keys(fc, s0, cubes, res, bool(training))
                    assert len(vk) == v.shape[0] and len(lvk) == L.shape[0], tag
                    assert abs(vk).max(initial=0) < 2 ** 31 and len(vk) < 2 ** 31
                    arrays = {"verts": v.detach().numpy(), "faces": f.numpy().astype(np.int32),
                              "L": L.detach().numpy(), "vkeys": vk.astype(np.int32), "lvkeys": lvk.astype(np.int32),
                              "ledges": le.astype(np.int8)}
                    for k, a in arrays.items():
                        if colours:
                            out[f"{geo}/{k}"] = a
                        else:                                      # the colours change no geometry bit
                            assert np.array_equal(out[f"{geo}/{k}"].view(np.uint8), a.view(np.uint8)), (tag, k)
                    if colours:
                        out[tag + "/colours"] = vc.detach().numpy()
                    sc_all = sc
                    if v.shape[0] == 0:
                        continue
                    loss_of(v, L, vc).backward()
                    rows = torch.unique(cubes[torch.from_numpy(sc)].reshape(-1))
                    rest = torch.ones(x.shape[0], dtype=torch.bool)
                    rest[rows] = False
                    for key, g in (("gx", x.grad), ("gs", s.grad), ("gc", c.grad if colours else None)):
                        if g is None:
                            continue
                        assert not g[rest].any(), (tag, key)
                        out[f"{tag}/{key}"] = g[rows].numpy()
                    if f"{name}/grows" in out:
                        assert np.array_equal(out[f"{name}/grows"], rows.numpy()), tag
                    out[f"{name}/grows"] = rows.numpy().astype(np.int32)
                    if given:
                        wrest = torch.ones(w.shape[0], dtype=torch.bool)
                        wrest[sc] = False
                        assert not w.grad[wrest].any(), tag
                        out[f"{name}/gw_rows"] = sc.astype(np.int32)
                        out[tag + "/gw"] = w.grad[sc].numpy()
    return sc_all


def trellis_case(cube, res, rng):
    """SparseFeatures2Mesh.__call__ (cube2mesh.py) up to the extractor call, with seeded sparse features."""
    R1 = res + 1
    ijk = np.stack(np.meshgrid(*[np.arange(res)] * 3, indexing="ij"), -1).reshape(-1, 3)
    ctr = (ijk + 0.5) / res - 0.5
    d = np.linalg.norm(ctr * np.array([1.0, 0.8, 1.1]), axis=-1) - 0.1
    coords = torch.from_numpy(ijk[np.abs(d) < 1.0 / res]).int()
    N = coords.shape[0]
    corner = (coords[:, None, :].double() + cube["cube_corners"][None].double()) / res - 0.5
    sdf = (torch.linalg.vector_norm(corner * torch.tensor([1.0, 0.8, 1.1], dtype=torch.float64), dim=-1) - 0.1)
    q = torch.round(sdf * 1024) + torch.from_numpy(rng.integers(-6, 7, (N, 8)))
    # after the -1/res = -32/1024 bias each corner is (16 m + 1) / 1024, so a mean of 1 to 8 of them is never 0: no
    # grid point has s == 0 exactly, which keeps the case off L_dev's kink
    q = 32 + 16 * torch.round((q - 33) / 16) + 1
    sdf = q.float()[..., None] / 1024
    deform = torch.from_numpy(rng.integers(-64, 65, (N, 8, 3))).float() / 64
    color = torch.from_numpy(rng.integers(-64, 65, (N, 8, 6))).float() / 16
    weights = torch.from_numpy(rng.integers(-64, 65, (N, 21))).float() / 32
    sdf = sdf + (-1.0 / res)
    v_pos, v_attrs, _ = cube["sparse_cube2verts"](coords, torch.cat([sdf, deform, color], -1), training=False)
    v_attrs_d = cube["get_dense_attrs"](v_pos, v_attrs, res=R1, sdf_init=True)
    weights_d = cube["get_dense_attrs"](coords, weights, res=res, sdf_init=False)
    reg_v, reg_c = cube["construct_dense_grid"](res, "cpu")
    x = cube["get_defomed_verts"](reg_v, v_attrs_d[..., 1:4], res)
    prows = (v_pos[:, 0] * R1 + v_pos[:, 1]) * R1 + v_pos[:, 2]
    wrows = (coords[:, 0].long() * res + coords[:, 1]) * res + coords[:, 2]
    return (x, v_attrs_d[..., 0].contiguous(), weights_d, v_attrs_d[..., 4:].contiguous(), reg_c,
            prows.long().sort().values, wrows.sort().values)


def main():
    TFC, cube = load_trellis()
    _, NodeFC = MG.load_reference()
    out = {}
    for res in (64, 256):
        v, c = cube["construct_dense_grid"](res, "cpu")
        out[f"dense_grid/{res}/sha256"] = np.array([hashlib.sha256(v.numpy().tobytes()).hexdigest(),
                                                    hashlib.sha256(c.numpy().tobytes()).hexdigest()])
        out[f"dense_grid/{res}/shapes"] = np.array([v.shape[0], c.shape[0]])
        del v, c
    rng = np.random.default_rng(2025)

    x, s, w, c, cubes, prows, wrows = trellis_case(cube, 32, rng)
    out["trellis/prows"], out["trellis/wrows"] = prows.numpy().astype(np.int32), wrows.numpy().astype(np.int32)
    for k, t, rows in (("x", x, prows), ("s", s, prows), ("w", w, wrows), ("c", c, prows)):
        out[f"trellis/{k}"] = t[rows].numpy()
    # the rebuild the tests do: dense defaults, then the stored rows
    a = torch.arange(33)
    pts = torch.stack(torch.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
    rx = pts / 32 - 0.5 + (1 - 1e-8) / (32 * 2) * torch.tanh(torch.zeros(pts.shape))
    rx[prows] = x[prows]
    rs, rc, rw = torch.ones(s.shape), torch.zeros(c.shape), torch.zeros(w.shape)
    rs[prows], rc[prows], rw[wrows] = s[prows], c[prows], w[wrows]
    for got, want in ((rx, x), (rs, s), (rc, c), (rw, w)):
        assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    run_case(TFC, NodeFC, "trellis", 32, x, s, w, c, cubes, out)

    def coded(name, res, s_fn, C, wss=(0.99,)):
        grid, cubes = NodeFC(device="cpu").construct_voxel_grid(res)
        N, F = grid.shape[0], res ** 3
        xq = rng.integers(-60, 61, (N, 3)).astype(np.int8)
        sq = s_fn(grid * 2, N).astype(np.int16)
        wq = rng.integers(-64, 65, (F, 21)).astype(np.int8)
        cq = rng.integers(-64, 65, (N, C)).astype(np.int8)
        out[f"{name}/xq"], out[f"{name}/sq"], out[f"{name}/wq"], out[f"{name}/cq"] = xq, sq, wq, cq
        x = grid * 2 + torch.from_numpy(xq).float() / 4096
        run_case(TFC, NodeFC, name, res, x, torch.from_numpy(sq).float() / 1024, torch.from_numpy(wq).float() / 32,
                 torch.from_numpy(cq).float() / 16, cubes, out, wss)

    coded("random", 5, lambda p, N: rng.integers(-900, 700, N), 6, (0.99, 0.5))
    sphere = lambda p, N: np.round(((p.norm(dim=-1) - 0.62).numpy() + 0.04 * rng.standard_normal(N)) * 1024)
    nonzero = lambda q: np.where(q == 0, 1, q)       # no s == 0: keeps the case off L_dev's kink
    coded("c1", 8, lambda p, N: nonzero(sphere(p, N)), 1)
    coded("inside", 6, lambda p, N: -np.ones(N) * 300, 3)
    coded("outside", 6, lambda p, N: np.ones(N) * 300, 3)
    out["functional"] = np.array(A_VEC + B_VEC + [LAM], np.float64)
    out["colour_functional"] = np.array(K_VEC, np.float64)
    path = os.path.join(HERE, "ref_trellis_flexicubes.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
