"""Generates tests/golden/ref_flexicubes.npz from the REFERENCE's own FlexiCubes code (tables.py and
FlexiCubes.__call__), run on the CPU.

    COMFYUI_3D_PACK=/path/to/ComfyUI-3D-Pack python tests/golden/make_golden_flexicubes.py [--reuse-grids]

(--reuse-grids copies the grid entries from the existing file: the reference's res-256 grid takes ~10 min on a CPU.)

Stores:
  * the reference's dmc_table, num_vd_table and check_table;
  * construct_voxel_grid outputs for res 6 and (4, 7, 5), and SHA-256 digests of (verts, cubes) bytes for res 100,
    127, 128 and 256;
  * seeded cases, each run with weight_scale 0.99 and 0.5, weights given and None, training on and off: the outputs
    with an order-free identity per vertex and L_dev entry, and the gradients of
    sum_v sin(a . v) + (b . v)^2 + lam * mean(L_dev) with respect to x, s and the [F,21] weight (surface rows only).
Inputs are stored as small integer codes with power-of-two scales, so the test rebuilds the exact fp32 inputs:
    x = grid * 2 + xq / 4096,  s = sq / 1024,  weight = wq / 32.
Nothing from the reference is copied into the repo: only the numeric outputs are stored."""
import argparse
import hashlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ["COMFYUI_3D_PACK"]
A_VEC, B_VEC, LAM = [0.7, -1.3, 0.4], [0.3, 0.5, -0.8], 2.5


def load_reference():
    tsrc = open(os.path.join(REF, "MVs_Algorithms/FlexiCubes/tables.py")).read()
    tables = types.ModuleType("FlexiCubes.tables")
    exec(compile(tsrc, "ref_flexi_tables", "exec"), tables.__dict__)
    sys.modules["FlexiCubes.tables"] = tables
    fsrc = open(os.path.join(REF, "MVs_Algorithms/FlexiCubes/flexicubes.py")).read().replace(
        "from .tables import *", "from FlexiCubes.tables import *")
    fns = {}
    exec(compile(fsrc, "ref_flexicubes", "exec"), fns)
    return tables, fns["FlexiCubes"]


def res3(res):
    return (res, res, res) if isinstance(res, int) else tuple(res)


def ref_keys(fc, s, cube_fx8, res, training):
    """Order-free identities of the reference's outputs, in the reference's output order, read from its own
    intermediate results."""
    R = res3(res)
    Sy, Sz = R[1] + 1, R[2] + 1
    surf, occ = fc._identify_surf_cubes(s, cube_fx8)
    case_ids = fc._get_case_id(occ, surf, list(res) if isinstance(res, tuple) else res)
    surf_edges, idx_map, counts, surf_mask = fc._identify_surf_edges(s, cube_fx8, surf)
    sc = torch.nonzero(surf)[:, 0]
    num_vd = fc.num_vd_table[case_ids]
    vkeys, lvk, le = [], [], []
    for num in torch.unique(num_vd).tolist():
        for loc in torch.nonzero(num_vd == num)[:, 0].tolist():
            case = int(case_ids[loc])
            for g in range(num):
                es = [int(e) for e in fc.dmc_table[case, g] if e != -1]
                k = int(sc[loc]) * 4096 + sum(1 << e for e in es)
                vkeys.append(k)
                lvk += [k] * len(es)
                le += es
    if training:
        group_mask = (counts == 4) & surf_mask
        edge_indices, _ = torch.sort(idx_map.reshape(-1)[group_mask], stable=True)
        E = surf_edges[edge_indices.reshape(-1, 4)[:, 0]]
        flip = s[E[:, 0]] > 0
        E = torch.cat([E[flip], E[~flip]])
        lo, d = E.min(1).values, (E[:, 0] - E[:, 1]).abs()
        axis = torch.where(d == Sy * Sz, 0, torch.where(d == Sz, 1, 2))
        vkeys += (-(1 + lo * 3 + axis)).tolist()
    return np.array(vkeys, np.int64), np.array(lvk, np.int64), np.array(le, np.int64), sc.numpy()


def run_case(FC, name, res, xq, sq, wq, out):
    R = res3(res)
    grid, cubes = FC(device="cpu").construct_voxel_grid(res)
    x0 = grid * 2 + torch.from_numpy(xq).float() / 4096
    s0 = torch.from_numpy(sq).float() / 1024
    w0 = torch.from_numpy(wq).float() / 32
    out[f"{name}/res"] = np.array(R)
    out[f"{name}/xq"], out[f"{name}/sq"], out[f"{name}/wq"] = xq, sq, wq
    for ws in (0.99, 0.5):
        fc = FC(device="cpu", weight_scale=ws)
        for given in (True, False):
            for training in (False, True):
                x = x0.clone().requires_grad_(True)
                s = s0.clone().requires_grad_(True)
                w = w0.clone().requires_grad_(True)
                kw = dict(beta_fx12=w[:, :12], alpha_fx8=w[:, 12:20], gamma_f=w[:, 20]) if given else {}
                v, f, L = fc(x, s, cubes, res, training=training, **kw)
                tag = f"{name}/{ws}/{int(given)}/{int(training)}"
                out[tag + "/verts"], out[tag + "/faces"], out[tag + "/L"] = \
                    v.detach().numpy(), f.numpy(), L.detach().numpy()
                with torch.no_grad():
                    vk, lvk, le, sc = ref_keys(fc, s0, cubes, res, training)
                assert len(vk) == v.shape[0] and len(lvk) == L.shape[0], (tag, len(vk), v.shape, len(lvk), L.shape)
                out[tag + "/vkeys"], out[tag + "/lvkeys"], out[tag + "/ledges"] = vk, lvk, le
                if v.shape[0] == 0:
                    continue
                vv = v
                loss = (torch.sin(vv @ torch.tensor(A_VEC)) + (vv @ torch.tensor(B_VEC)) ** 2).sum() + \
                    LAM * L.mean()
                loss.backward()
                out[tag + "/gx"], out[tag + "/gs"] = x.grad.numpy(), s.grad.numpy()
                if given:
                    out[tag + "/gw_rows"] = sc
                    out[tag + "/gw"] = w.grad[sc].numpy()
                    rest = torch.ones(w.shape[0], dtype=torch.bool)
                    rest[sc] = False
                    assert not w.grad[rest].any()


def count_inversions(tables, s, res):
    """(# inverted cubes with 5 inside corners, # with 6) under the ambiguity rule, from the reference's table."""
    R = res3(res)
    occ = (s < 0).reshape(R[0] + 1, R[1] + 1, R[2] + 1)
    ck = np.array(tables.check_table)
    case = np.zeros(R, np.int64)
    for c in range(8):
        case += occ[c & 1:R[0] + (c & 1), (c >> 1) & 1:R[1] + ((c >> 1) & 1), c >> 2:R[2] + (c >> 2)].numpy().astype(
            np.int64) << c
    flag = ck[case, 0] == 1
    n5 = n6 = 0
    for idx in zip(*np.nonzero(flag)):
        nb = np.array(idx) + ck[case[idx], 1:4]
        if (nb >= 0).all() and (nb < np.array(R)).all() and flag[tuple(nb)]:
            n = bin(int(case[idx])).count("1")
            n5 += n == 5
            n6 += n == 6
    return n5, n6


def main():
    tables, FC = load_reference()
    out = {"dmc_table": np.array(tables.dmc_table, np.int64), "num_vd_table": np.array(tables.num_vd_table, np.int64),
           "check_table": np.array(tables.check_table, np.int64)}
    fc = FC(device="cpu")
    ap = argparse.ArgumentParser()
    ap.add_argument("--reuse-grids", action="store_true")
    path = os.path.join(HERE, "ref_flexicubes.npz")
    if ap.parse_args().reuse_grids:
        old = np.load(path)
        out.update({k: old[k] for k in old.files if k.startswith("grid/")})
    grids = () if "grid/256/sha256" in out else (("6", 6), ("4_7_5", (4, 7, 5)))
    for tag, res in grids:
        v, c = fc.construct_voxel_grid(res)
        out[f"grid/{tag}/verts"], out[f"grid/{tag}/cubes"] = v.numpy(), c.numpy()
    for res in (100, 127, 128, 256) if grids else ():
        v, c = fc.construct_voxel_grid(res)
        out[f"grid/{res}/sha256"] = np.array([hashlib.sha256(v.numpy().tobytes()).hexdigest(),
                                              hashlib.sha256(c.numpy().tobytes()).hexdigest()])
        out[f"grid/{res}/shapes"] = np.array([v.shape[0], c.shape[0]])
    rng = np.random.default_rng(2024)

    def inputs(res, s_fn, deform=True):
        R = res3(res)
        grid, _ = fc.construct_voxel_grid(res)
        N, F = grid.shape[0], R[0] * R[1] * R[2]
        xq = rng.integers(-60, 61, (N, 3)).astype(np.int8) if deform else np.zeros((N, 3), np.int8)
        sq = s_fn(grid * 2, N).astype(np.int16)
        wq = rng.integers(-64, 65, (F, 21)).astype(np.int8)
        return xq, sq, wq

    sphere = lambda p, N: np.round(((p.norm(dim=-1) - 0.62).numpy() + 0.04 * rng.standard_normal(N)) * 1024)
    run_case(FC, "sphere", 12, *inputs(12, sphere), out)
    # random SDFs: both ambiguity inversions (5 and 6 inside corners) must occur
    for seed_try in range(100):
        xq, sq, wq = inputs(7, lambda p, N: rng.integers(-900, 700, N))
        n5, n6 = count_inversions(tables, torch.from_numpy(sq), 7)
        if n5 and n6:
            break
    else:
        raise RuntimeError("no random field hit both inversions")
    out["random/inversions"] = np.array([n5, n6])
    run_case(FC, "random", 7, xq, sq, wq, out)
    plane = lambda p, N: np.round((p @ torch.tensor([0.5, -0.7, 0.3]) + 0.1).numpy() * 1024)
    run_case(FC, "boundary", (7, 9, 8), *inputs((7, 9, 8), plane), out)
    zeros = lambda p, N: rng.integers(-1, 2, N) * 256
    xq, sq, wq = inputs(6, zeros)
    assert (sq == 0).sum() > 10
    run_case(FC, "zeros", 6, xq, sq, wq, out)
    run_case(FC, "inside", 8, *inputs(8, lambda p, N: -np.ones(N) * 300), out)
    run_case(FC, "outside", 8, *inputs(8, lambda p, N: np.ones(N) * 300), out)
    out["functional"] = np.array(A_VEC + B_VEC + [LAM], np.float64)
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {os.path.getsize(path) / 1e6:.2f} MB, random inversions {n5}/{n6}")


if __name__ == "__main__":
    main()
