"""Generates tests/golden/ref_scatter.npz by running the REFERENCE's own torch_scatter callers on the CPU with a
recording torch_scatter stand-in built on oracle/scatter_oracle.py.

    COMFYUI_3D_PACK=/path/to/ComfyUI-3D-Pack python tests/golden/make_golden_scatter.py

Callers run:
  1. FlexiCubes loss.py::mesh_developable_reg on a seeded noisy icosphere, then the backward of a fixed weighted sum
     of its output (scatter_add: fp32 [F,9] with dim=-2, fp32 [F] with dim=-1, int32 [F] into an int32 out).
  2. Unique3D mesh_reconstruction MeshOptimizer (opt.py) steps and remesh() on an icosphere pulled toward an
     ellipsoid (scatter_mean into out, return ignored; scatter_max of expanded int64 src with a 1-D and a full index).
  3. TriplaneGaussian's two forms (models/pointclouds/pointnet.py:63,75) at reduced T and C, built here with the
     reference's argument pattern: its module cannot be imported without omegaconf, which this environment lacks.
For each recorded call the file holds the reduce, dim, dim_size (when passed), src (values, with its strides in
`src_strides`: 0 where expanded, permuted order otherwise), the index as passed, out before and after, argmax, and,
for differentiable calls, the upstream gradient and the resulting src gradient.  Only a bounded subset of calls is
kept.  Nothing from the reference or from torch_scatter is stored: only numbers."""
import importlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import scatter_oracle as O  # noqa: E402

REF = os.environ["COMFYUI_3D_PACK"]
CALLS = []
KEEP = {}                      # per call site label: how many calls to keep
SITE = ["?"]


class _Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, src, reduce, index, dim, out, dim_size, rec):
        r = O.scatter(reduce, src.detach().numpy(), index.numpy(), dim,
                      out=None if out is None else out.detach().numpy().copy(), dim_size=dim_size)
        ctx.r, ctx.reduce, ctx.dim, ctx.rec = r, reduce, dim, rec
        if rec is not None:
            rec["out_after"] = r["out"].copy()
            if "argmax" in r:
                rec["argmax"] = r["argmax"].copy()
        res = torch.from_numpy(np.ascontiguousarray(r["out"]))
        am = torch.from_numpy(np.ascontiguousarray(r["argmax"])) if "argmax" in r else None
        return res, am

    @staticmethod
    def backward(ctx, g, _):
        gs, _ = O.scatter_backward(ctx.reduce, g.numpy(), ctx.r, ctx.dim)
        if ctx.rec is not None:
            ctx.rec["grad_out"] = g.numpy().copy()
            ctx.rec["grad_src"] = gs.copy()
        return torch.from_numpy(np.ascontiguousarray(gs)), None, None, None, None, None, None


def _record(reduce, src, index, dim, out, dim_size):
    label = f"{SITE[0]}:{reduce}:{src.dtype}:{index.dim()}"
    if KEEP.get(label, 0) >= 2:
        return None
    KEEP[label] = KEEP.get(label, 0) + 1
    rec = dict(site=SITE[0], reduce=reduce, dim=dim, src=src.detach().numpy().copy(),
               src_strides=np.array(src.stride(), np.int64), index=index.numpy().copy())
    if dim_size is not None:
        rec["dim_size"] = dim_size
    if out is not None:
        rec["out_before"] = out.detach().numpy().copy()
    CALLS.append(rec)
    return rec


def _call(reduce, src, index, dim=-1, out=None, dim_size=None):
    rec = _record(reduce, src, index, dim, out, dim_size)
    res, am = _Fn.apply(src, reduce, index, dim, out, dim_size, rec)
    if out is not None:                               # in place, the same object returned
        with torch.no_grad():
            out.copy_(res)
        if res.requires_grad:
            out = res                                 # keeps the graph (the reference reassigns the return value)
        res = out
    return (res, am) if reduce == "max" else res


def install_stand_in():
    m = types.ModuleType("torch_scatter")
    m.scatter_sum = m.scatter_add = lambda src, index, dim=-1, out=None, dim_size=None: _call("sum", src, index, dim, out, dim_size)
    m.scatter_mean = lambda src, index, dim=-1, out=None, dim_size=None: _call("mean", src, index, dim, out, dim_size)
    m.scatter_max = lambda src, index, dim=-1, out=None, dim_size=None: _call("max", src, index, dim, out, dim_size)
    sys.modules["torch_scatter"] = m


def icosphere(level, seed, noise):
    t = (1 + 5 ** 0.5) / 2
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
         [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]]
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6],
         [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10],
         [8, 6, 7], [9, 8, 1]]
    v = [np.array(p, float) / np.linalg.norm(p) for p in v]
    for _ in range(level):
        mid, nf = {}, []
        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = v[a] + v[b]
                v.append(p / np.linalg.norm(p))
                mid[k] = len(v) - 1
            return mid[k]
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        f = nf
    v = np.array(v) * (1 + noise * np.random.default_rng(seed).standard_normal((len(v), 1)))
    return torch.tensor(v, dtype=torch.float32), torch.tensor(f, dtype=torch.int64)


def run_flexicubes():
    SITE[0] = "flexicubes"
    ns = {}
    exec(compile(open(os.path.join(REF, "MVs_Algorithms/FlexiCubes/loss.py")).read(), "ref_fc_loss", "exec"), ns)
    v, f = icosphere(2, seed=5, noise=0.05)
    v.requires_grad_(True)
    out = ns["mesh_developable_reg"](types.SimpleNamespace(vertices=v, faces=f))
    w = torch.linspace(0.5, 1.5, out.shape[0])
    (out * w).sum().backward()


def run_unique3d():
    SITE[0] = "unique3d"
    d = os.path.join(REF, "Gen_3D_Modules/Unique3D/mesh_reconstruction")
    pkg = types.ModuleType("u3d_mr")
    pkg.__path__ = [d]
    sys.modules["u3d_mr"] = pkg
    opt = importlib.import_module("u3d_mr.opt")
    v, f = icosphere(2, seed=9, noise=0.02)
    o = opt.MeshOptimizer(v.clone(), f.clone(), edge_len_lims=(0.05, 0.15))
    axes = torch.tensor([1.4, 1.0, 0.7])
    for step in range(15):
        SITE[0] = f"unique3d{step % 3}"
        o.zero_grad()
        vv = o.vertices
        loss = ((vv / axes).norm(dim=-1) - 1).square().sum()
        loss.backward()
        o.step()
        o.remesh()
    print("unique3d:", o.vertices.shape[0], "vertices,", o.faces.shape[0], "faces")


def run_triplane():
    SITE[0] = "triplane"
    g = torch.Generator().manual_seed(11)
    B, T, C, plane = 1, 1024, 16, 32
    index = torch.randint(0, plane * plane, (B, 1, T), generator=g)
    c = torch.randn(B, T, C, generator=g).requires_grad_(True)
    fea_plane = c.new_zeros(B, C, plane * plane)
    fea = _call("mean", c.permute(0, 2, 1), index, -1, fea_plane, None)       # pointnet.py:63
    fea2 = _call("max", c.permute(0, 2, 1), index, -1, None, plane * plane)[0]  # pointnet.py:75
    w = torch.randn(B, C, plane * plane, generator=g)
    ((fea * w).sum() + (fea2 * w.flip(-1)).sum()).backward()


def main():
    install_stand_in()
    run_flexicubes()
    run_unique3d()
    run_triplane()
    z = {"ncalls": np.int64(len(CALLS))}
    for i, rec in enumerate(CALLS):
        for k, val in rec.items():
            z[f"c{i}_{k}"] = np.asarray(val)
    path = os.path.join(HERE, "ref_scatter.npz")
    np.savez_compressed(path, **z)
    print(len(CALLS), "calls,", os.path.getsize(path), "bytes:",
          [(r["site"], r["reduce"], str(r["src"].dtype), r["src"].shape, "grad" if "grad_src" in r else "")
           for r in CALLS])


if __name__ == "__main__":
    main()
