"""Generates tests/golden/ref_pointnet2.npz by running the REFERENCE's own pointnet2_ops callers (TriplaneGaussian's
snowflake decoder, models/snowflake/) on the CPU with a recording pointnet2_ops stand-in built on
oracle/pointnet2_oracle.py.

    COMFYUI_3D_PACK=/path/to/ComfyUI-3D-Pack python tests/golden/make_golden_pointnet2.py

Callers run, with seeded weights in eval mode:
  1. SPD_pp(dim_feat=128, up_factor=2, i=0) on 2048 points, then SPD_pp(dim_feat=128, up_factor=4, i=1) on its 4096
     (SkipTransformer's grouping_operation of [1,64,N] keys and [1,3,N] positions with query_knn's int32 16-NN
     indices, self included), then the backward of a fixed weighted sum of the 16384 output points and features.
  2. fps_subsample of that [1,16384,3] cloud to 2048 points.
  3. sample_and_group (ball query) and sample_and_group_knn on a seeded [1,3,1024] cloud with [1,16,1024] features,
     and PointNet_FP_Module (three_nn + three_interpolate) from 256 to 1024 points, with the backward of a weighted
     sum of their outputs.
For each call the file holds the operator, the arguments as the caller passed them (the [B,N,3] and [B,C,N] layouts
and int32 indices), and the result: whole when small, as the CRC32 of its bits otherwise.  Feature tensors with more
than 4 channels are kept at their first 4 channels (the operators act on each channel alone) and their results are
those of the kept channels.  Gradients are kept for the backward calls whose upstream gradient is small enough.
Nothing from the reference or from pointnet2_ops is stored: only numbers."""
import os
import sys
import types
import zlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import pointnet2_oracle as O  # noqa: E402

REF = os.environ["COMFYUI_3D_PACK"]
KEEP_C = 4                 # channels kept of a feature tensor
WHOLE = 4096               # results with at most this many elements are stored whole
GRAD_MAX = 12288           # upstream gradients with at most this many (kept) elements are stored
CALLS = []
SITE = ["?"]


def crc(a):
    return zlib.crc32(np.ascontiguousarray(a).tobytes()) & 0xffffffff


def _feat(t):
    return t.detach().numpy()[:, :KEEP_C].copy()


def _rec(op, **arrays):
    r = {"op": op, "site": SITE[0]}
    r.update(arrays)
    CALLS.append(r)
    return r


def _result(r, name, a):
    if a.size <= WHOLE:
        r[name] = a.copy()
    r[name + "_crc"] = np.uint32(crc(a))


class _FPS(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, npoint):
        r = _rec("furthest_point_sample", xyz=xyz.numpy().copy(), npoint=np.int64(npoint))
        out = O.furthest_point_sample(xyz.numpy(), npoint)
        _result(r, "out", out)
        out = torch.from_numpy(out)
        ctx.mark_non_differentiable(out)
        return out

    @staticmethod
    def backward(ctx, g):
        return None, None


class _Gather(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, idx, op):
        assert idx.dtype == torch.int32 and features.dtype == torch.float32
        r = _rec(op, features=_feat(features), idx=idx.numpy().copy(), C=np.int64(features.shape[1]))
        _result(r, "out", O.gather(r["features"], r["idx"]))
        ctx.r, ctx.N = r, features.shape[2]
        ctx.save_for_backward(idx)
        return torch.from_numpy(O.gather(features.detach().numpy(), idx.numpy()))

    @staticmethod
    def backward(ctx, g):
        (idx,) = ctx.saved_tensors
        gk = g.numpy()[:, :KEEP_C]
        if gk.size <= GRAD_MAX:
            ctx.r["grad_out"] = gk.copy()
            ctx.r["grad_features_crc"] = np.uint32(crc(O.gather_grad(gk, idx.numpy(), ctx.N)))
        return torch.from_numpy(O.gather_grad(g.numpy(), idx.numpy(), ctx.N)), None, None


class _BallQuery(torch.autograd.Function):
    @staticmethod
    def forward(ctx, radius, nsample, xyz, new_xyz):
        r = _rec("ball_query", radius=np.float64(radius), nsample=np.int64(nsample), xyz=xyz.numpy().copy(),
                 new_xyz=new_xyz.numpy().copy())
        out = O.ball_query(radius, nsample, xyz.numpy(), new_xyz.numpy())
        _result(r, "out", out)
        out = torch.from_numpy(out)
        ctx.mark_non_differentiable(out)
        return out

    @staticmethod
    def backward(ctx, g):
        return None, None, None, None


class _ThreeNN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, unknown, known):
        r = _rec("three_nn", unknown=unknown.numpy().copy(), known=known.numpy().copy())
        dist, idx = O.three_nn(unknown.numpy(), known.numpy())
        _result(r, "dist", dist)
        _result(r, "idx", idx)
        dist, idx = torch.from_numpy(dist), torch.from_numpy(idx)
        ctx.mark_non_differentiable(dist, idx)
        return dist, idx

    @staticmethod
    def backward(ctx, g, gi):
        return None, None


class _ThreeInterp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, idx, weight):
        r = _rec("three_interpolate", features=_feat(features), idx=idx.numpy().copy(),
                 weight=weight.detach().numpy().copy(), C=np.int64(features.shape[1]))
        _result(r, "out", O.three_interpolate(r["features"], r["idx"], r["weight"]))
        ctx.r, ctx.m = r, features.shape[2]
        ctx.save_for_backward(idx, weight)
        return torch.from_numpy(O.three_interpolate(features.detach().numpy(), idx.numpy(), weight.detach().numpy()))

    @staticmethod
    def backward(ctx, g):
        idx, weight = ctx.saved_tensors
        gk = g.numpy()[:, :KEEP_C]
        if gk.size <= GRAD_MAX:
            ctx.r["grad_out"] = gk.copy()
            ctx.r["grad_features_crc"] = np.uint32(crc(O.three_interpolate_grad(gk, idx.numpy(), weight.numpy(), ctx.m)))
        return torch.from_numpy(O.three_interpolate_grad(g.numpy(), idx.numpy(), weight.detach().numpy(), ctx.m)), None, None


def _install_stub():
    utils = types.ModuleType("pointnet2_ops.pointnet2_utils")
    utils.furthest_point_sample = lambda xyz, npoint: _FPS.apply(xyz, npoint)
    utils.gather_operation = lambda f, i: _Gather.apply(f, i, "gather_operation")
    utils.grouping_operation = lambda f, i: _Gather.apply(f, i, "grouping_operation")
    utils.ball_query = _BallQuery.apply
    utils.three_nn = _ThreeNN.apply
    utils.three_interpolate = _ThreeInterp.apply
    pkg = types.ModuleType("pointnet2_ops")
    pkg.pointnet2_utils = utils
    sys.modules["pointnet2_ops"] = pkg
    sys.modules["pointnet2_ops.pointnet2_utils"] = utils


def _seeded(module, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in module.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * (1.0 / max(1, p[0].numel()) ** 0.5))
        for name, b in module.named_buffers():
            if name.endswith("running_var"):
                b.copy_(torch.rand(b.shape, generator=g) + 0.5)
            elif name.endswith("running_mean"):
                b.copy_(torch.randn(b.shape, generator=g) * 0.1)
    return module.eval()


def main():
    _install_stub()
    sys.path.insert(0, os.path.join(REF, "Gen_3D_Modules", "TriplaneGaussian", "models"))
    from snowflake import utils as U
    from snowflake.SPD_pp import SPD_pp
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(1)

    SITE[0] = "spd_pp"
    pcd = (torch.rand(1, 3, 2048, generator=g) * 2 - 1).requires_grad_(True)
    cond0 = torch.randn(1, 128, 2048, generator=g)
    cond1 = torch.randn(1, 128, 4096, generator=g)
    s0 = _seeded(SPD_pp(dim_feat=128, up_factor=2, i=0), 2)
    s1 = _seeded(SPD_pp(dim_feat=128, up_factor=4, i=1), 3)
    p1, k1 = s0(pcd, cond0)
    p2, k2 = s1(p1, cond1, k1)
    w = torch.randn(p2.shape, generator=g)
    wk = torch.randn(k2.shape, generator=g)
    ((p2 * w).sum() + (k2 * wk).sum() * 1e-3).backward()

    SITE[0] = "fps_subsample"
    with torch.no_grad():
        sub = U.fps_subsample(p2.detach().permute(0, 2, 1).contiguous(), 2048)
    assert sub.shape == (1, 2048, 3)

    SITE[0] = "sample_and_group"
    xyz = (torch.rand(1, 3, 1024, generator=g) * 2 - 1).requires_grad_(True)
    pts = torch.randn(1, 16, 1024, generator=g).requires_grad_(True)
    nx, npnts, idx, gx = U.sample_and_group(xyz, pts, 256, 32, 0.2)
    loss = (npnts * torch.randn(npnts.shape, generator=g)).sum() + (nx * torch.randn(nx.shape, generator=g)).sum()
    SITE[0] = "sample_and_group_knn"
    nx2, np2, idx2, gx2 = U.sample_and_group_knn(xyz, pts, 256, 16)
    loss = loss + (np2 * torch.randn(np2.shape, generator=g)).sum()
    SITE[0] = "pointnet_fp"
    fp = _seeded(U.PointNet_FP_Module(32, [32, 32], use_points1=True, in_channel_points1=16), 4)
    p2s = torch.randn(1, 32, 256, generator=g).requires_grad_(True)
    out = fp(xyz, nx2, pts, p2s)
    loss = loss + (out * torch.randn(out.shape, generator=g)).sum()
    loss.backward()

    arrays = {"n_calls": np.int64(len(CALLS))}
    seen = {}                  # an argument repeated across calls is stored once; later calls hold "@<key>"
    for i, r in enumerate(CALLS):
        for k, v in r.items():
            v = np.asarray(v)
            h = (v.dtype.str, v.shape, crc(v))
            if v.size > 64 and h in seen:
                v = np.asarray("@" + seen[h])
            else:
                seen[h] = f"c{i}_{k}"
            arrays[f"c{i}_{k}"] = v
    path = os.path.join(HERE, "ref_pointnet2.npz")
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path), "bytes,", len(CALLS), "calls:",
          ", ".join(f"{r['site']}:{r['op']}" for r in CALLS))


if __name__ == "__main__":
    main()
