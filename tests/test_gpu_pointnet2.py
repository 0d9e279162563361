"""GPU tests of the pointnet2_ops drop-in (gs_b200.pointnet2, csrc/pn2_ops.cu) against the numpy oracle
(oracle/pointnet2_oracle.py) and the calls recorded from TriplaneGaussian's own callers
(tests/golden/ref_pointnet2.npz).  Every comparison is bit for bit."""
import os
import zlib

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import pointnet2_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _U():
    from pointnet2_ops import pointnet2_utils
    return pointnet2_utils


def _t(a, grad=False):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV).requires_grad_(grad)


def _bits(a):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _eq(got, want, what=""):
    g, w = _bits(got), _bits(want)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = np.argwhere(g != w)
    assert bad.size == 0, f"{what}: {len(bad)} differ, first at {bad[:3].tolist()}"


def _cloud(rng, B, N, kind="uniform"):
    if kind == "uniform":
        return (rng.random((B, N, 3)) * 2 - 1).astype(np.float32)
    if kind == "lattice":                                    # equal distances everywhere: the tie rule decides
        return (rng.integers(-4, 5, (B, N, 3)) / 4.0).astype(np.float32)
    if kind == "dupes":
        base = (rng.random((B, max(1, N // 8), 3)) * 2 - 1).astype(np.float32)
        return base[:, rng.integers(0, base.shape[1], N)]
    if kind == "origin":                                     # many points inside the 1e-3 magnitude the FPS skips
        x = (rng.random((B, N, 3)) * 2 - 1).astype(np.float32)
        x[:, rng.random(N) < 0.5] *= np.float32(0.015)
        x[:, 0] = 0
        return x
    raise ValueError(kind)


# ---- furthest point sampling ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,N,npoint,kind", [
    (1, 1, 1, "uniform"), (1, 1, 4, "uniform"), (2, 33, 1, "uniform"), (1, 100, 150, "uniform"),
    (3, 1000, 100, "uniform"), (2, 1025, 300, "lattice"), (1, 2049, 256, "dupes"), (2, 5000, 200, "origin"),
    (1, 16384, 2048, "uniform"), (1, 16383, 64, "lattice"), (2, 16385, 300, "uniform"), (1, 40000, 129, "dupes"),
])
def test_fps(B, N, npoint, kind):
    rng = np.random.default_rng(N + npoint)
    xyz = _cloud(rng, B, N, kind)
    out = _U().furthest_point_sample(_t(xyz), npoint)
    assert out.dtype == torch.int32 and not out.requires_grad
    _eq(out, O.furthest_point_sample(xyz, npoint), "fps")


def test_fps_all_skipped_and_nan():
    xyz = np.zeros((2, 50, 3), np.float32)
    xyz[1, 7] = np.nan
    xyz[1, 20] = [1, 2, 3]
    for npoint in (1, 5, 80):
        _eq(_U().furthest_point_sample(_t(xyz), npoint), O.furthest_point_sample(xyz, npoint), f"npoint {npoint}")


# ---- ball query ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,N,P,S,radius,kind", [
    (1, 1000, 200, 32, 0.2, "uniform"), (2, 1025, 64, 16, 0.5, "lattice"), (1, 4097, 50, 64, 3.0, "uniform"),
    (2, 300, 40, 8, 0.0, "uniform"), (1, 31, 5, 40, 10.0, "uniform"), (1, 2000, 100, 1, 0.1, "dupes"),
    (1, 500, 300, 7, 0.25, "lattice"),
])
def test_ball_query(B, N, P, S, radius, kind):
    rng = np.random.default_rng(N + P)
    xyz = _cloud(rng, B, N, kind)
    q = np.concatenate([xyz[:, :P // 2], _cloud(rng, B, P - P // 2, kind) * 1.5], 1)     # hits and far queries
    if P > 3:
        q[:, 3] = 100.0                                            # no neighbour
    xyz[:, 5] = np.nan
    out = _U().ball_query(radius, S, _t(xyz), _t(q))
    _eq(out, O.ball_query(radius, S, xyz, q), "ball_query")


# ---- three-NN --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,n,m,kind", [
    (1, 1024, 256, "uniform"), (2, 777, 33, "lattice"), (1, 100, 1, "uniform"), (1, 100, 2, "uniform"),
    (1, 100, 3, "dupes"), (3, 513, 4097, "uniform"), (1, 300, 64, "dupes"),
])
def test_three_nn(B, n, m, kind):
    rng = np.random.default_rng(n + m)
    u, k = _cloud(rng, B, n, kind), _cloud(rng, B, m, kind)
    if m > 4:
        k[:, 2] = np.nan
        u[:, 1] = np.nan
    dist, idx = _U().three_nn(_t(u), _t(k))
    d, i = O.three_nn(u, k)
    _eq(dist, d, "dist")
    _eq(idx, i, "idx")


# ---- gathers and three-interpolate, forward and backward ----------------------------------------------------------------
def _grad_run(fn, feats, *args, grad_out):
    f = _t(feats, True)
    out = fn(f, *args)
    out.backward(_t(grad_out))
    return out, f.grad


@pytest.mark.parametrize("B,C,N,P,S,oob", [
    (1, 64, 4096, 4096, 16, False), (1, 3, 2048, 2048, 16, False), (2, 7, 1000, 300, 32, True), (3, 1, 5, 9, 4, True),
    (1, 16, 33, 1, 1, True),
])
def test_grouping(B, C, N, P, S, oob):
    rng = np.random.default_rng(C * N)
    f = rng.standard_normal((B, C, N)).astype(np.float32)
    idx = rng.integers(-3 if oob else 0, N + 3 if oob else N, (B, P, S)).astype(np.int32)
    idx[:, 0, :] = 0                                          # many hits on one slot
    g = rng.standard_normal((B, C, P, S)).astype(np.float32)
    out, gf = _grad_run(_U().grouping_operation, f, _t(idx), grad_out=g)
    _eq(out, O.gather(f, idx), "grouping")
    _eq(gf, O.gather_grad(g, idx, N), "grouping grad")
    _, gf2 = _grad_run(_U().grouping_operation, f, _t(idx), grad_out=g)
    _eq(gf2, gf, "grouping grad run to run")


@pytest.mark.parametrize("B,C,N,M,oob", [(1, 3, 16384, 2048, False), (2, 5, 100, 300, True), (1, 1, 1, 3, True)])
def test_gather(B, C, N, M, oob):
    rng = np.random.default_rng(N + M)
    f = rng.standard_normal((B, C, N)).astype(np.float32)
    idx = rng.integers(-2 if oob else 0, N + 2 if oob else N, (B, M)).astype(np.int32)
    g = rng.standard_normal((B, C, M)).astype(np.float32)
    out, gf = _grad_run(_U().gather_operation, f, _t(idx), grad_out=g)
    _eq(out, O.gather(f, idx), "gather")
    _eq(gf, O.gather_grad(g, idx, N), "gather grad")


@pytest.mark.parametrize("B,C,m,n,oob", [(1, 32, 256, 1024, False), (2, 128, 512, 2048, False), (2, 3, 10, 100, True),
                                         (1, 5, 1, 7, True)])
def test_three_interpolate(B, C, m, n, oob):
    rng = np.random.default_rng(m + n)
    f = rng.standard_normal((B, C, m)).astype(np.float32)
    idx = rng.integers(-1 if oob else 0, m + 1 if oob else m, (B, n, 3)).astype(np.int32)
    w = rng.random((B, n, 3)).astype(np.float32)
    g = rng.standard_normal((B, C, n)).astype(np.float32)
    out, gf = _grad_run(_U().three_interpolate, f, _t(idx), _t(w), grad_out=g)
    _eq(out, O.three_interpolate(f, idx, w), "three_interpolate")
    _eq(gf, O.three_interpolate_grad(g, idx, w, m), "three_interpolate grad")
    _, gf2 = _grad_run(_U().three_interpolate, f, _t(idx), _t(w), grad_out=g)
    _eq(gf2, gf, "three_interpolate grad run to run")


# ---- layouts, modes, streams, errors ---------------------------------------------------------------------------------
def test_non_contiguous_inputs():
    rng = np.random.default_rng(5)
    xyz = _cloud(rng, 2, 700, "uniform")
    xt = _t(xyz.transpose(0, 2, 1).copy()).permute(0, 2, 1)          # [B,N,3] view of a [B,3,N] tensor
    assert not xt.is_contiguous()
    _eq(_U().furthest_point_sample(xt, 50), O.furthest_point_sample(xyz, 50), "fps")
    _eq(_U().ball_query(0.3, 8, xt, xt[:, ::7]), O.ball_query(0.3, 8, xyz, xyz[:, ::7]), "ball_query")
    d, i = _U().three_nn(xt[:, ::2], xt[:, 1::5])
    od, oi = O.three_nn(xyz[:, ::2], xyz[:, 1::5])
    _eq(d, od, "dist")
    _eq(i, oi, "idx")
    f = rng.standard_normal((2, 300, 6)).astype(np.float32)
    ft = _t(f).permute(0, 2, 1)
    idx = rng.integers(0, 300, (2, 40, 5)).astype(np.int32)
    it = _t(idx.transpose(0, 2, 1).copy()).permute(0, 2, 1)
    _eq(_U().grouping_operation(ft, it), O.gather(f.transpose(0, 2, 1), idx), "grouping")
    g = _t(rng.standard_normal((2, 40, 6, 5)).astype(np.float32)).permute(0, 2, 1, 3)   # non-contiguous upstream grad
    fl = ft.detach().clone().requires_grad_(True)
    _U().grouping_operation(fl, it).backward(g)
    _eq(fl.grad, O.gather_grad(g.cpu().numpy(), idx, 300), "grouping grad")


def test_inference_mode_and_side_stream():
    rng = np.random.default_rng(6)
    xyz = _cloud(rng, 1, 3000, "uniform")
    f = rng.standard_normal((1, 8, 3000)).astype(np.float32)
    idx = rng.integers(0, 3000, (1, 100, 16)).astype(np.int32)
    want = O.furthest_point_sample(xyz, 200)
    with torch.inference_mode():
        _eq(_U().furthest_point_sample(_t(xyz), 200), want, "fps (inference)")
        _eq(_U().grouping_operation(_t(f), _t(idx)), O.gather(f, idx), "grouping (inference)")
    x, ft, it = _t(xyz), _t(f), _t(idx)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        a = _U().furthest_point_sample(x, 200)
        b = _U().grouping_operation(ft, it)
    s.synchronize()
    _eq(a, want, "fps (side stream)")
    _eq(b, O.gather(f, idx), "grouping (side stream)")


def test_argument_errors():
    U = _U()
    x = torch.zeros(1, 8, 3, device=DEV)
    f = torch.zeros(1, 4, 8, device=DEV)
    i3 = torch.zeros(1, 2, 3, dtype=torch.int32, device=DEV)
    with pytest.raises(TypeError):
        U.furthest_point_sample(x.half(), 2)
    with pytest.raises(TypeError):
        U.grouping_operation(f, i3.long())
    with pytest.raises(ValueError):
        U.furthest_point_sample(torch.zeros(1, 0, 3, device=DEV), 2)
    with pytest.raises(ValueError):
        U.furthest_point_sample(torch.zeros(1, 8, 2, device=DEV), 2)
    with pytest.raises(ValueError):
        U.gather_operation(torch.zeros(1, 4, 0, device=DEV), torch.zeros(1, 2, dtype=torch.int32, device=DEV))
    with pytest.raises(ValueError):
        U.grouping_operation(f, torch.zeros(2, 2, 3, dtype=torch.int32, device=DEV))
    with pytest.raises(ValueError):
        U.three_nn(x, torch.zeros(1, 0, 3, device=DEV))
    with pytest.raises(ValueError):
        U.three_interpolate(f, i3, torch.zeros(1, 3, 3, device=DEV))
    with pytest.raises(ValueError):
        U.ball_query(0.1, -1, x, x)
    with pytest.raises(RuntimeError):
        U.three_nn(x, x.cpu())


# ---- the reference's own calls ---------------------------------------------------------------------------------------
def _crc(a):
    return zlib.crc32(np.ascontiguousarray(_bits(a)).tobytes()) & 0xffffffff


def test_golden_replay():
    U = _U()
    calls = O.golden_calls(os.path.join(GOLDEN, "ref_pointnet2.npz"))
    for c in calls:
        op, what = c["op"], f"{c['site']}:{c['op']}"
        if op == "furthest_point_sample":
            res = {"out": U.furthest_point_sample(_t(c["xyz"]), int(c["npoint"]))}
        elif op == "ball_query":
            res = {"out": U.ball_query(float(c["radius"]), int(c["nsample"]), _t(c["xyz"]), _t(c["new_xyz"]))}
        elif op == "three_nn":
            d, i = U.three_nn(_t(c["unknown"]), _t(c["known"]))
            res = {"dist": d, "idx": i}
        else:
            f = _t(c["features"], True)
            if op == "three_interpolate":
                out = U.three_interpolate(f, _t(c["idx"]), _t(c["weight"]))
            else:
                out = getattr(U, op)(f, _t(c["idx"]))
            res = {"out": out}
            if "grad_out" in c:
                out.backward(_t(c["grad_out"]))
                res["grad_features"] = f.grad
        for k, v in res.items():
            assert _crc(v) == int(c[k + "_crc"]), f"{what} {k}"
            if k in c:
                _eq(v, c[k], f"{what} {k}")
