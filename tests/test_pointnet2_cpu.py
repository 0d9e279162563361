"""CPU tests of the pointnet2_ops oracle (oracle/pointnet2_oracle.py), the golden calls recorded from TriplaneGaussian's
own callers (tests/golden/ref_pointnet2.npz), and the pointnet2_ops import shim.

The oracle is anchored on independent float64 restatements: on coordinates that are multiples of 1/64 every squared
distance is exact in fp32, so FPS, ball query and three-NN must agree with float64 brute force index for index,
ties included; gradients are checked against torch autograd in float64."""
import os
import zlib

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from oracle import pointnet2_oracle as O

NPZ = os.path.join(GOLDEN, "ref_pointnet2.npz")


def _lattice(rng, shape, span=64):
    return (rng.integers(-span, span + 1, shape) / 64.0).astype(np.float32)


def _fps64(xyz, npoint):
    """float64 FPS by definition: max running distance, smallest index on ties, skipped points never picked."""
    xyz = xyz.astype(np.float64)
    skip = (xyz ** 2).sum(-1) <= 1e-3
    out = [0]
    temp = np.full(len(xyz), np.inf)
    for _ in range(1, npoint):
        temp = np.minimum(temp, ((xyz - xyz[out[-1]]) ** 2).sum(-1))
        cand = [(-temp[k], k) for k in range(len(xyz)) if not skip[k]]
        out.append(min(cand)[1] if cand else 0)
    return np.array(out, np.int32)


def test_fps_against_float64_brute_force():
    rng = np.random.default_rng(0)
    for N, npoint in ((1, 3), (37, 37), (300, 80), (130, 200)):
        xyz = _lattice(rng, (2, N, 3))
        xyz[:, ::7] = 0                                    # points the skip rule drops
        got = O.furthest_point_sample(xyz, npoint)
        for b in range(2):
            np.testing.assert_array_equal(got[b], _fps64(xyz[b], npoint))


def test_fps_skip_rule_and_all_skipped():
    xyz = np.array([[[0.01, 0.01, 0.01], [0.02, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 0.0]]], np.float32)
    # 3e-4 and 4e-4 are skipped, so only point 2 can be picked; later steps repeat it (distance 0 beats the skipped)
    np.testing.assert_array_equal(O.furthest_point_sample(xyz, 5), [[0, 2, 2, 2, 2]])
    np.testing.assert_array_equal(O.furthest_point_sample(np.zeros((1, 4, 3), np.float32), 3), [[0, 0, 0]])
    # the fp32 magnitude is compared as a double
    assert O.fps_skipped(np.array([0.0316, 0, 0], np.float32)) and not O.fps_skipped(np.array([0.0317, 0, 0], np.float32))


def _ball64(radius, nsample, xyz, q):
    out = np.zeros((len(q), nsample), np.int32)
    for i, p in enumerate(q.astype(np.float64)):
        hits = [k for k in range(len(xyz)) if ((xyz[k].astype(np.float64) - p) ** 2).sum() < radius * radius]
        hits = hits[:nsample]
        if hits:
            out[i] = hits[0]
            out[i, :len(hits)] = hits
    return out


@pytest.mark.parametrize("radius", [0.0, 0.25, 0.5, 3.0])
def test_ball_query_against_float64_brute_force(radius):
    rng = np.random.default_rng(1)
    xyz = _lattice(rng, (1, 200, 3), 16)
    q = _lattice(rng, (1, 40, 3), 16)
    np.testing.assert_array_equal(O.ball_query(radius, 8, xyz, q)[0], _ball64(radius, 8, xyz[0], q[0]))


@pytest.mark.parametrize("m", [1, 2, 3, 50])
def test_three_nn_against_float64_lexsort(m):
    rng = np.random.default_rng(2)
    u = _lattice(rng, (1, 60, 3), 8)
    k = _lattice(rng, (1, m, 3), 8)
    dist, idx = O.three_nn(u, k)
    d64 = ((u[0, :, None, :].astype(np.float64) - k[0, None, :, :]) ** 2).sum(-1)
    for i in range(60):
        order = np.lexsort((np.arange(m), d64[i]))[:3]
        np.testing.assert_array_equal(idx[0, i, :len(order)], order)
        np.testing.assert_array_equal(dist[0, i, :len(order)], np.sqrt(d64[i, order]).astype(np.float32))
        assert np.all(np.isinf(dist[0, i, len(order):])) and np.all(idx[0, i, len(order):] == 0)


def test_three_nn_nan_never_enters():
    u = np.zeros((1, 1, 3), np.float32)
    k = np.array([[[np.nan, 0, 0], [1, 0, 0], [2, 0, 0], [0.5, 0, 0]]], np.float32)
    dist, idx = O.three_nn(u, k)
    np.testing.assert_array_equal(idx, [[[3, 1, 2]]])
    np.testing.assert_array_equal(dist, [[[0.5, 1, 2]]])


def test_gather_and_interpolate_gradients_against_torch_float64():
    rng = np.random.default_rng(3)
    B, C, N, n = 2, 5, 40, 30
    f = rng.standard_normal((B, C, N))
    idx = rng.integers(-2, N + 2, (B, n, 3)).astype(np.int32)        # out-of-range entries read 0 and get no gradient
    w = rng.random((B, n, 3))
    g = rng.standard_normal((B, C, n))
    ft = torch.tensor(f, requires_grad=True)
    ok = torch.tensor((idx >= 0) & (idx < N))
    safe = torch.tensor(np.where(idx >= 0, np.where(idx < N, idx, 0), 0)).long()
    gathered = torch.gather(ft, 2, safe.view(B, 1, n * 3).expand(B, C, n * 3)).view(B, C, n, 3)
    gathered = gathered * ok.view(B, 1, n, 3)
    out = (gathered * torch.tensor(w).view(B, 1, n, 3)).sum(-1)
    out.backward(torch.tensor(g), retain_graph=True)
    np.testing.assert_allclose(O.three_interpolate(f, idx, w), out.detach().numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(O.three_interpolate_grad(g, idx, w, N, np.float64), ft.grad.numpy(), rtol=1e-12, atol=1e-12)
    ft.grad = None
    (gathered.reshape(B, C, n, 3) * torch.tensor(g)[..., None]).sum().backward()
    np.testing.assert_allclose(O.gather_grad(np.repeat(g[..., None], 3, -1), idx, N, np.float64), ft.grad.numpy(),
                               rtol=1e-12, atol=1e-12)


def test_fp32_fold_is_the_ascending_left_fold():
    rng = np.random.default_rng(4)
    g = (rng.standard_normal((1, 2, 500)) * 10.0 ** rng.integers(-4, 5, (1, 2, 500))).astype(np.float32)
    idx = rng.integers(0, 7, (1, 500)).astype(np.int32)
    got = O.gather_grad(g, idx, 7)
    for c in range(2):
        for j in range(7):
            acc = np.float32(0)
            for p in np.flatnonzero(idx[0] == j):
                acc = np.float32(acc + g[0, c, p])
            assert got[0, c, j].view(np.uint32) == acc.view(np.uint32)


def test_golden_file_is_self_consistent():
    calls = O.golden_calls(NPZ)
    sites = {(c["site"], c["op"]) for c in calls}
    assert ("spd_pp", "grouping_operation") in sites and ("fps_subsample", "furthest_point_sample") in sites
    assert {"ball_query", "three_nn", "three_interpolate", "gather_operation"} <= {c["op"] for c in calls}
    grads = 0
    for c in calls:
        for k, v in O.replay(c).items():
            assert zlib.crc32(np.ascontiguousarray(v).tobytes()) & 0xffffffff == int(c[k + "_crc"]), (c["site"], c["op"], k)
            if k in c:
                np.testing.assert_array_equal(v, c[k])
        grads += "grad_out" in c
        if "idx" in c and c["op"] != "three_nn":
            assert c["idx"].dtype == np.int32
    assert grads >= 3
    spd = [c for c in calls if c["site"] == "spd_pp"]
    assert {c["idx"].shape for c in spd} == {(1, 2048, 16), (1, 4096, 16)}
    for c in spd:                                     # query_knn includes the point itself
        assert np.array_equal(c["idx"][0, :, 0], np.arange(c["idx"].shape[1])) or \
            np.mean(c["idx"][0, :, 0] == np.arange(c["idx"].shape[1])) > 0.99


def test_shim_names():
    import pointnet2_ops
    from pointnet2_ops import pointnet2_modules, pointnet2_utils as U
    assert pointnet2_ops.__version__ == "3.0.0"
    assert pointnet2_ops.__file__.startswith(os.path.join(ROOT, "comfyui-3d-pack_b200"))
    for name in ("furthest_point_sample", "gather_operation", "grouping_operation", "ball_query", "three_nn",
                 "three_interpolate"):
        assert callable(getattr(U, name))
    for name in ("FurthestPointSampling", "GatherOperation", "GroupingOperation", "BallQuery", "ThreeNN",
                 "ThreeInterpolate"):
        assert issubclass(getattr(U, name), torch.autograd.Function)
    for fn in (U.QueryAndGroup, U.GroupAll, pointnet2_modules.PointnetSAModule, pointnet2_modules.PointnetSAModuleMSG,
               pointnet2_modules.PointnetFPModule):
        with pytest.raises(NotImplementedError):
            fn(0.1, 16)


def test_c_abi_scratch_bytes():
    from gs_b200 import _lib
    sb = _lib.lib.gs_b200_pn2_backward_scratch_bytes
    assert sb(2, 3, 100, 50, 1) > sb(2, 3, 100, 50, 0) > 0
    assert sb(1, 1, 0, 1, 0) == 0 and sb(1, 1, 1, -1, 0) == 0
    assert sb(1, 1, 8, 1 << 32, 0) == 0          # M is int64: 2^32 index entries are refused, not truncated to 0


def test_cpu_tensors_and_dtypes_raise_before_gpu_work():
    from pointnet2_ops import pointnet2_utils as U
    xyz = torch.zeros(1, 8, 3)
    f = torch.zeros(1, 4, 8)
    i2 = torch.zeros(1, 2, dtype=torch.int32)
    i3 = torch.zeros(1, 2, 3, dtype=torch.int32)
    calls = [lambda a: U.furthest_point_sample(a, 4), lambda a: U.gather_operation(f, a),
             lambda a: U.ball_query(0.1, 4, a, xyz), lambda a: U.three_nn(a, xyz),
             lambda a: U.three_interpolate(f, i3, a), lambda a: U.grouping_operation(f, a)]
    for fn, a in zip(calls, (xyz, i2, xyz, xyz, i3.float(), i3)):
        with pytest.raises(RuntimeError, match="CPU"):
            fn(a)
        with pytest.raises(TypeError):
            fn(a.double() if a.is_floating_point() else a.long())
        with pytest.raises(TypeError):
            fn(a.numpy())
