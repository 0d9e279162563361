"""CPU tests of the submanifold sparse-conv oracle (oracle/spconv_oracle.py) and the spconv import shim.

The oracle is anchored on independent references: torch.nn.functional.conv3d in float64 on fully occupied grids,
a per-voxel brute-force loop on sparse edge sets, and torch autograd of the dense conv for the gradients."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import spconv_oracle as O


def _dense(ind, feats, B, X, Y, Z):
    d = np.zeros((B, feats.shape[1], X, Y, Z))
    for i, (b, x, y, z) in enumerate(ind):
        d[b, :, x, y, z] = feats[i]
    return d


@pytest.mark.parametrize("k", [1, 3])
def test_oracle_matches_dense_conv3d(k):
    rng = np.random.default_rng(k)
    B, X, Y, Z, Cin, Cout = 2, 3, 4, 5, 3, 4
    ind = O.dense_to_rows(B, X, Y, Z)
    perm = rng.permutation(len(ind))
    ind = ind[perm]
    x = rng.standard_normal((len(ind), Cin))
    W = rng.standard_normal((Cout, k, k, k, Cin))
    b = rng.standard_normal(Cout)
    out, bound = O.forward(x, W, b, O.brute_map(ind, (X, Y, Z), B, k))
    ref = F.conv3d(torch.from_numpy(_dense(ind, x, B, X, Y, Z)), torch.from_numpy(W).permute(0, 4, 1, 2, 3),
                   torch.from_numpy(b), padding=(k - 1) // 2).numpy()
    got = ref[ind[:, 0], :, ind[:, 1], ind[:, 2], ind[:, 3]]
    np.testing.assert_allclose(out, got, rtol=0, atol=1e-12)
    assert (bound >= np.abs(out) - 1e-12).all()


def _loop_conv(ind, x, W, b, spatial, B):
    """one voxel at a time, by the definition"""
    X, Y, Z = spatial
    k = W.shape[1]
    r = (k - 1) // 2
    rows = {}
    for i, c in enumerate(map(tuple, ind)):
        if 0 <= c[0] < B and 0 <= c[1] < X and 0 <= c[2] < Y and 0 <= c[3] < Z:
            rows.setdefault(c, i)
    out = np.zeros((len(ind), W.shape[0]))
    for i, (bb, x0, y0, z0) in enumerate(ind):
        out[i] = b
        if (bb, x0, y0, z0) not in rows:
            continue
        for a in range(k):
            for c in range(k):
                for d in range(k):
                    j = rows.get((bb, x0 + a - r, y0 + c - r, z0 + d - r))
                    if j is not None:
                        out[i] += W[:, a, c, d, :] @ x[j]
    return out


@pytest.mark.parametrize("name", [s[0] for s in O.edge_sets()])
def test_oracle_matches_brute_force_loop_on_edge_sets(name):
    ind, spatial, B = next((i, s, b) for n, i, s, b in O.edge_sets() if n == name)
    rng = np.random.default_rng(7)
    x = rng.standard_normal((len(ind), 5))
    W = rng.standard_normal((3, 3, 3, 3, 5))
    b = rng.standard_normal(3)
    out, _ = O.forward(x, W, b, O.brute_map(ind, spatial, B, 3))
    np.testing.assert_allclose(out, _loop_conv(ind, x, W, b, spatial, B), rtol=0, atol=1e-11)


def test_brute_map_edges():
    ind = np.array([[0, 4, 3, 5], [1, 0, 0, 0], [0, 4, 3, 5], [1, 0, 0, 1], [3, 0, 0, 0]], np.int32)
    nbr = O.brute_map(ind, (5, 4, 6), 2, 3)
    assert nbr[0, 13] == 0 and nbr[2, 13] == 0            # duplicates resolve to the smallest row
    assert nbr[1, 14] == 3 and nbr[3, 12] == 1            # +z / -z inside batch 1
    # batch 0's corner (4, 3, 5) and batch 1's origin are adjacent keys, but not neighbours
    assert (nbr[0] != 1).all() and (nbr[1] != 0).all()
    assert (nbr[4] == -1).all() and (nbr[:4] != 4).all()  # a row outside the batch has and is no neighbour
    assert (O.brute_map(ind, (5, 4, 6), 2, 1)[:, 0] == np.arange(5)).all()


@pytest.mark.parametrize("k", [1, 3])
def test_oracle_backward_matches_dense_autograd(k):
    rng = np.random.default_rng(10 + k)
    B, X, Y, Z, Cin, Cout = 2, 3, 3, 4, 3, 2
    ind = O.dense_to_rows(B, X, Y, Z)[rng.permutation(B * X * Y * Z)]
    x = rng.standard_normal((len(ind), Cin))
    W = rng.standard_normal((Cout, k, k, k, Cin))
    b = rng.standard_normal(Cout)
    go = rng.standard_normal((len(ind), Cout))
    dx, dW, db, _, _ = O.backward(x, W, O.brute_map(ind, (X, Y, Z), B, k), go)
    xt = torch.from_numpy(x).requires_grad_(True)
    Wt = torch.from_numpy(W).requires_grad_(True)
    bt = torch.from_numpy(b).requires_grad_(True)
    idx = torch.from_numpy(ind).long()
    dense = torch.zeros(B, X, Y, Z, Cin, dtype=torch.float64).index_put((idx[:, 0], idx[:, 1], idx[:, 2], idx[:, 3]), xt)
    y = F.conv3d(dense.permute(0, 4, 1, 2, 3), Wt.permute(0, 4, 1, 2, 3), bt, padding=(k - 1) // 2)
    rows = y[idx[:, 0], :, idx[:, 1], idx[:, 2], idx[:, 3]]
    (rows * torch.from_numpy(go)).sum().backward()
    np.testing.assert_allclose(dx, xt.grad.numpy(), atol=1e-11)
    np.testing.assert_allclose(dW, Wt.grad.numpy(), atol=1e-11)
    np.testing.assert_allclose(db, bt.grad.numpy(), atol=1e-11)


def test_oracle_backward_with_duplicates_is_the_adjoint():
    """<forward(x), g> = <x, dgrad(g)> and d/dW likewise, on a set with duplicate coordinates and outside rows"""
    ind, spatial, B = next((i, s, b) for n, i, s, b in O.edge_sets() if n == "random_dups_unsorted")
    rng = np.random.default_rng(3)
    nbr = O.brute_map(ind, spatial, B, 3)
    x = rng.standard_normal((len(ind), 4))
    W = rng.standard_normal((2, 3, 3, 3, 4))
    go = rng.standard_normal((len(ind), 2))
    out, _ = O.forward(x, W, None, nbr)
    dx, dW, db, _, _ = O.backward(x, W, nbr, go)
    assert np.isclose((out * go).sum(), (x * dx).sum(), rtol=1e-12)
    assert np.isclose((out * go).sum(), (W * dW).sum(), rtol=1e-12)
    assert np.allclose(db, go.sum(0))


def test_shell_and_subdivide():
    s = O.sphere_shell(32)
    assert len(s) > 0 and s.min() >= 0 and s[:, 1:].max() < 32
    d = O.subdivide(s)
    assert len(d) == 8 * len(s) and d[:, 1:].max() < 64
    assert len({tuple(r) for r in d}) == len(d)


# ---- the import shim -------------------------------------------------------------------------------------------------
def test_shim_names():
    import spconv
    import spconv.pytorch as sp
    for n in ("SparseConvTensor", "SubMConv3d", "SparseConv3d", "SparseInverseConv3d", "ConvAlgo"):
        assert hasattr(sp, n), n
    assert {a.name for a in sp.ConvAlgo} >= {"Native", "MaskImplicitGemm", "MaskSplitImplicitGemm"}
    assert spconv.pytorch is sp


def test_sparse_conv_tensor_as_trellis_builds_it():
    import spconv.pytorch as sp
    coords = torch.tensor([[0, 1, 2, 3], [0, 4, 0, 1], [1, 2, 2, 2]], dtype=torch.int32)
    feats = torch.randn(3, 2, 4)
    # SparseTensor.__init__ (spconv backend): spatial shape from coords, a list of 0-d tensors
    spatial_shape = list(coords.max(0)[0] + 1)[1:]
    data = sp.SparseConvTensor(feats.reshape(feats.shape[0], -1), coords, spatial_shape, 2)
    data._features = feats
    assert data.features is feats and data.spatial_shape == [5, 3, 4] and data.batch_size == 2
    # SparseTensor.replace: every attribute it copies
    new = sp.SparseConvTensor(data.features.reshape(data.features.shape[0], -1), data.indices, data.spatial_shape,
                              data.batch_size, data.grid, data.voxel_num, data.indice_dict)
    new._features = feats * 2
    for a in ("benchmark", "benchmark_record", "thrust_allocator", "_timer", "force_algo", "int8_scale"):
        setattr(new, a, getattr(data, a))
    new.indices = coords
    assert new.indice_dict is data.indice_dict
    r = data.replace_feature(feats[:, 0])
    assert r.indices is coords and r.indice_dict is data.indice_dict and r.features.shape == (3, 4)
    d = sp.SparseConvTensor(feats[:, 0], coords, [5, 3, 4], 2).dense()
    assert d.shape == (2, 4, 5, 3, 4)
    assert torch.equal(d[1, :, 2, 2, 2], feats[2, 0]) and torch.equal(d[0, :, 4, 0, 1], feats[1, 0])
    assert float(d.abs().sum()) == pytest.approx(float(feats[:, 0].abs().sum()))


def test_subm_weight_layout_and_names():
    import spconv.pytorch as sp
    c = sp.SubMConv3d(7, 5, 3, dilation=1, bias=True, indice_key="res_64", algo=sp.ConvAlgo.MaskImplicitGemm)
    sd = c.state_dict()
    assert set(sd) == {"weight", "bias"}
    assert sd["weight"].shape == (5, 3, 3, 3, 7) and sd["bias"].shape == (5,)
    c1 = sp.SubMConv3d(7, 5, 1, bias=False)
    assert c1.weight.shape == (5, 1, 1, 1, 7) and c1.bias is None and "bias" not in c1.state_dict()
    m = torch.nn.Module()
    m.conv = sp.SubMConv3d(4, 4, 3, algo=None)
    m.load_state_dict({"conv.weight": torch.zeros(4, 3, 3, 3, 4), "conv.bias": torch.zeros(4)}, strict=True)


def test_not_implemented_cases():
    import spconv.pytorch as sp
    with pytest.raises(NotImplementedError):
        sp.SparseConv3d(4, 4, 3, stride=2)
    with pytest.raises(NotImplementedError):
        sp.SparseInverseConv3d(4, 4, 3)
    with pytest.raises(NotImplementedError):
        sp.SubMConv3d(4, 4, 3, dilation=2)
    for k in (2, 4, 5):
        with pytest.raises(NotImplementedError):
            sp.SubMConv3d(4, 4, k)


def test_argument_errors_before_gpu_work():
    import spconv.pytorch as sp
    from gs_b200 import spconv as S
    coords = torch.zeros(3, 4, dtype=torch.int32)
    x = sp.SparseConvTensor(torch.zeros(3, 4), coords, [4, 4, 4], 1)
    with pytest.raises(RuntimeError, match="CPU"):
        sp.SubMConv3d(4, 4, 3)(x)
    with pytest.raises(ValueError, match="int32"):
        S.build_map(torch.zeros(3, 4, dtype=torch.int64), [4, 4, 4], 1)
    with pytest.raises(ValueError, match="N, 4"):
        S.build_map(torch.zeros(3, 3, dtype=torch.int32), [4, 4, 4], 1)
    for dt in (torch.bfloat16, torch.float64):
        with pytest.raises(TypeError):
            sp.SubMConv3d(4, 4, 3)(sp.SparseConvTensor(torch.zeros(3, 4, dtype=dt), coords, [4, 4, 4], 1))
    with pytest.raises(ValueError):
        S.spatial_dims([4, 4])
    with pytest.raises(ValueError):
        S.spatial_dims([4, 0, 4])
    with pytest.raises(ValueError):
        S.spatial_dims("abc")
    with pytest.raises(TypeError):
        sp.SubMConv3d(4, 4, 3)(torch.zeros(3, 4))
    with pytest.raises(ValueError):
        sp.SubMConv3d(5, 4, 3)(x)


def test_c_abi_scratch_bytes():
    from gs_b200 import _lib
    sb = _lib.lib.gs_b200_spconv_map_scratch_bytes
    assert sb(_lib.SPCONV_MAX_ROWS) > sb(1000) > 0
    assert sb(_lib.SPCONV_MAX_ROWS + 1) == 0 and sb(-1) == 0
    assert sb(1 << 32) == 0                      # N is int64: 2^32 rows are refused, not truncated to 0
