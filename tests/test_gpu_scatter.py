"""GPU tests of the torch_scatter drop-in (gs_b200.scatter, csrc/gs_scatter.cu) against the numpy oracle
(oracle/scatter_oracle.py) and the calls recorded from the reference's own callers (tests/golden/ref_scatter.npz).

Every comparison is bit for bit: fp32 sums and means are the ascending-position fold, integer sums and all max
results are exact, and gradients are gathers plus at most one division."""
import os
import warnings
import zlib

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import scatter_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
OPS = [("sum", np.float32), ("sum", np.int32), ("sum", np.int64), ("mean", np.float32),
       ("max", np.float32), ("max", np.int32), ("max", np.int64)]


def _ts():
    import torch_scatter
    return torch_scatter


def _fn(reduce):
    return {"sum": _ts().scatter_sum, "add": _ts().scatter_add, "mean": _ts().scatter_mean, "max": _ts().scatter_max}[reduce]


def _bits(a):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _eq(a, b):
    return np.array_equal(_bits(a), _bits(b))


def _strided(values, strides, grad=False):
    """(leaf, view): a CUDA tensor holding `values` with the recorded layout, stride-0 dims expanded and the rest in
    stride order, as a view of a contiguous leaf."""
    nd = values.ndim
    base = values[tuple(slice(0, 1) if strides[d] == 0 else slice(None) for d in range(nd))]
    perm = sorted(range(nd), key=lambda d: -abs(int(strides[d])))
    inv = np.argsort(perm).tolist()
    leaf = torch.from_numpy(np.ascontiguousarray(base.transpose(perm))).to(DEV).requires_grad_(grad)
    return leaf, leaf.permute(*inv).expand(values.shape)


def _values(rng, shape, dtype, reduce):
    if dtype == np.float32:
        v = rng.standard_normal(shape) * 10.0 ** rng.integers(-3, 4, shape)
        if reduce == "max":
            v = np.round(v * 4) / 4                     # exact ties
        return v.astype(np.float32)
    hi = 2 ** 40 if dtype == np.int64 else 2 ** 20
    if reduce == "max":
        hi = 50
    return rng.integers(-hi, hi, shape).astype(dtype)


def _index(rng, n, D, dist):
    if dist == "uniform":
        return rng.integers(0, D, n)
    if dist == "skewed":
        return np.minimum((D * rng.random(n) ** 4).astype(np.int64), D - 1)
    return np.full(n, D // 2, np.int64)


# ---- replay of the reference's recorded calls ------------------------------------------------------------------
def _recorded():
    z = np.load(os.path.join(GOLDEN, "ref_scatter.npz"))
    return z, int(z["ncalls"])


def test_replay_every_recorded_reference_call():
    z, n = _recorded()
    for i in range(n):
        p = f"c{i}_"
        red, dim = str(z[p + "reduce"]), int(z[p + "dim"])
        grad = (p + "grad_out") in z
        _, src = _strided(z[p + "src"], z[p + "src_strides"], grad)
        if grad:
            src.retain_grad()
        index = torch.from_numpy(z[p + "index"]).to(DEV)
        out = torch.from_numpy(z[p + "out_before"]).to(DEV) if (p + "out_before") in z else None
        ds = int(z[p + "dim_size"]) if (p + "dim_size") in z else None
        res = _fn(red)(src, index, dim=dim, out=out, dim_size=ds)
        val = res[0] if red == "max" else res
        if out is not None:
            assert val is out, i
        assert _eq(val, z[p + "out_after"]), (i, red)
        if red == "max":
            assert _eq(res[1], z[p + "argmax"]), i
        if grad:
            (val * torch.from_numpy(z[p + "grad_out"]).to(DEV)).sum().backward()
            assert _eq(src.grad, z[p + "grad_src"]), (i, red)


# ---- sweep against the oracle: each op and dtype x each caller's form x out / dim_size / inferred ----------------
def _form(name, rng, E, dtype, reduce, dist="uniform"):
    """(src numpy values, src tensor, index numpy as passed, dim, D)"""
    D = max(1, E // 7)
    if name == "fc9":                                   # FlexiCubes loss.py:58, [F,9] dim=-2, 1-D index
        v = _values(rng, (E, 9), dtype, reduce)
        return v, torch.from_numpy(v).to(DEV), _index(rng, E, D, dist), -2, D
    if name == "vec":                                   # loss.py:63,68 and remesh.py:218, 1-D
        v = _values(rng, (E,), dtype, reduce)
        return v, torch.from_numpy(v).to(DEV), _index(rng, E, D, dist), -1, D
    if name == "u3d":                                   # opt.py:137, [2E,S] with an [2E,1] index, dim=0
        v = _values(rng, (E, 3), dtype, reduce)
        return v, torch.from_numpy(v).to(DEV), _index(rng, E, D, dist)[:, None], 0, D
    if name == "rank4":                                 # remesh.py:336, expanded src, full [E',4] index
        r = _values(rng, (E,), dtype, reduce)
        v = np.broadcast_to(r[:, None], (E, 4))
        return v, torch.from_numpy(r).to(DEV)[:, None].expand(-1, 4), _index(rng, 4 * E, D, dist).reshape(E, 4), 0, D
    assert name == "tgs"                                # pointnet.py:63,75, permuted [B,C,T], [B,1,T] index, dim=-1
    B, C, T = 2, 24, E
    v = _values(rng, (B, T, C), dtype, reduce)
    return (v.transpose(0, 2, 1), torch.from_numpy(v).to(DEV).permute(0, 2, 1),
            np.stack([_index(rng, T, D, dist) for _ in range(B)])[:, None, :], -1, D)


def _check(reduce, v, src, idx_np, dim, D, mode, rng):
    ds = D + 3 if mode == "dim_size" else None
    index = torch.from_numpy(np.ascontiguousarray(idx_np)).to(DEV)
    out_np = None
    out = None
    if mode == "out":
        shape = list(v.shape)
        shape[dim] = D + 2
        out_np = _values(rng, tuple(shape), v.dtype, reduce)
        out = torch.from_numpy(out_np.copy()).to(DEV)
    r = O.scatter(reduce, v, idx_np, dim, out=out_np, dim_size=ds)
    res = _fn(reduce)(src, index, dim=dim, out=out, dim_size=ds)
    val = res[0] if reduce == "max" else res
    if out is not None:
        assert val is out
    assert val.shape == r["out"].shape
    assert _eq(val, r["out"]), (reduce, v.dtype, mode)
    if reduce == "max":
        assert _eq(res[1], r["argmax"])
    return r


@pytest.mark.parametrize("mode", ["out", "dim_size", "inferred"])
@pytest.mark.parametrize("form", ["fc9", "vec", "u3d", "rank4", "tgs"])
@pytest.mark.parametrize("reduce,dtype", OPS, ids=[f"{r}-{np.dtype(d).name}" for r, d in OPS])
def test_sweep_forms_against_the_oracle(reduce, dtype, form, mode):
    rng = np.random.default_rng(zlib.crc32(f"{reduce}{np.dtype(dtype).name}{form}{mode}".encode()))
    v, src, idx, dim, D = _form(form, rng, 3001, dtype, reduce)
    _check(reduce, v, src, idx, dim, D, mode, rng)


@pytest.mark.parametrize("dist", ["uniform", "skewed", "equal"])
@pytest.mark.parametrize("E", [1, 4097, 2 ** 16 + 3, 2 ** 22])
@pytest.mark.parametrize("reduce,dtype", [("sum", np.float32), ("mean", np.float32), ("max", np.float32),
                                          ("sum", np.int64), ("max", np.int32)])
def test_sweep_sizes_and_index_distributions(reduce, dtype, E, dist):
    rng = np.random.default_rng(E + len(dist))
    v, src, idx, dim, D = _form("vec", rng, E, dtype, reduce, dist)
    _check(reduce, v, src, idx, dim, D, "inferred", rng)
    if E <= 2 ** 16 + 3:
        v, src, idx, dim, D = _form("fc9", rng, E, dtype, reduce, dist)
        _check(reduce, v, src, idx, dim, D, "out", rng)


@pytest.mark.parametrize("reduce", ["mean", "max"])
def test_triplane_gaussian_full_size(reduce):
    """pointnet.py at its configured size: c [1,16384,512] permuted to [1,512,T], plane 32^2, with gradients."""
    rng = np.random.default_rng(5)
    T, C, P = 16384, 512, 32 * 32
    c_np = rng.standard_normal((1, T, C)).astype(np.float32)
    idx_np = rng.integers(0, P, (1, 1, T))
    c = torch.from_numpy(c_np).to(DEV).requires_grad_(True)
    index = torch.from_numpy(idx_np).to(DEV)
    g_np = rng.standard_normal((1, C, P)).astype(np.float32)
    if reduce == "mean":
        out = c.new_zeros(1, C, P)
        val = _ts().scatter_mean(c.permute(0, 2, 1), index, out=out)
        assert val is out
        r = O.scatter("mean", c_np.transpose(0, 2, 1), idx_np, -1, out=np.zeros((1, C, P), np.float32))
    else:
        val = _ts().scatter_max(c.permute(0, 2, 1), index, dim_size=P)[0]
        r = O.scatter("max", c_np.transpose(0, 2, 1), idx_np, -1, dim_size=P)
    assert _eq(val, r["out"])
    (val * torch.from_numpy(g_np).to(DEV)).sum().backward()
    gs, _ = O.scatter_backward(reduce, g_np, r, -1)
    assert _eq(c.grad, gs.transpose(0, 2, 1))


# ---- edges --------------------------------------------------------------------------------------------------------
def test_empty_source_and_dim_size_above_max():
    z = torch.zeros(0, device=DEV)
    zi = torch.zeros(0, dtype=torch.int64, device=DEV)
    assert _ts().scatter_sum(z, zi).shape == (0,)
    assert _ts().scatter_sum(z, zi, dim_size=4).tolist() == [0, 0, 0, 0]
    o, a = _ts().scatter_max(z, zi, dim_size=3)
    assert o.tolist() == [0, 0, 0] and a.tolist() == [0, 0, 0]
    assert _ts().scatter_mean(torch.zeros(0, 5, device=DEV), zi, dim=0, dim_size=2).tolist() == [[0.0] * 5] * 2
    s = torch.tensor([1.0, 2.0, 3.0], device=DEV)
    i = torch.tensor([0, 2, 0], device=DEV)
    assert _ts().scatter_sum(s, i, dim_size=6).tolist() == [4.0, 0, 2.0, 0, 0, 0]
    assert _ts().scatter_mean(s, i, dim_size=5).tolist() == [2.0, 0, 2.0, 0, 0]


def test_max_edge_cases_match_the_oracle():
    nan, inf, fmax = float("nan"), float("inf"), float(np.finfo(np.float32).max)
    src_np = np.array([1.0, 3.0, 3.0, nan, -inf, -fmax, 2.0, -0.0, 0.0, 5.0], np.float32)
    idx_np = np.array([0, 0, 0, 1, 2, 2, 3, 4, 4, 6])
    src, idx = torch.from_numpy(src_np).to(DEV), torch.from_numpy(idx_np).to(DEV)
    for out_np in (None, np.array([3.0, nan, -inf, 2.0, 1.0, -1.0, 4.0], np.float32),
                   np.array([-0.0, -inf, -fmax, nan, -0.0, 0.0, 5.0], np.float32)):
        r = O.scatter("max", src_np, idx_np, 0, out=None if out_np is None else out_np.copy())
        out = None if out_np is None else torch.from_numpy(out_np.copy()).to(DEV)
        o, a = _ts().scatter_max(src, idx, out=out)
        assert _eq(o, r["out"]) and _eq(a, r["argmax"])
    for dt in (torch.int32, torch.int64):
        lo = torch.iinfo(dt).min
        s = torch.tensor([lo, 4, 4, -2, lo], dtype=dt, device=DEV)
        o, a = _ts().scatter_max(s, torch.tensor([0, 1, 1, 2, 2], device=DEV), dim_size=4)
        assert o.tolist() == [0, 4, -2, 0] and a.tolist() == [5, 1, 3, 5]


def test_repeated_calls_give_identical_bits_and_strided_inputs_match_contiguous():
    rng = np.random.default_rng(2)
    v = rng.standard_normal((4, 9, 3000)).astype(np.float32)
    idx = torch.from_numpy(rng.integers(0, 50, (4, 1, 3000))).to(DEV)
    big = torch.from_numpy(np.ascontiguousarray(v.transpose(2, 0, 1))).to(DEV)     # [T,B,C]
    strided = big.permute(1, 2, 0)                                                 # [B,C,T] view
    cont = strided.contiguous()
    for red in ("sum", "mean", "max"):
        a = _fn(red)(strided, idx, dim=-1)
        b = _fn(red)(cont, idx.expand(4, 9, 3000).contiguous(), dim=-1)
        c = _fn(red)(strided, idx, dim=-1)
        a, b, c = [(x[0] if red == "max" else x) for x in (a, b, c)]
        assert _eq(a, b) and _eq(a, c), red
    out = torch.zeros(9, 4, 60, device=DEV).permute(1, 0, 2)                      # non-contiguous out
    ref = _ts().scatter_sum(cont, idx, dim=-1, dim_size=60)
    got = _ts().scatter_sum(strided, idx, dim=-1, out=out)
    assert got is out and _eq(got, ref)


@pytest.mark.parametrize("reduce", ["sum", "mean", "max"])
def test_gradients_wrt_src_and_out_equal_the_oracle(reduce):
    rng = np.random.default_rng(4)
    v = _values(rng, (5000, 6), np.float32, "max" if reduce == "max" else "sum")
    idx_np = rng.integers(0, 700, 5000)
    o_np = rng.standard_normal((703, 6)).astype(np.float32)
    g_np = rng.standard_normal((703, 6)).astype(np.float32)
    src = torch.from_numpy(v).to(DEV).requires_grad_(True)
    leaf = torch.from_numpy(o_np).to(DEV).requires_grad_(True)
    out = leaf * 1.0
    res = _fn(reduce)(src, torch.from_numpy(idx_np).to(DEV), dim=0, out=out)
    val = res[0] if reduce == "max" else res
    assert val is out
    (val * torch.from_numpy(g_np).to(DEV)).sum().backward()
    r = O.scatter(reduce, v, idx_np, 0, out=o_np.copy())
    assert _eq(val, r["out"])
    gs, go = O.scatter_backward(reduce, g_np, r, 0)
    assert _eq(src.grad, gs)
    if reduce == "max":
        assert leaf.grad is None or not leaf.grad.any()
    else:
        assert _eq(leaf.grad, go)


# ---- errors, host reads, streams, grad modes ----------------------------------------------------------------------
def test_out_of_range_indices_raise_before_out_is_touched_and_wrong_dtypes_raise():
    src = torch.arange(6, dtype=torch.float32, device=DEV)
    for bad, val in (([0, 1, 5, 2, 0, 1], 5), ([0, -1, 1, 2, 0, 1], -1)):
        out = torch.full((5,), 7.0, device=DEV)
        for fn in (_ts().scatter_sum, _ts().scatter_mean, _ts().scatter_max):
            with pytest.raises(RuntimeError, match=rf"index value {val} is out of bounds for dim_size 5"):
                fn(src, torch.tensor(bad, device=DEV), out=out)
            assert out.tolist() == [7.0] * 5
    with pytest.raises(RuntimeError, match="index value 3 is out of bounds for dim_size 3"):
        _ts().scatter_sum(src, torch.tensor([0, 1, 3, 0, 0, 0], device=DEV), dim_size=3)
    with pytest.raises(NotImplementedError, match="supported"):
        _ts().scatter_sum(src.double(), torch.zeros(6, dtype=torch.int64, device=DEV))
    with pytest.raises(NotImplementedError, match="torch.float32"):
        _ts().scatter_mean(src.long(), torch.zeros(6, dtype=torch.int64, device=DEV))
    with pytest.raises(NotImplementedError, match="torch.int64"):
        _ts().scatter_max(src, torch.zeros(6, dtype=torch.int32, device=DEV))
    with pytest.raises(RuntimeError, match="no CPU path"):
        _ts().scatter_sum(src, torch.zeros(6, dtype=torch.int64))
    with pytest.raises(RuntimeError):
        _ts().scatter_sum(torch.ones(4, 3, device=DEV), torch.zeros(4, 2, dtype=torch.int64, device=DEV), dim=0)


def test_one_host_read_per_forward_none_in_backward_and_the_current_stream():
    from gs_b200 import _lib
    rng = np.random.default_rng(8)
    src = torch.from_numpy(rng.standard_normal((20000, 9)).astype(np.float32)).to(DEV).requires_grad_(True)
    idx = torch.from_numpy(rng.integers(0, 3000, 20000)).to(DEV)
    for red in ("sum", "mean", "max"):
        _fn(red)(src, idx, dim=0)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("warn")
        try:
            with warnings.catch_warnings(record=True) as rec:
                warnings.simplefilter("always")
                res = _fn(red)(src, idx, dim=0)
            val = res[0] if red == "max" else res
            loss = (val * val.detach()).sum()
            torch.cuda.set_sync_debug_mode("error")
            n0 = _lib.lib.gs_b200_launch_count()
            src.grad = None
            loss.backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        syncs = [r for r in rec if "synchroniz" in str(r.message)]
        assert len(syncs) == 1, (red, [str(r.message) for r in syncs])
        assert _lib.lib.gs_b200_launch_count() - n0 == 1
    ref = _ts().scatter_sum(src.detach(), idx, dim=0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        on_side = _ts().scatter_sum(src.detach(), idx, dim=0)
    torch.cuda.current_stream().wait_stream(s)
    assert _eq(on_side, ref)
    with torch.inference_mode():
        a = _ts().scatter_mean(src, idx, dim=0)
        o = torch.zeros(3000, 9, device=DEV)
        assert _ts().scatter_sum(src, idx, dim=0, out=o) is o
    with torch.no_grad():
        b = _ts().scatter_mean(src, idx, dim=0)
        m = _ts().scatter_max(src, idx, dim=0)
    assert _eq(a, b) and not b.requires_grad and not m[0].requires_grad and _eq(o, ref)
