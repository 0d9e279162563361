"""CPU tests of the scatter oracle (oracle/scatter_oracle.py) and the torch_scatter import shim.

torch's CPU scatter_add_ is an independent implementation of the fp32 order the kernels keep (ascending position,
one fp32 add each), so the oracle's sums are anchored on it bit for bit.  The max rules are checked on hand cases."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from oracle import scatter_oracle as O

F32_MAX = np.finfo(np.float32).max


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _torch_add(src, index, dim, dim_size, out=None):
    idx = torch.from_numpy(np.ascontiguousarray(O.broadcast_index(index, src.shape, dim % src.ndim)))
    shape = list(src.shape)
    shape[dim] = dim_size
    o = torch.zeros(shape, dtype=torch.float32) if out is None else torch.from_numpy(out.copy())
    return o.scatter_add_(dim, idx, torch.from_numpy(src)).numpy()


@pytest.mark.parametrize("form", ["1d", "ec_dim0", "bct_dim-1", "1d_out"])
def test_oracle_sum_equals_torch_cpu_scatter_add_bit_for_bit(form):
    rng = np.random.default_rng(7)
    torch.set_num_threads(8)
    for trial in range(3):
        if form.startswith("1d"):
            E, D = 50000, 97
            src = (rng.standard_normal(E) * 10 ** rng.uniform(-3, 3, E)).astype(np.float32)
            index, dim = rng.integers(0, D, E), 0
        elif form == "ec_dim0":
            E, C, D = 20000, 7, 300
            src = rng.standard_normal((E, C)).astype(np.float32)
            index, dim = rng.integers(0, D, (E, 1)), 0
        else:
            B, C, T, D = 2, 16, 3000, 64
            src = rng.standard_normal((B, T, C)).astype(np.float32).transpose(0, 2, 1)   # permuted, like pointnet.py
            index, dim = rng.integers(0, D, (B, 1, T)), -1
        out = rng.standard_normal(D).astype(np.float32) if form == "1d_out" else None
        got = O.scatter("sum", src, index, dim, out=out, dim_size=D)["out"]
        ref = _torch_add(np.ascontiguousarray(src), index, dim, D, out)
        assert np.array_equal(_bits(got), _bits(ref)), (form, trial)


def test_oracle_mean_divides_the_fold_once_by_the_count():
    rng = np.random.default_rng(3)
    src = rng.standard_normal((1000, 5)).astype(np.float32)
    index = rng.integers(0, 40, (1000, 1))
    index[index == 7] = 8                               # an empty slot
    out = rng.standard_normal((40, 5)).astype(np.float32)
    r = O.scatter("mean", src, index, 0, out=out)
    s = _torch_add(src, index, 0, 40, out)
    cnt = np.bincount(index[:, 0], minlength=40).astype(np.float32)
    assert np.array_equal(_bits(r["out"]), _bits((s / np.maximum(cnt, 1)[:, None]).astype(np.float32)))
    assert np.array_equal(r["out"][7], out[7])


def test_oracle_max_hand_cases():
    nan, inf = np.float32(np.nan), np.float32(np.inf)
    src = np.array([1.0, 3.0, 3.0, nan, -inf, -F32_MAX, 2.0, -0.0, 0.0, 5.0], np.float32)
    idx = np.array([0, 0, 0, 1, 2, 2, 3, 4, 4, 6])
    r = O.scatter("max", src, idx, 0)
    # ties: first 3 wins; NaN never wins; -inf and -FLT_MAX do not beat the start -FLT_MAX (slot 2 -> 0);
    # -0 then +0: the first zero wins with its own sign; slot 5 is empty
    assert r["out"].tolist()[:4] == [3.0, 0.0, 0.0, 2.0]
    assert r["argmax"].tolist() == [1, 10, 10, 6, 7, 10, 9]
    assert np.signbit(r["out"][4]) and r["out"][5] == 0 and r["out"][6] == 5
    out = np.array([3.0, nan, -inf, 2.0, 1.0, -1.0, 4.0], np.float32)
    r = O.scatter("max", src, idx, 0, out=out.copy())
    # a tie with out's initial value loses (argmax = size); NaN start never replaced; -inf start beaten by -FLT_MAX
    assert r["argmax"].tolist() == [10, 10, 5, 10, 10, 10, 9]
    assert _bits(r["out"]).tolist() == _bits(np.array([3.0, nan, -F32_MAX, 2.0, 1.0, -1.0, 5.0], np.float32)).tolist()
    for dt in (np.int32, np.int64):
        lo = np.iinfo(dt).min
        s = np.array([lo, 4, 4, -2], dt)
        r = O.scatter("max", s, np.array([0, 1, 1, 2]), 0, dim_size=4)
        assert r["out"].tolist() == [0, 4, -2, 0] and r["argmax"].tolist() == [4, 1, 3, 4]
    r = O.scatter("max", np.zeros(0, np.float32), np.zeros(0, np.int64), 0, dim_size=3)
    assert r["out"].tolist() == [0, 0, 0] and r["argmax"].tolist() == [0, 0, 0]
    r = O.scatter("sum", np.zeros(0, np.float32), np.zeros(0, np.int64), 0)
    assert r["out"].shape == (0,)


def test_oracle_gradients_are_gathers():
    rng = np.random.default_rng(1)
    src = rng.standard_normal((30, 4)).astype(np.float32)
    idx = rng.integers(0, 6, 30)
    g = rng.standard_normal((6, 4)).astype(np.float32)
    for red in ("sum", "mean", "max"):
        f = O.scatter(red, src, idx, 0)
        t = torch.from_numpy(src).double().requires_grad_(True)
        it = torch.from_numpy(idx)[:, None].expand(30, 4)
        if red == "max":                                # torch_scatter's backward: scatter grad_out to the argmax
            ref = torch.zeros(31, 4).scatter_(0, torch.from_numpy(f["argmax"]), torch.from_numpy(g))[:30]
            gs, _ = O.scatter_backward(red, g, f, 0)
            assert np.array_equal(gs, ref.numpy())
            continue
        o = torch.zeros(6, 4, dtype=torch.float64).scatter_add(0, it, t)
        if red == "mean":
            o = o / torch.from_numpy(np.maximum(f["count"], 1)).double()
        (o * torch.from_numpy(g).double()).sum().backward()
        gs, _ = O.scatter_backward(red, g, f, 0)
        assert np.allclose(gs, t.grad.numpy(), rtol=1e-6, atol=0)


def test_oracle_reproduces_the_recorded_reference_calls():
    path = os.path.join(GOLDEN, "ref_scatter.npz")
    z = np.load(path, allow_pickle=False)
    n = int(z["ncalls"])
    assert n >= 6
    for i in range(n):
        p = f"c{i}_"
        red, dim = str(z[p + "reduce"]), int(z[p + "dim"])
        src, index = z[p + "src"], z[p + "index"]
        out = z[p + "out_before"] if (p + "out_before") in z else None
        ds = int(z[p + "dim_size"]) if (p + "dim_size") in z else None
        r = O.scatter(red, src, index, dim, out=out, dim_size=ds)
        assert np.array_equal(_bits(r["out"]), _bits(z[p + "out_after"])), i
        if red == "max":
            assert np.array_equal(r["argmax"], z[p + "argmax"]), i
        if (p + "grad_out") in z:
            gs, _ = O.scatter_backward(red, z[p + "grad_out"], r, dim)
            assert np.array_equal(_bits(gs), _bits(z[p + "grad_src"])), i


def test_torch_scatter_import_resolves_to_the_shim():
    import torch_scatter
    assert os.path.realpath(torch_scatter.__file__).startswith(os.path.realpath(os.path.join(ROOT, "comfyui-3d-pack_b200")))
    assert torch_scatter.__version__ == "2.1.2"
    for name in ("scatter_sum", "scatter_add", "scatter_mean", "scatter_max"):
        assert callable(getattr(torch_scatter, name))
    assert torch_scatter.scatter_add is torch_scatter.scatter_sum
    for name in ("scatter", "scatter_min", "scatter_mul", "segment_csr", "segment_sum_coo", "gather_csr",
                 "scatter_softmax", "scatter_logsumexp"):
        with pytest.raises(NotImplementedError, match="scatter_sum, scatter_add, scatter_mean and scatter_max"):
            getattr(torch_scatter, name)(torch.zeros(3), torch.zeros(3, dtype=torch.long))


def test_torch_scatter_cpu_tensors_raise_no_cpu_path():
    import torch_scatter
    src, idx = torch.ones(4), torch.tensor([0, 1, 1, 0])
    for fn in (torch_scatter.scatter_sum, torch_scatter.scatter_mean, torch_scatter.scatter_max):
        with pytest.raises(RuntimeError, match="no CPU path"):
            fn(src, idx)
