"""numpy restatement of the scatter rules gs_b200.scatter implements (torch_scatter 2.1's scatter_sum / scatter_mean /
scatter_max, with a fixed order).  Independent of the kernels: each rule is written in its sequential form.

- index broadcast: a 1-D index is reshaped to sit at `dim`, trailing axes are added, then it is broadcast to src.
- sum: starts from out (or 0) and adds src in ascending position along `dim`; for fp32 each add is one fp32 add
  (np.add.at applies its updates in index order, which is that left fold).
- mean (fp32): the sum, then one fp32 division by max(count, 1); count = index entries per slot.
- max: the running value is replaced only by a strictly greater element, starting from out (or the dtype's lowest);
  argmax = first position holding the final value among those greater than the start, or src.shape[dim] if none;
  without out, slots nothing won are 0.
"""
import numpy as np

LOWEST = {np.dtype(np.float32): np.float32(-np.finfo(np.float32).max),
          np.dtype(np.int32): np.int32(np.iinfo(np.int32).min),
          np.dtype(np.int64): np.int64(np.iinfo(np.int64).min)}


def broadcast_index(index, shape, dim):
    index = np.asarray(index)
    if index.ndim == 1:
        index = index.reshape((1,) * dim + index.shape)
    index = index.reshape(index.shape + (1,) * (len(shape) - index.ndim))
    return np.broadcast_to(index, shape)


def _to_rows(a, dim):
    """[size(dim), rest] view: position along dim first, every other coordinate flattened (row-major)."""
    a = np.moveaxis(a, dim, 0)
    return a.reshape(a.shape[0], int(np.prod(a.shape[1:], dtype=np.int64)))


def _from_rows(a, shape, dim):
    moved = (shape[dim],) + tuple(s for d, s in enumerate(shape) if d != dim)
    return np.moveaxis(a.reshape(moved), 0, dim)


def scatter(reduce, src, index, dim=-1, out=None, dim_size=None):
    """dict(out, argmax (max), count (mean / sum: index entries per output slot, out-shaped int64), index)."""
    src = np.asarray(src)
    dim = dim % src.ndim
    idx = broadcast_index(index, src.shape, dim).astype(np.int64)
    if out is not None:
        dim_size = out.shape[dim]
    elif dim_size is None:
        dim_size = int(idx.max()) + 1 if idx.size else 0
    oshape = list(src.shape)
    oshape[dim] = dim_size
    L = src.shape[dim]
    s2, i2 = _to_rows(src, dim), _to_rows(idx, dim)
    if i2.size and (i2.min() < 0 or i2.max() >= dim_size):
        raise IndexError("index out of range")
    R = s2.shape[1]
    cols = np.broadcast_to(np.arange(R)[None, :], i2.shape)
    init = (_to_rows(np.array(out, copy=True), dim) if out is not None else None)
    count = np.zeros((dim_size, R), np.int64)
    np.add.at(count, (i2, cols), 1)
    res = {"index": idx, "count": _from_rows(count, oshape, dim)}
    if reduce in ("sum", "add", "mean"):
        acc = init.copy() if init is not None else np.zeros((dim_size, R), src.dtype)
        np.add.at(acc, (i2, cols), s2)
        if reduce == "mean":
            acc = (acc / np.maximum(count, 1).astype(np.float32)).astype(np.float32)
        res["out"] = _from_rows(acc, oshape, dim)
        return res
    assert reduce == "max"
    start = init if init is not None else np.full((dim_size, R), LOWEST[src.dtype], src.dtype)
    p = np.broadcast_to(np.arange(L)[:, None], i2.shape)
    with np.errstate(invalid="ignore"):
        live = s2 > start[i2, cols]                      # strictly greater than the start; NaN never is
    tgt = (i2 * R + cols)[live]
    val, pos = s2[live], p[live]
    neg = -val.astype(np.float64) if src.dtype.kind == "f" else -val.astype(np.int64)   # live ints exceed the lowest
    order = np.lexsort((pos, neg, tgt))                 # per slot: largest value, then smallest position
    tgt, pos = tgt[order], pos[order]
    first = np.ones(tgt.shape, bool)
    first[1:] = tgt[1:] != tgt[:-1]
    arg = np.full(dim_size * R, L, np.int64)
    arg[tgt[first]] = pos[first]
    arg = arg.reshape(dim_size, R)
    won = arg < L
    o = start.copy() if init is not None else np.zeros((dim_size, R), src.dtype)
    wr, wc = np.nonzero(won)
    o[wr, wc] = s2[arg[wr, wc], wc]                     # the winner's own bits
    res["out"] = _from_rows(o, oshape, dim)
    res["argmax"] = _from_rows(arg, oshape, dim)
    return res


def scatter_backward(reduce, grad_out, fwd, dim):
    """(grad_src, grad_out_in) for an fp32 call whose forward returned `fwd`; grad_out_in is None for max."""
    idx = fwd["index"]
    dim = dim % idx.ndim
    g = np.asarray(grad_out, np.float32)
    g2, i2 = _to_rows(g, dim), _to_rows(idx, dim)
    cols = np.broadcast_to(np.arange(i2.shape[1])[None, :], i2.shape)
    if reduce in ("sum", "add"):
        return _from_rows(g2[i2, cols], idx.shape, dim), g
    if reduce == "mean":
        c = np.maximum(_to_rows(fwd["count"], dim), 1).astype(np.float32)
        return _from_rows((g2[i2, cols] / c[i2, cols]).astype(np.float32), idx.shape, dim), \
            _from_rows((g2 / c).astype(np.float32), g.shape, dim)
    a2 = _to_rows(fwd["argmax"], dim)
    p = np.broadcast_to(np.arange(i2.shape[0])[:, None], i2.shape)
    gs = np.where(a2[i2, cols] == p, g2[i2, cols], np.float32(0)).astype(np.float32)
    return _from_rows(gs, idx.shape, dim), None
