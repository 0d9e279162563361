"""float64 restatement of the submanifold sparse convolution (include/gs_b200.h, "spconv"; gs_b200/spconv.py).

Rows are (b, x, y, z); weight is [Cout, k, k, k, Cin]; offset o = ((o0+r)*k + o1+r)*k + o2+r reads the row at
(b, x+o0, y+o1, z+o2).  A neighbour that is absent, outside the grid or in another batch item contributes nothing;
duplicate coordinates resolve to their smallest row; a row outside the grid or batch is nobody's neighbour and has
none.  k = 1 reads every row's own features.  The map here is built by brute force from a dict, independently of
the kernels' sort-and-search.
"""
import numpy as np


def brute_map(indices, spatial_shape, batch_size, k):
    """nbr int64 [N, k^3], -1 where absent."""
    ind = np.asarray(indices, dtype=np.int64).reshape(-1, 4)
    N = ind.shape[0]
    if k == 1:
        return np.arange(N, dtype=np.int64).reshape(N, 1)
    X, Y, Z = (int(v) for v in spatial_shape)
    B = int(batch_size)
    r = (k - 1) // 2

    def valid(b, x, y, z):
        return 0 <= b < B and 0 <= x < X and 0 <= y < Y and 0 <= z < Z

    first = {}
    for i in range(N):
        c = tuple(int(v) for v in ind[i])
        if valid(*c) and c not in first:
            first[c] = i
    nbr = np.full((N, k ** 3), -1, dtype=np.int64)
    for i in range(N):
        b, x, y, z = (int(v) for v in ind[i])
        if not valid(b, x, y, z):
            continue
        for a in range(k):
            for bb in range(k):
                for c in range(k):
                    nbr[i, (a * k + bb) * k + c] = first.get((b, x + a - r, y + bb - r, z + c - r), -1)
    return nbr


def _gather(x, nbr_col):
    g = np.zeros((nbr_col.shape[0], x.shape[1]), dtype=np.float64)
    on = nbr_col >= 0
    g[on] = x[nbr_col[on]]
    return g


def forward(features, weight, bias, nbr):
    """(out, bound): out [N, Cout] in float64 and bound = |bias| + sum |W| |x| per element, the scale of the rounding
    error of any summation order."""
    x = np.asarray(features, dtype=np.float64)
    W = np.asarray(weight, dtype=np.float64)
    Cout, Cin = W.shape[0], W.shape[-1]
    K3 = nbr.shape[1]
    Wf = W.reshape(Cout, K3, Cin)
    out = np.zeros((x.shape[0], Cout))
    bound = np.zeros((x.shape[0], Cout))
    for o in range(K3):
        g = _gather(x, nbr[:, o])
        out += g @ Wf[:, o, :].T
        bound += np.abs(g) @ np.abs(Wf[:, o, :]).T
    if bias is not None:
        b = np.asarray(bias, dtype=np.float64)
        out += b
        bound += np.abs(b)
    return out, bound


def backward(features, weight, nbr, grad_out):
    """(dgrad [N, Cin], wgrad [Cout, k, k, k, Cin], dbias [Cout], dgrad_bound, wgrad_bound) in float64: the exact
    adjoint of forward() over the same map, with sum |.| |.| bounds for dgrad and wgrad."""
    x = np.asarray(features, dtype=np.float64)
    W = np.asarray(weight, dtype=np.float64)
    go = np.asarray(grad_out, dtype=np.float64)
    Cout, Cin = W.shape[0], W.shape[-1]
    K3 = nbr.shape[1]
    Wf = W.reshape(Cout, K3, Cin)
    dx = np.zeros_like(x)
    dxb = np.zeros_like(x)
    dW = np.zeros((Cout, K3, Cin))
    dWb = np.zeros((Cout, K3, Cin))
    for o in range(K3):
        col = nbr[:, o]
        on = col >= 0
        np.add.at(dx, col[on], go[on] @ Wf[:, o, :])
        np.add.at(dxb, col[on], np.abs(go[on]) @ np.abs(Wf[:, o, :]))
        g = _gather(x, col)
        dW[:, o, :] = go.T @ g
        dWb[:, o, :] = np.abs(go).T @ np.abs(g)
    return dx, dW.reshape(W.shape), go.sum(0), dxb, dWb.reshape(W.shape)


def dense_to_rows(B, X, Y, Z):
    """indices [B*X*Y*Z, 4] of a fully occupied grid in C order."""
    g = np.stack(np.meshgrid(np.arange(B), np.arange(X), np.arange(Y), np.arange(Z), indexing="ij"), -1)
    return g.reshape(-1, 4).astype(np.int32)


def sphere_shell(res, radius=0.4, thickness=1.5, batch=1):
    """indices of a sphere shell of voxels in a res^3 grid (a surface-sparse set like TRELLIS's structured latents)."""
    c = (np.arange(res) + 0.5) / res - 0.5
    X, Y, Zc = np.meshgrid(c, c, c, indexing="ij")
    d = np.abs(np.sqrt(X ** 2 + Y ** 2 + Zc ** 2) - radius) * res
    xyz = np.argwhere(d <= thickness / 2)
    out = [np.concatenate([np.full((len(xyz), 1), b), xyz], 1) for b in range(batch)]
    return np.concatenate(out, 0).astype(np.int32)


def subdivide(indices):
    """each voxel -> its 8 children at twice the resolution (TRELLIS's SparseSubdivide), grouped by parent."""
    ind = np.asarray(indices, dtype=np.int32)
    ch = np.array([[0, a, b, c] for a in (0, 1) for b in (0, 1) for c in (0, 1)], dtype=np.int32)
    out = ind[:, None, :] * np.array([1, 2, 2, 2], dtype=np.int32) + ch[None]
    return out.reshape(-1, 4)


def edge_sets(seed=0):
    """(name, indices int32 [N, 4], spatial_shape, batch_size) sets at the map's edges: every face and corner of the
    grid, two batch items that touch in key space, unsorted rows, duplicate coordinates, isolated voxels, one row,
    and rows outside the grid or batch."""
    rng = np.random.default_rng(seed)
    out = []
    X, Y, Z = 5, 4, 6
    corners = np.array([[b, x, y, z] for b in (0, 1) for x in (0, X - 1) for y in (0, Y - 1) for z in (0, Z - 1)])
    faces = np.array([[b, x, y, z] for b in (0, 1) for x in range(X) for y in range(Y) for z in range(Z)
                      if x in (0, X - 1) or y in (0, Y - 1) or z in (0, Z - 1)])
    out.append(("corners", corners, (X, Y, Z), 2))
    out.append(("faces_unsorted", faces[rng.permutation(len(faces))], (X, Y, Z), 2))
    # batch 0's last voxel and batch 1's first are adjacent keys; z-rows ending at Z-1 next to rows starting at 0
    touch = np.array([[0, X - 1, Y - 1, Z - 1], [1, 0, 0, 0], [0, 2, 1, Z - 1], [0, 2, 2, 0], [1, 0, 0, 1],
                      [0, X - 1, Y - 1, Z - 2], [1, 1, 0, 0]])
    out.append(("batch_touch", touch, (X, Y, Z), 2))
    full = dense_to_rows(2, X, Y, Z)
    sub = full[rng.random(len(full)) < 0.35]
    dup = np.concatenate([sub, sub[rng.integers(0, len(sub), 40)], sub[:5]])
    out.append(("random_dups_unsorted", dup[rng.permutation(len(dup))], (X, Y, Z), 2))
    iso = np.array([[0, 0, 0, 0], [0, 2, 2, 2], [0, 4, 0, 5], [1, 2, 0, 3]])
    out.append(("isolated", iso, (X, Y, Z), 2))
    out.append(("one_row", np.array([[0, 1, 1, 1]]), (X, Y, Z), 1))
    bad = np.concatenate([sub[:30], np.array([[2, 0, 0, 0], [-1, 1, 1, 1], [0, X, 0, 0], [0, 0, -1, 0],
                                              [0, 0, 0, Z], [1, 1, 1, 1]])])
    out.append(("outside_rows", bad[rng.permutation(len(bad))], (X, Y, Z), 2))
    shell = sphere_shell(16)
    out.append(("shell16", shell[rng.permutation(len(shell))], (16, 16, 16), 1))
    return [(n, np.ascontiguousarray(i, dtype=np.int32), s, b) for n, i, s, b in out]
