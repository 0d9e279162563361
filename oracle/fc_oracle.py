"""FlexiCubes triangle-mesh extraction restated in plain torch, in any dtype and on any device, differentiated by
autograd.  The reference the CUDA kernels (csrc/ngp_flexicubes.cu) are tested against.

It is written from the extraction's rules on a regular grid of Rx x Ry x Rz cubes (S = R + 1 points per axis):
- point (i, j, k) has id (i * Sy + j) * Sz + k; cube (i, j, k) has id (i * Ry + j) * Rz + k; corner c of a cube is
  the point at offset (c & 1, (c >> 1) & 1, c >> 2).  A point is inside iff s < 0.
- the case table (groups of crossed edges, num_vd, ambiguity rows) comes from scripts/gen_fc_table.py.
- weights: beta = tanh(raw) * ws + 1, alpha likewise, gamma = sigmoid(raw) * ws + (1 - ws) / 2; a weight that is None
  is all ones.
- a flagged surface cube whose neighbour in the flagged direction is inside the grid and is itself a flagged surface
  cube (by its original case) takes the complement case.
- dual vertex of a group: sum(beta_e * ue_e) / sum(beta_e), ue_e the crossing of edge e with end weights s * alpha.
- L_dev, one entry per (dual vertex, group edge): |d_e - mean(d)|, d_e = |zc_e - vd|, zc_e the crossing with
  weights s.
- a crossed grid edge shared by 4 cubes makes a quad of the 4 cubes' dual vertices on that edge, cubes ascending,
  cycled [0,1,3,2] if s at the edge's first end > 0 else [2,3,1,0].  The first end is the lower one for axes 0 and
  2 and the upper one for axis 1.  Without training each quad splits along 0-2 if gamma0 * gamma2 > gamma1 * gamma3
  ([0,1,2],[0,2,3]), else ([0,1,3],[3,1,2]); with training a centre vertex is appended and the quad is fanned into
  four triangles (q_i, q_i+1, centre).

Output order (the kernels use the same): dual vertices by (cube, group), then centres; quads by (owning cube, axis),
the owning cube being the lowest of the four.  `keys` name every output independently of any order: a dual vertex
is cube * 4096 + (bit mask of its edges), a centre is -(1 + point * 3 + axis) for its grid edge, and an L_dev entry
is (its vertex's key, its cube edge)."""
import os
import sys

import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUBE_EDGES = [0, 1, 1, 5, 4, 5, 0, 4, 2, 3, 3, 7, 6, 7, 2, 6, 2, 0, 3, 1, 7, 5, 6, 4]
# per axis: the cube-local edge of the 4 cubes around a grid edge, cubes ascending
QUAD_EDGES = ([6, 4, 2, 0], [10, 9, 11, 8], [5, 1, 7, 3])
_TABLES = None


def tables():
    """(groups [256,4,7] long with -1 padding, num_vd [256], check [256,5]) from the generator's rules."""
    global _TABLES
    if _TABLES is None:
        sys.path.insert(0, os.path.join(_ROOT, "scripts"))
        import gen_fc_table as G
        groups, check = G.build_table()
        g = torch.full((256, G.MAX_GROUPS, G.MAX_GROUP_EDGES), -1, dtype=torch.long)
        for c, gs in enumerate(groups):
            for i, es in enumerate(gs):
                g[c, i, :len(es)] = torch.tensor(es)
        _TABLES = (g, torch.tensor([len(x) for x in groups]), torch.tensor(check))
    return _TABLES


def _res3(res):
    return (res, res, res) if isinstance(res, int) else tuple(int(r) for r in res)


def grid_ids(res, device):
    """(corner point ids [F,8], cube coords [F,3]) of the regular grid."""
    Rx, Ry, Rz = _res3(res)
    Sy, Sz = Ry + 1, Rz + 1
    ijk = torch.stack(torch.meshgrid(torch.arange(Rx, device=device), torch.arange(Ry, device=device),
                                     torch.arange(Rz, device=device), indexing="ij"), -1).reshape(-1, 3)
    c = torch.arange(8, device=device)
    off = torch.stack([c & 1, (c >> 1) & 1, c >> 2], -1)
    p = ijk[:, None, :] + off[None]
    return (p[..., 0] * Sy + p[..., 1]) * Sz + p[..., 2], ijk


def flexicubes(x, s, res, beta=None, alpha=None, gamma=None, training=False, weight_scale=0.99, dtype=None):
    """Returns (vertices [V,3], faces long [T,3], L_dev [E], keys) with keys = (vertex keys [V], L_dev vertex keys [E],
    L_dev edges [E]).  Differentiable in x, s and the raw weights through autograd."""
    dt = dtype or x.dtype
    dev = x.device
    Rx, Ry, Rz = _res3(res)
    F = Rx * Ry * Rz
    x, s = x.to(dt), s.to(dt)
    ws = weight_scale
    groups_t, num_vd_t, check_t = (t.to(dev) for t in tables())
    corners, ijk = grid_ids(res, dev)
    occ = s < 0
    case = (occ[corners].long() << torch.arange(8, device=dev)).sum(-1)
    surf = (case > 0) & (case < 255)
    # ambiguity: both this cube and its neighbour in the flagged direction are flagged (original cases)
    flag = (check_t[case, 0] == 1) & surf
    nb = ijk + check_t[case, 1:4]
    inb = ((nb >= 0) & (nb < torch.tensor([Rx, Ry, Rz], device=dev))).all(-1)
    nbi = ((nb[:, 0] * Ry + nb[:, 1]) * Rz + nb[:, 2]).clamp(0, F - 1)
    invert = flag & inb & flag[nbi]
    case = torch.where(invert, 255 - case, case)

    one = lambda n: torch.ones(n, dtype=dt, device=dev)
    be = torch.tanh(beta.to(dt)) * ws + 1 if beta is not None else one((F, 12))
    al = torch.tanh(alpha.to(dt)) * ws + 1 if alpha is not None else one((F, 8))
    ga = torch.sigmoid(gamma.to(dt)) * ws + (1 - ws) / 2 if gamma is not None else one((F,))

    # (cube, group, edge) entries, cube then group then edge order
    sc = torch.nonzero(surf)[:, 0]
    G = groups_t[case[sc]]                                   # [Ns,4,7]
    valid = G >= 0
    gvalid = valid.any(-1)                                   # [Ns,4]
    nvd = int(gvalid.sum())
    vd_id = torch.full(gvalid.shape, -1, dtype=torch.long, device=dev)
    vd_id[gvalid] = torch.arange(nvd, device=dev)
    ent_cube = sc[:, None, None].expand_as(G)[valid]
    ent_vd = vd_id[:, :, None].expand_as(G)[valid]
    ent_e = G[valid]
    ce = torch.tensor(CUBE_EDGES, device=dev).reshape(12, 2)
    ca, cb = ce[ent_e, 0], ce[ent_e, 1]
    pa, pb = corners[ent_cube, ca], corners[ent_cube, cb]
    xa, xb, sa, sb = x[pa], x[pb], s[pa, None], s[pb, None]
    wa, wb = sa * al[ent_cube, ca, None], sb * al[ent_cube, cb, None]
    ue = (xa * wb - xb * wa) / (wb - wa)
    zc = (xa * sb - xb * sa) / (sb - sa)
    b = be[ent_cube, ent_e][:, None]
    num = torch.zeros((nvd, 3), dtype=dt, device=dev).index_add(0, ent_vd, ue * b)
    den = torch.zeros((nvd, 1), dtype=dt, device=dev).index_add(0, ent_vd, b)
    vd = num / den
    d = torch.linalg.vector_norm(zc - vd[ent_vd], dim=-1)
    cnt = torch.zeros(nvd, dtype=dt, device=dev).index_add(0, ent_vd, torch.ones_like(d))
    mean = torch.zeros(nvd, dtype=dt, device=dev).index_add(0, ent_vd, d) / cnt
    L = (d - mean[ent_vd]).abs()
    vd_cube = sc[:, None].expand_as(gvalid)[gvalid]
    vd_gamma = ga[vd_cube]
    emask = torch.zeros(nvd, dtype=torch.long, device=dev).index_add(0, ent_vd, 1 << ent_e)
    vkey = vd_cube * 4096 + emask

    # quads
    vd_of = torch.full((F, 12), -1, dtype=torch.long, device=dev)
    vd_of[ent_cube, ent_e] = ent_vd
    S = (Rx + 1, Ry + 1, Rz + 1)
    quads, owners, ckeys = [], [], []
    occ3 = occ.reshape(S)
    for a in range(3):
        lo = [1, 1, 1]; hi = [S[0] - 1, S[1] - 1, S[2] - 1]
        lo[a], hi[a] = 0, S[a] - 1
        sl = tuple(slice(l, h) for l, h in zip(lo, hi))
        sl1 = tuple(slice(l + (q == a), h + (q == a)) for q, (l, h) in enumerate(zip(lo, hi)))
        cross = occ3[sl] != occ3[sl1]
        p = torch.nonzero(cross) + torch.tensor(lo, device=dev)         # grid points of crossed interior edges
        if p.shape[0] == 0:
            continue
        b_, c_ = [q for q in range(3) if q != a]
        cubes = []
        for db in range(2):
            for dc in range(2):
                cc = p.clone()
                cc[:, b_] += db - 1
                cc[:, c_] += dc - 1
                cubes.append((cc[:, 0] * Ry + cc[:, 1]) * Rz + cc[:, 2])
        q = torch.stack([vd_of[cubes[t], QUAD_EDGES[a][t]] for t in range(4)], -1)
        first = p.clone()
        if a == 1:
            first[:, 1] += 1
        fid = (first[:, 0] * S[1] + first[:, 1]) * S[2] + first[:, 2]
        flip = s[fid] > 0
        q = torch.where(flip[:, None], q[:, [0, 1, 3, 2]], q[:, [2, 3, 1, 0]])
        quads.append(q)
        owners.append(cubes[0] * 3 + a)
        pid = (p[:, 0] * S[1] + p[:, 1]) * S[2] + p[:, 2]
        ckeys.append(-(1 + pid * 3 + a))
    if quads:
        order = torch.argsort(torch.cat(owners))
        q = torch.cat(quads)[order]
        ckey = torch.cat(ckeys)[order]
    else:
        q = torch.zeros((0, 4), dtype=torch.long, device=dev)
        ckey = torch.zeros(0, dtype=torch.long, device=dev)
    g = vd_gamma[q]
    g02, g13 = g[:, 0] * g[:, 2], g[:, 1] * g[:, 3]
    if not training:
        split = (g02 > g13)[:, None]
        f1 = torch.where(split, q[:, [0, 1, 2]], q[:, [0, 1, 3]])
        f2 = torch.where(split, q[:, [0, 2, 3]], q[:, [3, 1, 2]])
        faces = torch.stack([f1, f2], 1).reshape(-1, 3)
        verts, keys = vd, vkey
    else:
        v = vd[q]
        ctr = (((v[:, 0] + v[:, 2]) / 2) * g02[:, None] + ((v[:, 1] + v[:, 3]) / 2) * g13[:, None]) / \
            (g02 + g13 + 1e-8)[:, None]
        cid = torch.arange(q.shape[0], device=dev) + nvd
        faces = torch.stack([torch.stack([q[:, i], q[:, (i + 1) % 4], cid], -1) for i in range(4)], 1).reshape(-1, 3)
        verts, keys = torch.cat([vd, ctr]), torch.cat([vkey, ckey])
    return verts, faces, L, (keys, vkey[ent_vd], ent_e)


def canonical(verts, faces, L, keys):
    """Order-free form of a mesh: ({vertex key: position}, set of faces as key triples rotated to start at their
    least key, {(vertex key, edge): L_dev})."""
    vk, lk, le = (k.tolist() for k in keys)
    V = {k: v for k, v in zip(vk, verts.tolist())}
    Fs = set()
    for a, b, c in faces.tolist():
        t = (vk[a], vk[b], vk[c])
        i = t.index(min(t))
        Fs.add(t[i:] + t[:i])
    Ld = {(k, e): l for k, e, l in zip(lk, le, L.tolist())}
    return V, Fs, Ld


def functional(verts, L, a, b, lam):
    """An order-invariant scalar of the outputs: sum_v sin(a . v) + (b . v)^2 + lam * mean(L_dev)."""
    a, b = a.to(verts), b.to(verts)
    out = (torch.sin(verts @ a) + (verts @ b) ** 2).sum()
    return out + lam * L.mean() if L.numel() else out


# ---- fixture helpers (tests/golden/ref_flexicubes.npz, written by tests/golden/make_golden_flexicubes.py) ----------
VARIANTS = [(ws, given, training) for ws in (0.99, 0.5) for given in (1, 0) for training in (0, 1)]


def fixture_inputs(z, name, device="cpu"):
    """(res, x fp32 [N,3], s fp32 [N], weight fp32 [F,21]) of a fixture case, rebuilt exactly from its codes."""
    res = tuple(int(r) for r in z[f"{name}/res"])
    from gs_b200.isosurface import voxel_grid
    grid, _ = voxel_grid(res, device)
    x = grid * 2 + torch.from_numpy(z[f"{name}/xq"]).to(device).float() / 4096
    s = torch.from_numpy(z[f"{name}/sq"]).to(device).float() / 1024
    w = torch.from_numpy(z[f"{name}/wq"]).to(device).float() / 32
    return res, x, s, w


def run_with_grads(fn, x, s, w, given, z):
    """Runs fn(x, s, beta, alpha, gamma) -> (verts, faces, L, ...) and differentiates the fixture's functional.
    Returns (verts, faces, L, rest, {"gx", "gs", "gw"}), gradients None when the mesh is empty."""
    x = x.detach().clone().requires_grad_(True)
    s = s.detach().clone().requires_grad_(True)
    w = w.detach().clone().requires_grad_(True)
    kw = (w[:, :12], w[:, 12:20], w[:, 20]) if given else (None, None, None)
    out = fn(x, s, *kw)
    v, f, L = out[:3]
    grads = None
    if v.shape[0]:
        fa = torch.tensor(z["functional"], dtype=torch.float64)
        functional(v, L, fa[:3], fa[3:6], float(fa[6])).backward()
        grads = {"gx": x.grad, "gs": s.grad, "gw": w.grad if given else None}
    return v.detach(), f, L.detach(), out[3:], grads


def assert_matches_fixture(z, tag, verts, faces, L, keys, grads, gw_rows=None, atol=1e-5, grtol=1e-4):
    """Mesh up to relabelling (faces exactly, vertices and L_dev within atol) and gradients within grtol of each
    tensor's largest magnitude, against the fixture entry `tag` ("case/ws/given/training")."""
    rk = (torch.from_numpy(z[tag + "/vkeys"]), torch.from_numpy(z[tag + "/lvkeys"]), torch.from_numpy(z[tag + "/ledges"]))
    RV, RF, RL = canonical(torch.from_numpy(z[tag + "/verts"]), torch.from_numpy(z[tag + "/faces"]),
                           torch.from_numpy(z[tag + "/L"]), rk)
    V, Fs, Ld = canonical(verts.double().cpu(), faces.cpu(), L.double().cpu(), tuple(k.cpu() for k in keys))
    assert V.keys() == RV.keys(), (tag, len(V), len(RV))
    assert Fs == RF, (tag, len(Fs), len(RF), len(Fs ^ RF))
    assert Ld.keys() == RL.keys(), tag
    if V:
        dv = max(max(abs(a - b) for a, b in zip(V[k], RV[k])) for k in V)
        assert dv <= atol, (tag, "verts", dv)
    if Ld:
        dl = max(abs(Ld[k] - RL[k]) for k in Ld)
        assert dl <= atol, (tag, "L_dev", dl)
    if grads is None:
        assert tag + "/gx" not in z.files, tag
        return
    names = [("gx", grads["gx"]), ("gs", grads["gs"])]
    if grads.get("gw") is not None:
        rows = torch.from_numpy(z[tag + "/gw_rows"])
        gw = grads["gw"].cpu()
        rest = torch.ones(gw.shape[0], dtype=torch.bool)
        rest[rows] = False
        assert not gw[rest].any(), (tag, "weight gradient off the surface cubes")
        names.append(("gw", gw[rows]))
    for n, g in names:
        ref = torch.from_numpy(z[tag + "/" + n]).double()
        err = float((g.double().cpu() - ref).abs().max())
        scale = float(ref.abs().max())
        assert err <= grtol * max(scale, 1e-12), (tag, n, err, scale)
