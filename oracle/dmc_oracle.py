"""Dual marching cubes (the diso.DiffDMC contract of include/ngp_b200.h) restated in plain torch, in float64 by default,
on any device, differentiated by autograd.  The reference the CUDA kernels (csrc/ngp_dmc.cu) are tested against.

The rules, written from the contract and not from the kernels:
- the grid is padded by one ring of samples iso + 1 with deform 0; padded point (I, J, K) sits at
  (I-1, J-1, K-1) + deform.  A sample is below iff value < iso, iso rounded to fp32 first.
- a cube is live iff its 8 corners are finite; a live cube's case has bit c set iff corner c (offset (c & 1,
  (c >> 1) & 1, c >> 2)) is below; its dual vertices are the case's groups (fc_oracle.tables(), no ambiguity swap).
- a crossed edge is crossed from its lower end a: p_a + t (p_b - p_a), t = (iso - s_a) / (s_b - s_a); a vertex is
  the mean of its group's crossings, divided per column by dim - 1 with normalize.
- a quad per crossed edge whose 4 cubes are live, from the lowest cube, its right-hand normal pointing from the above
  end to the below end; split into (0,1,3),(1,2,3) iff that pair's largest corner cosine is strictly smaller than
  that of (0,1,2),(0,2,3) (cosines on the returned vertices).
- vertices by (padded cube, group), quads by (lower padded point, axis).  Empty iff no NaN and min >= iso or
  max <= iso.

Also: `counts` (vertex and quad counts only, cheap enough for 513^3), the mesh predicates of mc_oracle, and the
seeded TripoSG-like field used by the tests and scripts/bench_dmc.py."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.fc_oracle import CUBE_EDGES, tables
from oracle.mc_oracle import euler_characteristic, is_oriented_manifold, signed_volume  # noqa: F401

# local edge of the cube edge along axis a whose lower corner is corner c
EDGE_AT = {}
for _e in range(12):
    _c0, _c1 = sorted(CUBE_EDGES[2 * _e:2 * _e + 2])
    EDGE_AT[((_c0 ^ _c1).bit_length() - 1, _c0)] = _e
# (db, dc) of the 4 cubes P - db e_b - dc e_c around an edge along a ((a, b, c) cyclic), from the lowest cube, for a
# lower end above (normal +e_a) and below (normal -e_a)
CYCLE = (((1, 1), (0, 1), (0, 0), (1, 0)), ((1, 1), (1, 0), (0, 0), (0, 1)))
_GROUP_OF = None


def group_of():
    """[256, 12] long: the group of each edge per case, -1 if not crossed."""
    global _GROUP_OF
    if _GROUP_OF is None:
        groups = tables()[0]
        g = torch.full((256, 12), -1, dtype=torch.long)
        for c in range(256):
            for i in range(groups.shape[1]):
                for e in groups[c, i].tolist():
                    if e >= 0:
                        g[c, e] = i
        _GROUP_OF = g
    return _GROUP_OF


def iso32(iso):
    return float(np.float32(iso))


def is_empty(grid, iso):
    """diso's test: no NaN and (min >= iso or max <= iso)."""
    iso = iso32(iso)
    return not bool(torch.isnan(grid).any()) and (not bool((grid < iso).any()) or not bool((grid > iso).any()))


def _cases(vp, iso):
    """(case long [CX,CY,CZ], live bool) of every padded cube."""
    below, finite = vp < iso, torch.isfinite(vp)
    CX, CY, CZ = (s - 1 for s in vp.shape)
    case = torch.zeros((CX, CY, CZ), dtype=torch.long, device=vp.device)
    live = torch.ones((CX, CY, CZ), dtype=torch.bool, device=vp.device)
    for c in range(8):
        sl = (slice(c & 1, (c & 1) + CX), slice((c >> 1) & 1, ((c >> 1) & 1) + CY), slice(c >> 2, (c >> 2) + CZ))
        case |= below[sl].long() << c
        live &= finite[sl]
    return case, live


def _quad_mask(below, live, a):
    """(mask over the region of lower ends, region start) of the crossed edges along a whose 4 cubes are live."""
    P = below.shape
    lo = [1, 1, 1]
    lo[a] = 0
    sl = tuple(slice(lo[q], P[q] - 1) for q in range(3))
    up = tuple(slice(lo[q] + (q == a), P[q] - 1 + (q == a)) for q in range(3))
    m = below[sl] != below[up]
    b, c = (a + 1) % 3, (a + 2) % 3
    for db in range(2):
        for dc in range(2):
            d = [0, 0, 0]
            d[b], d[c] = db, dc
            m = m & live[tuple(slice(lo[q] - d[q], P[q] - 1 - d[q]) for q in range(3))]
    return m, lo


def _pad(grid, iso):
    return F.pad(grid, (1, 1, 1, 1, 1, 1), value=iso + 1.0)


def counts(grid, iso=0.0):
    """(V, Q) without building the mesh."""
    iso = iso32(iso)
    if is_empty(grid, iso):
        return 0, 0
    vp = _pad(grid.float(), iso)
    case, live = _cases(vp, iso)
    nvd = tables()[1].to(grid.device)
    V = int(torch.where(live, nvd[case], 0).sum())
    del case
    below = vp < iso
    Q = sum(int(_quad_mask(below, live, a)[0].sum()) for a in range(3))
    return V, Q


def dmc(grid, deform=None, iso=0.0, return_quads=False, normalize=True, dtype=torch.float64):
    """(verts [V,3], faces long [Q,4] or [2Q,3], info) with info = {"quads": long [Q,4], "margin": [Q] the gap between
    the two configs' largest corner cosines}.  Differentiable in grid and deform through autograd."""
    dev = grid.device
    X, Y, Z = grid.shape
    iso = iso32(iso)
    empty = {"quads": torch.zeros((0, 4), dtype=torch.long, device=dev), "margin": torch.zeros(0, dtype=dtype, device=dev)}
    if is_empty(grid, iso):
        return (torch.zeros((0, 3), dtype=dtype, device=dev),
                torch.zeros((0, 4 if return_quads else 3), dtype=torch.long, device=dev), empty)
    vp = _pad(grid.to(dtype), iso)
    PX, PY, PZ = vp.shape
    axes = [torch.arange(n, device=dev, dtype=dtype) - 1 for n in (PX, PY, PZ)]
    pos = torch.stack(torch.meshgrid(*axes, indexing="ij"), -1)
    if deform is not None:
        pos = pos + F.pad(deform.to(dtype), (0, 0, 1, 1, 1, 1, 1, 1))
    case, live = _cases(vp, iso)
    groups_t, num_vd_t, _ = (t.to(dev) for t in tables())
    gof = group_of().to(dev)
    cf, lf = case.reshape(-1), live.reshape(-1)
    nvd = torch.where(lf, num_vd_t[cf], 0)
    first = torch.cumsum(nvd, 0) - nvd
    V = int(nvd.sum())

    # crossings of every (surface cube, group, edge) entry
    sc = torch.nonzero(nvd)[:, 0]
    G = groups_t[cf[sc]]                                              # [Ns, 4, 7]
    valid = G >= 0
    ent_cube = sc[:, None, None].expand_as(G)[valid]
    ent_vid = (first[sc][:, None, None] + torch.arange(G.shape[1], device=dev)[None, :, None]).expand_as(G)[valid]
    e = G[valid]
    ce = torch.tensor(CUBE_EDGES, device=dev).reshape(12, 2)
    ca, cb = torch.minimum(ce[e, 0], ce[e, 1]), torch.maximum(ce[e, 0], ce[e, 1])
    CY, CZ = PY - 1, PZ - 1
    ci, cj, ck = ent_cube // (CY * CZ), (ent_cube // CZ) % CY, ent_cube % CZ

    def point(c):
        return ci + (c & 1), cj + ((c >> 1) & 1), ck + (c >> 2)

    pa, pb = point(ca), point(cb)
    sa, sb = vp[pa], vp[pb]
    t = ((iso - sa) / (sb - sa))[:, None]
    cr = pos[pa] + t * (pos[pb] - pos[pa])
    n = torch.zeros(V, dtype=dtype, device=dev).index_add(0, ent_vid, torch.ones_like(sa))
    verts = torch.zeros((V, 3), dtype=dtype, device=dev).index_add(0, ent_vid, cr) / n[:, None]
    if normalize:
        verts = verts / torch.tensor([X - 1, Y - 1, Z - 1], dtype=dtype, device=dev)

    # quads
    below = vp < iso
    quads, keys = [], []
    for a in range(3):
        m, lo = _quad_mask(below, live, a)
        P = torch.nonzero(m) + torch.tensor(lo, device=dev)
        if P.shape[0] == 0:
            continue
        b, c = (a + 1) % 3, (a + 2) % 3
        side = below[P[:, 0], P[:, 1], P[:, 2]]
        vid = {}
        for db in range(2):
            for dc in range(2):
                C = P.clone()
                C[:, b] -= db
                C[:, c] -= dc
                cid = (C[:, 0] * CY + C[:, 1]) * CZ + C[:, 2]
                vid[db, dc] = first[cid] + gof[cf[cid], EDGE_AT[a, (db << b) | (dc << c)]]
        q_above = torch.stack([vid[x] for x in CYCLE[0]], -1)
        q_below = torch.stack([vid[x] for x in CYCLE[1]], -1)
        quads.append(torch.where(side[:, None], q_below, q_above))
        keys.append(((P[:, 0] * PY + P[:, 1]) * PZ + P[:, 2]) * 3 + a)
    if quads:
        q = torch.cat(quads)[torch.argsort(torch.cat(keys))]
    else:
        q = torch.zeros((0, 4), dtype=torch.long, device=dev)

    with torch.no_grad():
        p = verts.detach()[q]                                         # [Q, 4, 3]
        m1 = torch.maximum(max_cos(p[:, 0], p[:, 1], p[:, 3]), max_cos(p[:, 1], p[:, 2], p[:, 3]))
        m2 = torch.maximum(max_cos(p[:, 0], p[:, 1], p[:, 2]), max_cos(p[:, 0], p[:, 2], p[:, 3]))
    if return_quads:
        faces = q
    else:
        one = (m1 < m2)[:, None]
        f1 = torch.where(one, q[:, [0, 1, 3]], q[:, [0, 1, 2]])
        f2 = torch.where(one, q[:, [1, 2, 3]], q[:, [0, 2, 3]])
        faces = torch.stack([f1, f2], 1).reshape(-1, 3)
    return verts, faces, {"quads": q, "margin": (m1 - m2).abs()}


def max_cos(a, b, c):
    """Largest corner cosine of triangles (a, b, c), edge vectors normalised as F.normalize does."""
    def cos(o, u, v):
        return (F.normalize(u - o, dim=-1, eps=1e-12) * F.normalize(v - o, dim=-1, eps=1e-12)).sum(-1)
    return torch.maximum(cos(a, b, c), torch.maximum(cos(b, c, a), cos(c, a, b)))


# ---- seeded inputs ---------------------------------------------------------------------------------------------
def triposg_field(n, seed=0, device="cpu", nan_band=False, blobs=6, noise=0.02):
    """TripoSG-like input of DiffDMC on an n^3 grid over [-1, 1]^3: sdf = -logits / (n - 1), the logits being 50 x the
    negated distance to a union of spheres plus uniform noise of +-noise (positive inside).  With nan_band, points
    away from the surface are NaN as a hierarchical decoder leaves them: an 8^3 block is evaluated iff it or a
    neighbouring block holds a point within 2 cells of the surface.  fp32 [n, n, n] on `device`."""
    rng = np.random.default_rng(seed)
    centres = torch.as_tensor(rng.uniform(-0.45, 0.45, (blobs, 3)), dtype=torch.float32, device=device)
    radii = torch.as_tensor(rng.uniform(0.15, 0.35, blobs), dtype=torch.float32, device=device)
    g = torch.Generator(device=device).manual_seed(seed)
    lin = torch.linspace(-1, 1, n, device=device)
    yy, zz = torch.meshgrid(lin, lin, indexing="ij")
    dist = torch.empty((n, n, n), dtype=torch.float32, device=device)
    for x in range(n):
        p = torch.stack([lin[x].expand(n, n), yy, zz], dim=-1)
        dist[x] = (torch.linalg.vector_norm(p[:, :, None] - centres, dim=-1) - radii).amin(-1)
    logits = -dist * 50 + (torch.rand((n, n, n), generator=g, device=device) * 2 - 1) * noise
    sdf = -logits / (n - 1)
    if nan_band:
        near = (dist.abs() < 2 * 2.0 / (n - 1)).float()[None, None]
        coarse = F.max_pool3d(near, 8, 8, ceil_mode=True)
        coarse = F.max_pool3d(coarse, 3, 1, 1)[0, 0]
        keep = coarse.repeat_interleave(8, 0).repeat_interleave(8, 1).repeat_interleave(8, 2)[:n, :n, :n] > 0
        sdf = torch.where(keep, sdf, torch.full_like(sdf, float("nan")))
    return sdf
