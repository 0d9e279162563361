"""Marching-cubes oracle: vectorised numpy over the committed case table (comfyui-3d-pack_b200/csrc/mc_table.cuh).

It reproduces the GPU path bit for bit: the same vertex order (owner grid point, axis), the same triangle order (cell,
table order) and the same fp32 expressions, t = (iso - v[a]) / (v[b] - v[a]) and coord = float(index) + t.  It works
in slabs along the first (slowest) axis, so a 256^3 or 512^3 volume fits in memory and the slab outputs concatenate
in the global order.  Also: mesh-topology checks and the seeded density used by the tests and scripts/bench_mc.py."""
import os
import re

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLE = os.path.join(ROOT, "comfyui-3d-pack_b200", "csrc", "mc_table.cuh")
_TABLE = None


def load_table(path=TABLE):
    """(counts uint8[256], edges uint8[256, 3 * MC_MAX_TRIS]) parsed from the header the kernels compile."""
    src = open(path).read()
    max_tris = int(re.search(r"#define MC_MAX_TRIS (\d+)", src).group(1))
    body = lambda name: src.split(name, 1)[1].split("= {", 1)[1].split("};", 1)[0]
    counts = np.array([int(x) for x in re.findall(r"\d+", body("mc_tri_count"))], dtype=np.uint8)
    edges = np.array([int(x) for x in re.findall(r"\d+", body("mc_tri_edges"))], dtype=np.uint8)
    assert counts.shape == (256,) and edges.size == 256 * 3 * max_tris
    return counts, edges.reshape(256, 3 * max_tris)


def _table():
    global _TABLE
    if _TABLE is None:
        _TABLE = load_table()
    return _TABLE


def edge_owner(e):
    """(axis, owner corner offset (ox, oy, oz)) of cell edge e = 4 * a + k; works on arrays."""
    e = np.asarray(e, dtype=np.int64)
    a, lo, hi = e >> 2, e & 1, (e >> 1) & 1
    ox = np.where(a == 0, 0, lo)
    oy = np.where(a == 0, lo, np.where(a == 1, 0, hi))
    oz = np.where(a == 2, 0, hi)
    return a, ox, oy, oz


def marching_cubes(volume, iso, slab=16):
    """(verts float32 [V,3], tris int32 [F,3]) with the GPU path's semantics (gs_b200.isosurface.marching_cubes)."""
    vol = np.ascontiguousarray(volume, dtype=np.float32)
    if vol.ndim != 3:
        raise ValueError("volume must be 3-D")
    iso = np.float32(iso)
    X, Y, Z = vol.shape
    if min(X, Y, Z) < 2:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32)
    if not np.isfinite(vol).all():
        raise ValueError("the volume holds a non-finite sample")
    counts, edges = _table()
    verts_out, tris_out, vstart = [], [], 0
    for x0 in range(0, X, slab):
        x1 = min(x0 + slab, X)           # owner rows whose vertices this slab emits
        xe = min(x1 + 1, X)              # owner rows its cells reference
        v = vol[x0:min(xe + 1, X)]
        up = v > iso
        nr = xe - x0
        cross = np.zeros((nr, Y, Z, 3), dtype=bool)
        nx = min(nr, X - 1 - x0)
        cross[:nx, :, :, 0] = up[:nx] != up[1:nx + 1]
        cross[:, :-1, :, 1] = up[:nr, :-1] != up[:nr, 1:]
        cross[:, :, :-1, 2] = up[:nr, :, :-1] != up[:nr, :, 1:]
        vid = (np.cumsum(cross.reshape(-1), dtype=np.int64) - 1 + vstart).reshape(cross.shape)

        px, py, pz, ax = np.nonzero(cross[:x1 - x0])
        coords = np.stack([px + x0, py, pz], axis=1).astype(np.float32)
        va = v[px, py, pz]
        vb = v[px + (ax == 0), py + (ax == 1), pz + (ax == 2)]
        t = (iso - va) / (vb - va)
        rows = np.arange(len(px))
        coords[rows, ax] = coords[rows, ax] + t
        verts_out.append(coords)
        vstart += len(px)

        nc = min(x1, X - 1) - x0         # cell rows (min corners) of this slab
        if nc <= 0:
            continue
        cube = np.zeros((nc, Y - 1, Z - 1), dtype=np.int64)
        for q in range(8):
            dx, dy, dz = q & 1, (q >> 1) & 1, q >> 2
            cube |= up[dx:dx + nc, dy:dy + Y - 1, dz:dz + Z - 1].astype(np.int64) << q
        nt = counts[cube].astype(np.int64)
        cx, cy, cz = np.nonzero(nt)
        n = nt[cx, cy, cz]
        cell = np.repeat(np.arange(len(cx)), n)
        k = np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)
        e = edges[cube[cx, cy, cz][cell][:, None], 3 * k[:, None] + np.arange(3)]
        a, ox, oy, oz = edge_owner(e)
        tris_out.append(vid[cx[cell][:, None] + ox, cy[cell][:, None] + oy, cz[cell][:, None] + oz, a].astype(np.int32))
    verts = np.concatenate(verts_out) if verts_out else np.zeros((0, 3), np.float32)
    tris = np.concatenate(tris_out) if tris_out else np.zeros((0, 3), np.int32)
    return verts, tris.reshape(-1, 3)


# ---- mesh checks -----------------------------------------------------------------------------------------------
def directed_edges(tris):
    t = np.asarray(tris, dtype=np.int64)
    return np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])


def _edge_keys(tris):
    d = directed_edges(tris)
    m = int(d.max()) + 1 if len(d) else 1
    return d[:, 0] * m + d[:, 1], d[:, 1] * m + d[:, 0]


def is_closed_oriented(tris):
    """Closed and consistently oriented: every directed edge occurs as often as its reverse."""
    key, rev = _edge_keys(tris)
    k, n = np.unique(key, return_counts=True)
    r, nr = np.unique(rev, return_counts=True)
    return bool(np.array_equal(k, r) and np.array_equal(n, nr))


def is_oriented_manifold(tris):
    """Every directed edge occurs exactly once and its reverse occurs too: a closed, oriented 2-manifold."""
    key, rev = _edge_keys(tris)
    uk = np.unique(key)
    return len(uk) == len(key) and bool(np.isin(rev, uk).all())


def euler_characteristic(n_verts, tris):
    e = np.sort(directed_edges(tris), axis=1)
    return int(n_verts) - len(np.unique(e, axis=0)) + len(tris)


def triangle_normals(verts, tris):
    v = np.asarray(verts, dtype=np.float64)
    t = np.asarray(tris, dtype=np.int64)
    return np.cross(v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]])


def signed_volume(verts, tris):
    v = np.asarray(verts, dtype=np.float64)
    t = np.asarray(tris, dtype=np.int64)
    return float(np.einsum("ij,ij->i", v[t[:, 0]], np.cross(v[t[:, 1]], v[t[:, 2]])).sum() / 6.0)


# ---- seeded inputs -----------------------------------------------------------------------------------------------
def blob_density(n, seed=0, device="cpu", blobs=12, noise=1.0):
    """Instant-NGP-like density on an n^3 grid over [-1, 1]^3 (torch.linspace, as mesh_utils.py:495-497 samples it):
    a sum of anisotropic, rotated Gaussian blobs with peaks 20..60, plus uniform noise in [-noise, noise).  Meant for
    the threshold 10 of marching_cubes_density_to_mesh.  fp32 [n, n, n] on `device`."""
    rng = np.random.default_rng(seed)
    centres = rng.uniform(-0.5, 0.5, (blobs, 3))
    scales = rng.uniform(0.06, 0.3, (blobs, 3))
    peaks = rng.uniform(20.0, 60.0, blobs)
    rots = np.linalg.qr(rng.normal(size=(blobs, 3, 3)))[0]
    g = torch.Generator(device=device).manual_seed(seed)
    lin = torch.linspace(-1, 1, n, device=device)
    out = torch.empty((n, n, n), dtype=torch.float32, device=device)
    yy, zz = torch.meshgrid(lin, lin, indexing="ij")
    for x in range(n):
        p = torch.stack([lin[x].expand(n, n), yy, zz], dim=-1)          # [n, n, 3]
        acc = torch.zeros((n, n), dtype=torch.float32, device=device)
        for b in range(blobs):
            r = torch.as_tensor(rots[b], dtype=torch.float32, device=device)
            q = (p - torch.as_tensor(centres[b], dtype=torch.float32, device=device)) @ r
            q = q / torch.as_tensor(scales[b], dtype=torch.float32, device=device)
            acc += float(peaks[b]) * torch.exp(-0.5 * (q * q).sum(-1))
        acc += (torch.rand((n, n), generator=g, device=device) * 2 - 1) * noise
        out[x] = acc
    return out
