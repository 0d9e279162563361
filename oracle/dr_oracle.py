"""CPU oracle for the mesh path (nvdiffrast surface) — TEST INFRASTRUCTURE ONLY.

    PARITY UNPINNED: nvdiffrast 0.3.3 (my-reqs.txt:74, dependencies.txt:3) is an un-vendored third-party
    package, absent from the reference source tree and not installable offline; the reference ships no tests or golden
    images for it (SURVEY.md §4, §8c).

Restates the published algorithms (Laine et al. 2020, "Modular Primitives for High-Performance
Differentiable Rendering"; buffer semantics per SURVEY.md App. A.2) for the four ops the reference calls:

  rasterize   diff_mesh_renderer.py:97, flexicubes_renderer.py:49, mesh_utils.py:531
  interpolate diff_mesh_renderer.py:104,110,131, FlexiCubes/util.py:90-93, mesh_utils.py:534
  texture     diff_mesh_renderer.py:105 (filter_mode='linear')
  antialias   diff_mesh_renderer.py:101,138, flexicubes_renderer.py:55

Conventions: pos is clip space [B,V,4]; pixel centres at +0.5; row 0 is the BOTTOM row (y up);
rast = (u, v, z/w, triangle_id+1) with u,v the perspective-correct barycentrics of vertices 0 and 1;
rast_db = (du/dX, du/dY, dv/dX, dv/dY) in pixel units; empty pixels are all zero.

Arithmetic contract (what makes triangle ids bit-exact against the CUDA path): coverage and depth are
decided with 2-D homogeneous edge functions (no clipping needed) in IEEE fp32, no FMA, operation order as
written in `_tri_setup` / `_edge_eval`; ties on shared edges are broken by a top-left rule on the edge
coefficients; the depth test keeps the smallest z/w, ties -> smallest triangle index.
Gradients: to pos through u,v only (z/w, id and rast_db are treated as constants, which is all the
reference's call sites need — `texture(filter_mode='linear')` ignores uv_da), to attr, tex, uv, color.
"""
from __future__ import annotations

import numpy as np
import torch


# --------------------------------------------------------------------------------------------------
# rasterize
# --------------------------------------------------------------------------------------------------
def _tri_setup(p0, p1, p2):
    """Rows of adj(M), M = [[x0,x1,x2],[y0,y1,y2],[w0,w1,w2]]: e_i(X,Y) = a_i X + b_i Y + c_i."""
    x0, y0, w0 = p0[..., 0], p0[..., 1], p0[..., 3]
    x1, y1, w1 = p1[..., 0], p1[..., 1], p1[..., 3]
    x2, y2, w2 = p2[..., 0], p2[..., 1], p2[..., 3]
    a0 = y1 * w2 - y2 * w1; b0 = x2 * w1 - x1 * w2; c0 = x1 * y2 - x2 * y1
    a1 = y2 * w0 - y0 * w2; b1 = x0 * w2 - x2 * w0; c1 = x2 * y0 - x0 * y2
    a2 = y0 * w1 - y1 * w0; b2 = x1 * w0 - x0 * w1; c2 = x0 * y1 - x1 * y0
    det = x0 * a0 + x1 * a1 + x2 * a2
    return (a0, b0, c0), (a1, b1, c1), (a2, b2, c2), det


def _pixel_ndc(h, w, dtype):
    xs = (torch.arange(w, dtype=dtype) + 0.5) * torch.tensor(2.0 / w, dtype=dtype) - 1.0
    ys = (torch.arange(h, dtype=dtype) + 0.5) * torch.tensor(2.0 / h, dtype=dtype) - 1.0
    return xs, ys


def _ordered_bits(zw: torch.Tensor) -> torch.Tensor:
    """float32 -> int64 key preserving order (standard sign-flip trick)."""
    b = zw.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    neg = (b >> 31) & 1
    k = torch.where(neg == 1, (~b) & 0xFFFFFFFF, b | 0x80000000)     # unsigned-ordered 32-bit key
    return k ^ 0x80000000          # top bit flipped so that (key << 32) orders correctly as a SIGNED int64


def rasterize_ids(pos: torch.Tensor, tri: torch.Tensor, resolution, chunk=512):
    """Integer part: winning triangle id+1 per pixel [B,h,w] (int64) — the bit-exact contract."""
    h, w = resolution
    B = pos.shape[0]
    pos = pos.detach().to(torch.float32)
    xs, ys = _pixel_ndc(h, w, torch.float32)
    X = xs[None, None, :]; Y = ys[None, :, None]
    out = torch.zeros(B, h, w, dtype=torch.int64)
    tri = tri.to(torch.int64)
    F = tri.shape[0]
    BIG = torch.tensor(0x7FFFFFFFFFFFFFFF, dtype=torch.int64)
    for b in range(B):
        best = torch.full((h, w), int(BIG), dtype=torch.int64)
        for s in range(0, F, chunk):
            t = tri[s:s + chunk]
            p0, p1, p2 = pos[b, t[:, 0]], pos[b, t[:, 1]], pos[b, t[:, 2]]
            (a0, b0, c0), (a1, b1, c1), (a2, b2, c2), det = _tri_setup(p0, p1, p2)
            sgn = torch.where(det < 0, -torch.ones_like(det), torch.ones_like(det))
            ok = det != 0

            def ev(a, bb, c):
                return (a[:, None, None] * X + bb[:, None, None] * Y) + c[:, None, None]

            def inside(e, a, bb):
                es = e * sgn[:, None, None]
                a_s = (a * sgn)[:, None, None]; b_s = (bb * sgn)[:, None, None]
                return (es > 0) | ((es == 0) & ((a_s > 0) | ((a_s == 0) & (b_s > 0))))
            e0, e1, e2 = ev(a0, b0, c0), ev(a1, b1, c1), ev(a2, b2, c2)
            cov = inside(e0, a0, b0) & inside(e1, a1, b1) & inside(e2, a2, b2) & ok[:, None, None]
            z0, z1, z2 = p0[:, 2], p1[:, 2], p2[:, 2]
            dets = torch.where(ok, det, torch.ones_like(det))
            zw = ((z0[:, None, None] * e0 + z1[:, None, None] * e1) + z2[:, None, None] * e2) / dets[:, None, None]
            cov = cov & (zw >= -1.0) & (zw <= 1.0)
            ids = torch.arange(s, s + t.shape[0], dtype=torch.int64)[:, None, None]
            key = (_ordered_bits(zw) << 32) | ids
            key = torch.where(cov, key, BIG)
            best = torch.minimum(best, key.min(dim=0).values)
        hit = best != BIG
        out[b] = torch.where(hit, (best & 0xFFFFFFFF) + 1, torch.zeros_like(best))
    return out


def rasterize(pos: torch.Tensor, tri: torch.Tensor, resolution):
    """(rast[B,h,w,4], rast_db[B,h,w,4]); differentiable wrt pos through u,v."""
    h, w = resolution
    B = pos.shape[0]
    dt = pos.dtype
    ids = rasterize_ids(pos, tri, resolution)                        # [B,h,w]
    xs, ys = _pixel_ndc(h, w, dt)
    X = xs[None, None, :].expand(B, h, w); Y = ys[None, :, None].expand(B, h, w)
    hit = ids > 0
    t = tri.to(torch.int64)[(ids - 1).clamp_min(0)]                  # [B,h,w,3]
    bidx = torch.arange(B)[:, None, None].expand(B, h, w)
    p0, p1, p2 = pos[bidx, t[..., 0]], pos[bidx, t[..., 1]], pos[bidx, t[..., 2]]
    (a0, b0, c0), (a1, b1, c1), (a2, b2, c2), det = _tri_setup(p0, p1, p2)
    e0 = (a0 * X + b0 * Y) + c0; e1 = (a1 * X + b1 * Y) + c1; e2 = (a2 * X + b2 * Y) + c2
    S = e0 + e1 + e2
    S = torch.where(hit, S, torch.ones_like(S))
    dets = torch.where(hit, det, torch.ones_like(det))
    u = e0 / S; v = e1 / S
    zw = (((p0[..., 2] * e0 + p1[..., 2] * e1) + p2[..., 2] * e2) / dets).detach()
    sa, sb = a0 + a1 + a2, b0 + b1 + b2
    sx, sy = 2.0 / w, 2.0 / h
    dudx = ((a0 * S - e0 * sa) / (S * S) * sx).detach(); dudy = ((b0 * S - e0 * sb) / (S * S) * sy).detach()
    dvdx = ((a1 * S - e1 * sa) / (S * S) * sx).detach(); dvdy = ((b1 * S - e1 * sb) / (S * S) * sy).detach()
    z = torch.zeros_like(u)
    rast = torch.stack([torch.where(hit, u, z), torch.where(hit, v, z), torch.where(hit, zw, z), ids.to(dt)], dim=-1)
    db = torch.stack([torch.where(hit, dudx, z), torch.where(hit, dudy, z), torch.where(hit, dvdx, z),
                      torch.where(hit, dvdy, z)], dim=-1)
    return rast, db


# --------------------------------------------------------------------------------------------------
# interpolate
# --------------------------------------------------------------------------------------------------
def interpolate(attr: torch.Tensor, rast: torch.Tensor, tri: torch.Tensor, rast_db=None, diff_attrs=None):
    """out[B,h,w,A] = u a0 + v a1 + (1-u-v) a2; out_da[B,h,w,2*nd] = (da/dX, da/dY) per differentiated attribute."""
    B, h, w, _ = rast.shape
    ids = rast[..., 3].detach().to(torch.int64)
    hit = ids > 0
    t = tri.to(torch.int64)[(ids - 1).clamp_min(0)]
    ab = attr if attr.shape[0] == B else attr.expand(B, -1, -1)
    bidx = torch.arange(B)[:, None, None].expand(B, h, w)
    a0, a1, a2 = ab[bidx, t[..., 0]], ab[bidx, t[..., 1]], ab[bidx, t[..., 2]]
    u, v = rast[..., 0:1], rast[..., 1:2]
    out = u * a0 + v * a1 + (1.0 - u - v) * a2
    out = torch.where(hit[..., None], out, torch.zeros_like(out))
    if rast_db is None or diff_attrs is None:
        return out, None
    A = attr.shape[-1]
    sel = list(range(A)) if diff_attrs == "all" else list(diff_attrs)
    d0 = (a0 - a2)[..., sel]; d1 = (a1 - a2)[..., sel]
    dax = rast_db[..., 0:1] * d0 + rast_db[..., 2:3] * d1
    day = rast_db[..., 1:2] * d0 + rast_db[..., 3:4] * d1
    da = torch.stack([dax, day], dim=-1).reshape(B, h, w, 2 * len(sel))
    da = torch.where(hit[..., None], da, torch.zeros_like(da))
    return out, da


# --------------------------------------------------------------------------------------------------
# texture (filter_mode='linear', boundary_mode='wrap')
# --------------------------------------------------------------------------------------------------
def mip_pyramid(tex: torch.Tensor, max_mip_level=None):
    """[tex, 2x2 box-filtered halves ...]: levels are added while both sides are even (down to 1 texel for power-of-two
    textures), at most max_mip_level of them."""
    levels = [tex]
    while levels[-1].shape[1] % 2 == 0 and levels[-1].shape[2] % 2 == 0 and (max_mip_level is None or len(levels) <= max_mip_level):
        t = levels[-1]
        levels.append(0.25 * (t[:, 0::2, 0::2] + t[:, 1::2, 0::2] + t[:, 0::2, 1::2] + t[:, 1::2, 1::2]))
    return levels


def mip_level(uv_da: torch.Tensor, Ht: int, Wt: int, n_levels: int, mip_level_bias=None):
    """Level of detail from the screen-space uv derivatives (du/dX, du/dY, dv/dX, dv/dY): half the log2 of the squared
    major axis of the pixel footprint in texel units (nvdiffrast calculateMipLevel), clamped to the pyramid."""
    dsdx, dsdy, dtdx, dtdy = uv_da[..., 0] * Wt, uv_da[..., 1] * Wt, uv_da[..., 2] * Ht, uv_da[..., 3] * Ht
    A = dsdx * dsdx + dtdx * dtdx
    Bq = dsdy * dsdy + dtdy * dtdy
    Cq = dsdx * dsdy + dtdx * dtdy
    major2 = 0.5 * (A + Bq) + torch.sqrt(0.25 * (A - Bq) * (A - Bq) + Cq * Cq)
    level = 0.5 * torch.log2(torch.clamp_min(major2, 1e-30))
    if mip_level_bias is not None:
        level = level + mip_level_bias
    return torch.clamp(level, 0.0, float(n_levels - 1))


def texture(tex: torch.Tensor, uv: torch.Tensor, filter_mode="linear", boundary_mode="wrap", uv_da=None, mip_level_bias=None,
            max_mip_level=None):
    """Bilinear lookup: texel (i,j) centre at ((i+0.5)/W, (j+0.5)/H), row 0 at v=0; wrap (or clamp) addressing.
    'linear-mipmap-linear' (what filter_mode='auto' means when uv_da is given, LGM nerf_marching_cubes_converter.py:230):
    bilinear in the two pyramid levels around `mip_level`, blended linearly."""
    if filter_mode == "linear-mipmap-linear":
        levels = mip_pyramid(tex, max_mip_level)
        lod = mip_level(uv_da, tex.shape[1], tex.shape[2], len(levels), mip_level_bias)
        out = 0
        for l, t in enumerate(levels):
            w = torch.clamp(1.0 - (lod - float(l)).abs(), min=0.0)              # tent weight = the two-level lerp
            out = out + w[..., None] * texture(t, uv, "linear", boundary_mode)
        return out
    assert filter_mode == "linear"
    T, Ht, Wt, C = tex.shape
    B = uv.shape[0]
    x = uv[..., 0] * Wt - 0.5
    y = uv[..., 1] * Ht - 0.5
    x0 = torch.floor(x.detach()); y0 = torch.floor(y.detach())
    fx = x - x0; fy = y - y0
    x0 = x0.to(torch.int64); y0 = y0.to(torch.int64)
    if boundary_mode == "wrap":
        xi0, xi1 = x0 % Wt, (x0 + 1) % Wt
        yi0, yi1 = y0 % Ht, (y0 + 1) % Ht
    else:
        xi0, xi1 = x0.clamp(0, Wt - 1), (x0 + 1).clamp(0, Wt - 1)
        yi0, yi1 = y0.clamp(0, Ht - 1), (y0 + 1).clamp(0, Ht - 1)
    tb = torch.arange(B)[:, None, None] if T == B and T > 1 else torch.zeros(B, 1, 1, dtype=torch.int64)
    tb = tb.expand_as(x0)
    t00, t10 = tex[tb, yi0, xi0], tex[tb, yi0, xi1]
    t01, t11 = tex[tb, yi1, xi0], tex[tb, yi1, xi1]
    fx = fx[..., None]; fy = fy[..., None]
    return (t00 * (1 - fx) + t10 * fx) * (1 - fy) + (t01 * (1 - fx) + t11 * fx) * fy


# --------------------------------------------------------------------------------------------------
# antialias
# --------------------------------------------------------------------------------------------------
def edge_opposites(tri: torch.Tensor) -> torch.Tensor:
    """[F,3] int64: for edge e of triangle f (edge e is opposite vertex e, i.e. joins vertices e+1, e+2) the
    opposite vertex of the other triangle sharing that undirected edge, -1 if none.  With more than two
    triangles on an edge the partner is the next one in (edge key, triangle index, edge index) order."""
    t = tri.to(torch.int64).numpy()
    F = t.shape[0]
    va = t[:, [1, 2, 0]].reshape(-1); vb = t[:, [2, 0, 1]].reshape(-1); vc = t.reshape(-1)
    lo = np.minimum(va, vb); hi = np.maximum(va, vb)
    key = lo * (int(t.max()) + 2 if F else 1) + hi
    order = np.argsort(key, kind="stable")
    out = np.full(3 * F, -1, dtype=np.int64)
    ks = key[order]
    same_next = np.concatenate([ks[1:] == ks[:-1], [False]])
    same_prev = np.concatenate([[False], ks[1:] == ks[:-1]])
    nxt = np.roll(order, -1); prv = np.roll(order, 1)
    # first of a run pairs with the next entry; others pair with the previous one
    partner = np.where(same_prev, prv, np.where(same_next, nxt, -1))
    out[order] = np.where(partner >= 0, vc[np.maximum(partner, 0)], -1)
    return torch.from_numpy(out.reshape(F, 3))


def antialias(color: torch.Tensor, rast: torch.Tensor, pos: torch.Tensor, tri: torch.Tensor):
    """Silhouette antialiasing by analytic coverage between adjacent pixel centres.

    For every horizontally / vertically adjacent pixel pair with different triangle ids: take the nearer
    surface's triangle (background counts as far), find its silhouette edge (no neighbour across it, or the
    neighbour folds back onto the same screen side) that crosses the segment between the two pixel centres at
    parameter t in [0,1] measured from the foreground pixel A towards B; if t > 0.5 pixel B receives
    (t-0.5) of A's colour, else pixel A receives (0.5-t) of B's colour.  Differentiable wrt color and pos.
    """
    B, h, w, C = color.shape
    dt = color.dtype
    ids = rast[..., 3].detach().to(torch.int64)
    zw = rast[..., 2].detach()
    opp = edge_opposites(tri)
    tri64 = tri.to(torch.int64)
    out = color.clone()
    sxy = torch.tensor([w * 0.5, h * 0.5], dtype=dt)
    for d in (0, 1):
        if d == 0:
            id0, id1 = ids[:, :, :-1], ids[:, :, 1:]; z0, z1 = zw[:, :, :-1], zw[:, :, 1:]
        else:
            id0, id1 = ids[:, :-1, :], ids[:, 1:, :]; z0, z1 = zw[:, :-1, :], zw[:, 1:, :]
        pair = id0 != id1
        bb, yy, xx = torch.nonzero(pair, as_tuple=True)
        if bb.numel() == 0:
            continue
        i0, i1 = id0[bb, yy, xx], id1[bb, yy, xx]
        zz0, zz1 = z0[bb, yy, xx], z1[bb, yy, xx]
        use0 = (i1 == 0) | ((i0 > 0) & (zz0 < zz1))          # foreground = pixel 0's triangle
        tsel = torch.where(use0, i0, i1) - 1
        ax = torch.where(use0, xx, xx + (1 if d == 0 else 0)); ay = torch.where(use0, yy, yy + (1 if d == 1 else 0))
        bx = torch.where(use0, xx + (1 if d == 0 else 0), xx); by = torch.where(use0, yy + (1 if d == 1 else 0), yy)
        ca = torch.stack([ax.to(dt) + 0.5, ay.to(dt) + 0.5], dim=-1)          # pixel-space centres
        cb = torch.stack([bx.to(dt) + 0.5, by.to(dt) + 0.5], dim=-1)
        tv = tri64[tsel]                                                       # [K,3]
        P = pos[bb[:, None], tv]                                               # [K,3,4]
        wpos = (P[..., 3] > 0).all(dim=1)
        Wc = torch.where(P[..., 3:4] > 0, P[..., 3:4], torch.ones_like(P[..., 3:4]))
        S = (P[..., :2] / Wc + 1.0) * sxy                                      # screen px, [K,3,2]
        best_t = torch.full((bb.numel(),), 2.0, dtype=dt)
        found = torch.zeros(bb.numel(), dtype=torch.bool)
        for e in range(3):
            va, vb, vc = (e + 1) % 3, (e + 2) % 3, e
            Pa, Pb, Pc = S[:, va], S[:, vb], S[:, vc]
            op = opp[tsel, e]
            has = op >= 0
            Po4 = pos[bb, op.clamp_min(0)]
            okw = Po4[:, 3] > 0
            Po = (Po4[:, :2] / torch.where(okw[:, None], Po4[:, 3:4], torch.ones_like(Po4[:, 3:4])) + 1.0) * sxy
            ed = Pb - Pa
            side_c = ed[:, 0] * (Pc[:, 1] - Pa[:, 1]) - ed[:, 1] * (Pc[:, 0] - Pa[:, 0])
            side_o = ed[:, 0] * (Po[:, 1] - Pa[:, 1]) - ed[:, 1] * (Po[:, 0] - Pa[:, 0])
            sil = (~has) | (has & okw & ((side_c.detach() * side_o.detach()) > 0))
            # crossing of the edge with the axis-aligned segment A->B
            ax_ = d  # axis along which A,B differ: 0 -> x, 1 -> y ; the other coordinate is fixed
            fix = 1 - ax_
            fa = Pa[:, fix] - ca[:, fix]; fb = Pb[:, fix] - ca[:, fix]
            spans = ((fa.detach() <= 0) & (fb.detach() > 0)) | ((fb.detach() <= 0) & (fa.detach() > 0))
            denom = torch.where(spans, fb - fa, torch.ones_like(fa))
            s_par = -fa / denom
            cross = Pa[:, ax_] + s_par * (Pb[:, ax_] - Pa[:, ax_])
            t = (cross - ca[:, ax_]) / (cb[:, ax_] - ca[:, ax_])
            ok = sil & spans & wpos & (t.detach() >= 0) & (t.detach() <= 1) & ~found
            best_t = torch.where(ok, t, best_t)
            found = found | ok
        if not bool(found.any()):
            continue
        sel = torch.nonzero(found, as_tuple=True)[0]
        t = best_t[sel]
        bsel = bb[sel]
        A_y, A_x, B_y, B_x = ay[sel], ax[sel], by[sel], bx[sel]
        colA = color[bsel, A_y, A_x]; colB = color[bsel, B_y, B_x]
        to_b = (t.detach() > 0.5)
        wgt = torch.where(to_b, t - 0.5, 0.5 - t)[:, None]
        delta = torch.where(to_b[:, None], wgt * (colA - colB), wgt * (colB - colA))
        ty = torch.where(to_b, B_y, A_y); tx = torch.where(to_b, B_x, A_x)
        flat = out.reshape(B * h * w, C)
        lin = (bsel * h + ty) * w + tx
        out = flat.index_add(0, lin, delta).reshape(B, h, w, C)
    return out


# --------------------------------------------------------------------------------------------------
# synthetic meshes / cameras
# --------------------------------------------------------------------------------------------------
def icosphere(subdiv: int = 2, radius: float = 0.5):
    t = (1.0 + 5 ** 0.5) / 2.0
    v = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], dtype=np.float64)
    f = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
                  [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5],
                  [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]], dtype=np.int64)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    for _ in range(subdiv):
        cache = {}; vl = list(v); nf = []

        def mid(a, b):
            k = (min(a, b), max(a, b))
            if k not in cache:
                m = (vl[a] + vl[b]) / 2; m /= np.linalg.norm(m)
                cache[k] = len(vl); vl.append(m)
            return cache[k]
        for a, b, c in f:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        v = np.array(vl); f = np.array(nf, dtype=np.int64)
    v = (v * radius).astype(np.float32)
    uv = np.stack([np.arctan2(v[:, 0], v[:, 2]) / (2 * np.pi) + 0.5, np.arccos(np.clip(v[:, 1] / radius, -1, 1)) / np.pi],
                  axis=1).astype(np.float32)
    return torch.from_numpy(v), torch.from_numpy(f.astype(np.int32)), torch.from_numpy(uv)


def gl_perspective(fovy_deg, aspect, near=0.01, far=100.0):
    """OrbitCamera.perspective (shared_utils/camera_utils.py:128-145) incl. the -1/y flip."""
    y = np.tan(np.deg2rad(fovy_deg) / 2)
    return np.array([[1 / (y * aspect), 0, 0, 0], [0, -1 / y, 0, 0],
                     [0, 0, -(far + near) / (far - near), -(2 * far * near) / (far - near)], [0, 0, -1, 0]],
                    dtype=np.float32)


def clip_positions(v: torch.Tensor, pose: np.ndarray, proj: np.ndarray) -> torch.Tensor:
    """v_clip as DiffRastRenderer.render builds it (diff_mesh_renderer.py:94-95)."""
    pose = torch.from_numpy(pose.astype(np.float32)); proj = torch.from_numpy(proj.astype(np.float32))
    v_cam = torch.matmul(torch.nn.functional.pad(v, pad=(0, 1), mode="constant", value=1.0), torch.inverse(pose).T).float().unsqueeze(0)
    return v_cam @ proj.T
