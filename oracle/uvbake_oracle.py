"""numpy restatement of StableFast3D's UV texture baker (texture_baker.slang's bake_uv and interpolate, as the reference's
generated CUDA computes them for sm_90a; csrc/uv_bake.cu states the arithmetic), bit for bit.

fp32 +, -, * and / are numpy's float32 operations (IEEE, round to nearest).  fma32 is an exact fp32 fused multiply-add:
the product of two fp32 values is exact in float64, and the one sum that float64 could round twice is corrected with an
error-free two-sum.

Two modes of rasterize:
  * brute force: every texel of the region tests every face in index order, the reference's loop;
  * box-limited: every face tests only the texels of its candidate box, computed with the kernel's rule (face_boxes);
    faces the rule cannot bound test the whole region, and faces that can never hit are dropped.
They agree exactly when the rule is conservative, which tests/test_uvbake_cpu.py checks on adversarial sweeps.
"""
import numpy as np

f32 = np.float32
U = f32(2.0 ** -24)
KMAX = f32(16384.0)
TINY = f32(2.0 ** -60)
HUGE = f32(2.0 ** 60)
WARP_AREA, CTA_AREA = 256, 8192
DROP, BOX, WHOLE = 0, 1, 2


def fma32(a, b, c):
    """Correctly rounded fp32 fma(a, b, c), elementwise."""
    a, b, c = (np.asarray(x, dtype=f32) for x in (a, b, c))
    with np.errstate(all="ignore"):
        p = a.astype(np.float64) * b.astype(np.float64)        # exact
        cd = c.astype(np.float64)
        s = p + cd
        bp = s - cd                                             # two-sum: s + err == p + c exactly (finite s)
        err = (p - bp) + (cd - (s - bp))
        r = s.astype(f32)
        # s rounds to r.  Only when s lies exactly halfway between r and its neighbour nb can the rounding of s have
        # mattered: ties-to-even chose r, and the exact sum s + err is past the midpoint (nb is right) iff err points
        # away from r; err == 0 is a true tie, which fma also breaks to even.
        d = s - r.astype(np.float64)
        nb = np.nextafter(r, np.where(d > 0, f32(np.inf), f32(-np.inf))).astype(f32)
        mid = np.isfinite(s) & (d != 0) & (s == (r.astype(np.float64) + nb.astype(np.float64)) * 0.5)
        r = np.where(mid & (err != 0) & (np.sign(err) == np.sign(d)), nb, r)
    return r


def dot2(sx, sy, tx, ty):
    return fma32(sy, ty, fma32(sx, tx, f32(0.0)))


def texel_xy(res, rows, cols):
    """x for columns [0, cols) and y for rows [0, rows), as the reference samples them."""
    with np.errstate(all="ignore"):
        x = np.clip(np.arange(cols, dtype=f32) / f32(res), f32(0), f32(1)).astype(f32)
        y = (f32(1) - np.clip(np.arange(rows, dtype=f32) / f32(res), f32(0), f32(1))).astype(f32)
    return x, y


def setup(uv, faces):
    """Per face: (ax, ay, e1x, e1y, e2x, e2y, d00, d01, d11, denom) and a validity mask (vertex ids in range)."""
    uv = np.asarray(uv, dtype=f32).reshape(-1, 2)
    faces = np.asarray(faces).reshape(-1, 3).astype(np.int64)
    NV = uv.shape[0]
    ok = ((faces >= 0) & (faces < NV)).all(1)
    idx = np.where(ok[:, None], faces, 0)
    if NV == 0:
        uv = np.zeros((1, 2), f32)
    a, b, c = uv[idx[:, 0]], uv[idx[:, 1]], uv[idx[:, 2]]
    with np.errstate(all="ignore"):
        e1x, e1y = b[:, 0] - a[:, 0], b[:, 1] - a[:, 1]
        e2x, e2y = c[:, 0] - a[:, 0], c[:, 1] - a[:, 1]
        d00 = dot2(e1x, e1y, e1x, e1y)
        d01 = dot2(e1x, e1y, e2x, e2y)
        d11 = dot2(e2x, e2y, e2x, e2y)
        denom = fma32(d00, d11, -(d01 * d01))
    return dict(ax=a[:, 0], ay=a[:, 1], bx=b[:, 0], by=b[:, 1], cx=c[:, 0], cy=c[:, 1], e1x=e1x, e1y=e1y, e2x=e2x,
                e2y=e2y, d00=d00, d01=d01, d11=d11, denom=denom), ok


def bary(S, i, x, y):
    """(hit, u, v, w) of faces S[.][i] at points (x, y) (broadcast)."""
    with np.errstate(all="ignore"):
        qx, qy = (x - S["ax"][i]).astype(f32), (y - S["ay"][i]).astype(f32)
        d20 = dot2(qx, qy, S["e1x"][i], S["e1y"][i])
        d21 = dot2(qx, qy, S["e2x"][i], S["e2y"][i])
        d01, d00, d11, den = S["d01"][i], S["d00"][i], S["d11"][i], S["denom"][i]
        v = (fma32(d11, d20, -(d01 * d21)) / den).astype(f32)
        w = (fma32(d00, d21, -(d01 * d20)) / den).astype(f32)
        u = ((f32(1) - v) - w).astype(f32)
        hit = (v >= 0) & (w >= 0) & ((v + w).astype(f32) <= 1)
    return hit, u, v, w


def face_boxes(S, ok, res, rows, cols):
    """The kernel's candidate rule: (kind, r0, r1, c0, c1) per face, kind DROP / BOX / WHOLE (csrc/uv_bake.cu)."""
    n = S["ax"].shape[0]
    r0, r1 = np.zeros(n, np.int64), np.full(n, rows - 1, np.int64)
    c0, c1 = np.zeros(n, np.int64), np.full(n, cols - 1, np.int64)
    kind = np.full(n, BOX, np.int64)
    with np.errstate(all="ignore"):
        fin = np.ones(n, bool)
        for k in ("ax", "ay", "bx", "by", "cx", "cy"):
            fin &= np.isfinite(S[k])
        den, d00, d11 = S["denom"], S["d00"], S["d11"]
        drop = ~ok | ~fin | ~(den != 0)
        whole = ~drop & ~((den > 0) & (d00 >= TINY) & (d11 >= TINY) & (d00 <= HUGE) & (d11 <= HUGE))
        K = (d00 * d11 / den).astype(f32)
        whole |= ~drop & ~whole & ~(K <= KMAX)
        ax, ay = S["ax"], S["ay"]
        rx = np.maximum(np.abs(ax), np.abs(f32(1) - ax))
        ry = np.maximum(np.abs(ay), np.abs(f32(1) - ay))
        R = np.sqrt((rx * rx + ry * ry).astype(f32)).astype(f32)
        c64 = f32(64) * U
        ev = (c64 * K * (f32(1) + R / np.sqrt(d00)) + TINY).astype(f32)
        ew = (c64 * K * (f32(1) + R / np.sqrt(d11)) + TINY).astype(f32)
        et = (f32(2) * (ev + ew) + f32(4) * U).astype(f32)
        mx = (et * (np.abs(S["e1x"]) + np.abs(S["e2x"])) * f32(1.01) + TINY).astype(f32)
        my = (et * (np.abs(S["e1y"]) + np.abs(S["e2y"])) * f32(1.01) + TINY).astype(f32)
        whole |= ~drop & ~whole & ~((mx < 2) & (my < 2))
        boxed = ~drop & ~whole
        xlo = np.maximum(np.minimum(ax, np.minimum(S["bx"], S["cx"])) - mx, f32(0)).astype(f32)
        xhi = np.minimum(np.maximum(ax, np.maximum(S["bx"], S["cx"])) + mx, f32(1)).astype(f32)
        ylo = np.maximum(np.minimum(ay, np.minimum(S["by"], S["cy"])) - my, f32(0)).astype(f32)
        yhi = np.minimum(np.maximum(ay, np.maximum(S["by"], S["cy"])) + my, f32(1)).astype(f32)
        drop |= boxed & ((xlo > xhi) | (ylo > yhi))
        boxed &= ~drop
        fr = f32(res)
        sel = boxed
        c0 = np.where(sel, np.maximum(c0, np.floor(np.where(sel, xlo, 0) * fr).astype(np.int64) - 2), c0)
        c1 = np.where(sel, np.minimum(c1, np.ceil(np.where(sel, xhi, 0) * fr).astype(np.int64) + 2), c1)
        r0 = np.where(sel, np.maximum(r0, np.floor((f32(1) - np.where(sel, yhi, 0)) * fr).astype(np.int64) - 2), r0)
        r1 = np.where(sel, np.minimum(r1, np.ceil((f32(1) - np.where(sel, ylo, 0)) * fr).astype(np.int64) + 2), r1)
        drop |= boxed & ((c0 > c1) | (r0 > r1))
    kind[whole] = WHOLE
    kind[drop] = DROP
    return kind, r0, r1, c0, c1


def queue_counts(uv, faces, res, rows=None, cols=None):
    """(thread, warp, cta, whole) face counts the kernel's queues get; whole-texture faces are in the CTA count too."""
    rows = res if rows is None else min(rows, res)
    cols = res if cols is None else min(cols, res)
    S, ok = setup(uv, faces)
    kind, r0, r1, c0, c1 = face_boxes(S, ok, res, rows, cols)
    area = (r1 - r0 + 1) * (c1 - c0 + 1)
    live = kind != DROP
    cta = live & ((kind == WHOLE) | (area > CTA_AREA))
    warp = live & ~cta & (area > WARP_AREA)
    return int((live & ~cta & ~warp).sum()), int(warp.sum()), int(cta.sum()), int((kind == WHOLE).sum())


def _resolve(S, winner, res, rows, cols, out):
    x, y = texel_xy(res, rows, cols)
    rr, cc = np.nonzero(winner >= 0)
    reg = np.zeros((rows, cols, 4), f32)
    reg[..., 3] = -1
    if rr.size:
        i = winner[rr, cc]
        _, u, v, w = bary(S, i, x[cc], y[rr])
        reg[rr, cc, 0], reg[rr, cc, 1], reg[rr, cc, 2] = u, v, w
        reg[rr, cc, 3] = i.astype(np.int32).astype(f32)
    out[:rows, :cols] = reg
    return out


def rasterize(uv, faces, res, rows=None, cols=None, out=None, mode="box", chunk=1 << 22):
    """out[res,res,4] fp32: (u, v, w, face) per texel of the region [0, rows) x [0, cols) (default: all), (0,0,0,-1)
    where no face hits; texels outside the region keep out's values (NaN when out is None)."""
    rows = res if rows is None else min(rows, res)
    cols = res if cols is None else min(cols, res)
    if out is None:
        out = np.full((res, res, 4), np.nan, f32)
    if rows <= 0 or cols <= 0:
        return out
    S, ok = setup(uv, faces)
    F = ok.shape[0]
    x, y = texel_xy(res, rows, cols)
    winner = np.full((rows, cols), -1, np.int64)
    if mode == "brute":
        live = np.nonzero(ok)[0]
        flat_y = np.repeat(y, cols)
        flat_x = np.tile(x, rows)
        best = np.full(rows * cols, F, np.int64)
        step = max(1, chunk // max(1, rows * cols))
        for s in range(0, live.size, step):
            fi = live[s:s + step]
            hit, _, _, _ = bary(S, fi[:, None], flat_x[None, :], flat_y[None, :])
            cand = np.where(hit, fi[:, None], F).min(0)
            best = np.minimum(best, cand)
        winner = np.where(best < F, best, -1).reshape(rows, cols)
    else:
        kind, r0, r1, c0, c1 = face_boxes(S, ok, res, rows, cols)
        best = np.full(rows * cols, F, np.int64)
        fi = np.nonzero(kind != DROP)[0]
        h = (r1 - r0 + 1)[fi]
        wdt = (c1 - c0 + 1)[fi]
        area = h * wdt
        start = 0
        while start < fi.size:      # batches of faces whose candidate pairs fit in `chunk`
            csum = np.cumsum(area[start:])
            stop = start + max(1, int(np.searchsorted(csum, chunk, side="right")))
            f_b, a_b, w_b = fi[start:stop], area[start:stop], wdt[start:stop]
            rep = np.repeat(np.arange(f_b.size), a_b)
            k = np.arange(rep.size) - np.repeat(np.cumsum(a_b) - a_b, a_b)
            row = r0[f_b][rep] + k // w_b[rep]
            col = c0[f_b][rep] + k % w_b[rep]
            face = f_b[rep]
            hit, _, _, _ = bary(S, face, x[col], y[row])
            np.minimum.at(best, (row * cols + col)[hit], face[hit])
            start = stop
        winner = np.where(best < F, best, -1).reshape(rows, cols)
    return _resolve(S, winner, res, rows, cols, out)


def interpolate(attr, rast, faces, rows=None, cols=None, out=None):
    """out[H,W,3] = fma(rz, a3, fma(rx, a1, ry * a2)) for face (int)rast.w over the region; 0 for a negative or
    out-of-range face or vertex id.  Texels outside the region keep out's values (0 when out is None)."""
    attr = np.asarray(attr, dtype=f32).reshape(-1, 3)
    rast = np.asarray(rast, dtype=f32)
    faces = np.asarray(faces).reshape(-1, 3).astype(np.int64)
    H, W = rast.shape[:2]
    rows = H if rows is None else min(rows, H)
    cols = W if cols is None else min(cols, W)
    if out is None:
        out = np.zeros((H, W, 3), f32)
    r = rast[:rows, :cols].reshape(-1, 4)
    with np.errstate(all="ignore"):
        wv = r[:, 3].astype(np.float64)
        i = np.where(np.isnan(wv), 0, np.trunc(np.clip(wv, -2.0 ** 31, 2.0 ** 31 - 1))).astype(np.int64)
    NF, NV = faces.shape[0], attr.shape[0]
    okf = (i >= 0) & (i < NF)
    tri = faces[np.where(okf, i, 0)] if NF else np.zeros((i.size, 3), np.int64)
    ok = okf & ((tri >= 0) & (tri < NV)).all(1)
    tri = np.where(ok[:, None], tri, 0)
    a = attr if NV else np.zeros((1, 3), f32)
    a1, a2, a3 = a[tri[:, 0]], a[tri[:, 1]], a[tri[:, 2]]
    with np.errstate(all="ignore"):
        res = fma32(r[:, 2:3], a3, fma32(r[:, 0:1], a1, (r[:, 1:2] * a2).astype(f32)))
    res = np.where(ok[:, None], res, f32(0)).astype(f32)
    out[:rows, :cols] = res.reshape(rows, cols, 3)
    return out


def soup(F, seed, kind="atlas"):
    """A seeded triangle soup laid out as SF3D's unwrap_uv leaves it (V = 3F, faces = arange(3F)): "atlas" tiles
    [0,1]^2 with jittered, mostly non-overlapping triangles of a few texels at 1024^2."""
    rng = np.random.default_rng(seed)
    n = int(np.ceil(np.sqrt(F / 2)))
    cell = 1.0 / n
    k = np.arange(F)
    cx, cy = (k // 2) % n, (k // 2) // n % n
    base = np.stack([cx * cell, cy * cell], 1)
    lo = np.array([[0, 0], [1, 0], [0, 1]], np.float64)
    hi = np.array([[1, 1], [0, 1], [1, 0]], np.float64)
    tri = np.where((k % 2 == 0)[:, None, None], lo[None], hi[None]) * cell * 0.94 + cell * 0.03
    tri = tri + base[:, None, :] + rng.normal(0, cell * 0.02, (F, 3, 2))
    uv = tri.reshape(-1, 2).astype(f32)
    faces = np.arange(3 * F, dtype=np.int32).reshape(-1, 3)
    return uv, faces


def _tris(rng, n, lo, hi, size):
    c = rng.uniform(lo, hi, (n, 1, 2))
    return c + rng.normal(0, 1, (n, 3, 2)) * np.asarray(size, np.float64).reshape(-1, 1, 1)


def _pack(tris):
    tris = np.asarray(tris, np.float64).reshape(-1, 3, 2)
    with np.errstate(all="ignore"):
        uv = tris.reshape(-1, 2).astype(f32)
    return uv, np.arange(uv.shape[0], dtype=np.int32).reshape(-1, 3)


def adversarial(seed=0):
    """{name: (uv, faces, res)}: soups at the edges of the candidate rule (slivers, collinear and duplicate vertices,
    computed denom < 0, faces outside [0,1] or covering the texture, overlaps, NaN / inf) and one per kernel queue."""
    rng = np.random.default_rng(seed)
    cases = {}
    # slivers: aspect ratios 10 .. 1e7 at every orientation, some with the sharp angle at the first vertex
    n = 240
    a = rng.uniform(0.05, 0.95, (n, 2))
    ang = rng.uniform(0, 2 * np.pi, n)
    L = rng.uniform(0.05, 0.9, n)
    wid = L / 10.0 ** rng.uniform(1, 7, n)
    d = np.stack([np.cos(ang), np.sin(ang)], 1)
    nrm = np.stack([-d[:, 1], d[:, 0]], 1)
    t = rng.uniform(0, 1, n)
    b = a + d * L[:, None]
    c = a + d * (L * t)[:, None] + nrm * wid[:, None]
    tris = np.stack([a, b, c], 1)
    roll = rng.integers(0, 3, n)
    tris = np.stack([np.roll(tris[i], roll[i], 0) for i in range(n)])
    cases["slivers"] = _pack(tris) + (64,)
    # collinear and duplicate vertices, exactly and to within rounding
    p = rng.uniform(0, 1, (n, 2))
    q = rng.uniform(0, 1, (n, 2))
    s = rng.uniform(-0.5, 1.5, n)
    coll = np.stack([p, q, p + (q - p) * s[:, None]], 1)
    coll[: n // 3, 2] = coll[: n // 3, 1]                            # duplicates
    coll[n // 3: n // 2, 1] = coll[n // 3: n // 2, 0]
    cases["collinear"] = _pack(coll) + (64,)
    # computed denom < 0: near-collinear triangles far from the origin, kept when the fp32 denom comes out negative
    keep = []
    while len(keep) < 120:
        m = 4000
        base = rng.uniform(-40, 40, (m, 1, 2))
        dd = rng.normal(0, 1, (m, 1, 2))
        tt = rng.uniform(-1, 1, (m, 3, 1))
        tri = base + dd * tt + rng.normal(0, 1e-6, (m, 3, 2))
        uv, fc = _pack(tri)
        S, _ = setup(uv, fc)
        keep += list(tri[S["denom"] < 0])
    far = np.array(keep[:60])                                        # as found, far outside the texture
    near = (far - far.mean((0, 1))) / 80.0 + 0.5                     # still near-collinear, across the texture
    cases["negative_denom"] = _pack(np.concatenate([far, near], 0)) + (64,)
    # outside [0,1], straddling it, covering the whole texture; overlapping faces of every size
    cases["outside"] = _pack(_tris(rng, 150, -3, 4, rng.uniform(0.01, 2, 150))) + (64,)
    big = np.array([[[-1, -1], [3, -1], [-1, 3]], [[-5, 0.5], [5, -9], [5, 9]], [[0, 0], [1, 0], [0, 1]],
                    [[1, 1], [0, 1], [1, 0]]], np.float64)
    cases["cover"] = _pack(np.concatenate([big, _tris(rng, 60, 0, 1, 0.2)], 0)) + (64,)
    cases["overlap"] = _pack(_tris(rng, 300, 0.2, 0.8, rng.uniform(0.001, 0.3, 300))) + (64,)
    # NaN and inf among the uvs
    tri = _tris(rng, 200, 0, 1, 0.1)
    kind = rng.integers(0, 4, 200)
    comp = rng.integers(0, 6, 200)
    vals = np.array([np.nan, np.inf, -np.inf, 3e38])
    for i in range(200):
        tri[i].reshape(-1)[comp[i]] = vals[kind[i]]
    cases["nonfinite"] = _pack(tri) + (64,)
    # exact hits on texel samples: vertices and edges through the points the texture samples
    g = rng.integers(0, 64, (200, 3, 2)).astype(np.float64) / 64.0
    g[..., 1] = 1 - g[..., 1]
    cases["on_samples"] = _pack(g) + (64,)
    return cases


def queue_cases(seed=0):
    """{name: (uv, faces, res)}: soups whose faces land in one queue of the kernel each: thread (boxes <= 256 texels),
    warp (<= 8192), CTA split across CTAs (few faces), CTA whole faces (more faces than the grid has CTAs), and the
    whole-texture path (faces no candidate box bounds)."""
    rng = np.random.default_rng(seed)
    cases = {}
    cases["thread"] = soup(3000, seed) + (256,)
    cases["warp"] = _pack(_tris(rng, 200, 0.2, 0.8, 0.06)) + (256,)
    cases["cta_split"] = _pack(_tris(rng, 40, 0.3, 0.7, 0.35)) + (256,)
    base = np.array([[0.02, 0.02], [1.1, 0.0], [0.0, 1.1]])
    many = base[None] + rng.uniform(-0.02, 0.02, (1200, 3, 2))
    cases["cta_whole"] = _pack(many) + (96,)
    n = 50
    a = rng.uniform(0.1, 0.9, (n, 2))
    ang = rng.uniform(0, 2 * np.pi, n)
    d = np.stack([np.cos(ang), np.sin(ang)], 1) * 0.3
    e = np.stack([-d[:, 1], d[:, 0]], 1) * 1e-4
    cases["whole_texture"] = _pack(np.stack([a, a + d, a + d * 0.5 + e], 1)) + (128,)
    return cases
