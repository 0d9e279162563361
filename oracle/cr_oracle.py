"""numpy restatement of Hunyuan3D's texture-bake rasterizer (`custom_rasterizer`), bit for bit with the reference's CPU
path as gcc builds it without FMA contraction.  Every fp32 operation below is one numpy float32 operation (one
rounding, no contraction); the reference's `1.0 / area` and `1.0 - beta - gamma` are evaluated in float64 and rounded
to float32, as its double literals make them.  The contract is stated in comfyui-3d-pack_b200/csrc/cr_raster.cu.

rasterize(V, F, W, H, D=None, trunc=1e-6) -> (findices int32 [H,W], barycentric float32 [H,W,3])
interpolate(col, findices, barycentric, tri) -> [1,H,W,C] float32, ((+0 + b0 c0) + b1 c1) + b2 c2, torch's CPU order
"""
import numpy as np

MAXINT = 2 ** 31 - 1
EMPTY = MAXINT * MAXINT + (MAXINT - 1)
f32, f64 = np.float32, np.float64
INT_LO, INT_HI = f32(-2.0 ** 31), f32(2.0 ** 31)


def screen(V, W, H):
    """(x_s, y_s, z_s) float32 per vertex of V[N,4]."""
    V = np.asarray(V, dtype=f32)
    x, y, z, w = V[:, 0], V[:, 1], V[:, 2], V[:, 3]
    with np.errstate(all="ignore"):
        xs = (x / w * f32(0.5) + f32(0.5)) * f32(W - 1) + f32(0.5)
        ys = (f32(0.5) + f32(0.5) * y / w) * f32(H - 1) + f32(0.5)
        zs = z / w * f32(0.49999) + f32(0.5)
    return xs, ys, zs


def _in_int(v):
    return (v >= INT_LO) & (v < INT_HI)


def _trunc_int(v):
    """C's (int) of a float32 as x86's cvttss2si gives it: INT_MIN outside the int range and for NaN."""
    ok = _in_int(v)
    return np.where(ok, np.trunc(np.where(ok, v, f32(0))).astype(np.int64), np.int64(-2 ** 31))


def _bary(x0, y0, x1, y1, x2, y2, area, inv, px, py):
    beta_tri = (x2 - x0) * (py - y0) - (px - x0) * (y2 - y0)
    gamma_tri = (px - x0) * (y1 - y0) - (x1 - x0) * (py - y0)
    b = beta_tri * inv
    c = gamma_tri * inv
    a = ((f64(1.0) - b.astype(f64)) - c.astype(f64)).astype(f32)
    return a, b, c


def face_boxes(V, F, W, H):
    """Per face: (valid, xlo, xhi, ylo, yhi) of the candidate pixels, inclusive and clipped (empty when hi < lo)."""
    xs, ys, zs = screen(V, W, H)
    F = np.asarray(F, dtype=np.int64).reshape(-1, 3)
    N = xs.shape[0]
    idok = ((F >= 0) & (F < N)).all(1)
    Fc = np.where(idok[:, None], F, 0)
    X, Y, Z = xs[Fc], ys[Fc], zs[Fc]
    valid = idok & np.isfinite(Z).all(1) & _in_int(X).all(1) & _in_int(Y).all(1)
    with np.errstate(all="ignore"):
        Xs, Ys = np.where(valid[:, None], X, f32(0)), np.where(valid[:, None], Y, f32(0))
        xlo = np.maximum(0, np.trunc(Xs.min(1)).astype(np.int64))
        ylo = np.maximum(0, np.trunc(Ys.min(1)).astype(np.int64))
        xhi = np.minimum(W - 1, np.ceil(Xs.max(1) + f32(1)).astype(np.int64) - 1)
        yhi = np.minimum(H - 1, np.ceil(Ys.max(1) + f32(1)).astype(np.int64) - 1)
    return valid, xlo, xhi, ylo, yhi


def zbuffer(V, F, W, H, D=None, trunc=1e-6):
    """The reference's z_min after every face: uint64 [H*W] tokens, EMPTY where nothing won."""
    xs, ys, zs = screen(V, W, H)
    F = np.asarray(F, dtype=np.int64).reshape(-1, 3)
    valid, xlo, xhi, ylo, yhi = face_boxes(V, F, W, H)
    z = np.full(H * W, EMPTY, dtype=np.uint64)
    Dflat = None if D is None else np.asarray(D, dtype=f32).reshape(-1)
    tr = f32(trunc)
    for f in np.nonzero(valid & (xhi >= xlo) & (yhi >= ylo))[0]:
        i0, i1, i2 = F[f]
        x0, y0, z0, x1, y1, z1, x2, y2, z2 = xs[i0], ys[i0], zs[i0], xs[i1], ys[i1], zs[i1], xs[i2], ys[i2], zs[i2]
        area = (x2 - x0) * (y1 - y0) - (x1 - x0) * (y2 - y0)
        if area == 0:
            continue
        inv = f32(f64(1.0) / f64(area))
        py, px = np.meshgrid(np.arange(ylo[f], yhi[f] + 1), np.arange(xlo[f], xhi[f] + 1), indexing="ij")
        px, py = px.reshape(-1), py.reshape(-1)
        with np.errstate(all="ignore"):
            a, b, c = _bary(x0, y0, x1, y1, x2, y2, area, inv, px.astype(f32) + f32(0.5), py.astype(f32) + f32(0.5))
            inside = (a >= 0) & (a <= 1) & (b >= 0) & (b <= 1) & (c >= 0) & (c <= 1)
            pix = py * W + px
            depth = a * z0 + b * z1 + c * z2
            thres = f32(0) if Dflat is None else Dflat[pix] * f32(0.49999) + f32(0.5) + tr
            keep = inside & ~(depth < thres)
            q = _trunc_int(depth * f32(262144))
            token = q.astype(np.uint64) * np.uint64(MAXINT) + np.uint64(f + 1)
        np.minimum.at(z, pix[keep], token[keep])
    return z


def resolve(V, F, W, H, z):
    """findices int32 [H,W] and barycentric float32 [H,W,3] from the z-buffer, as the reference's resolve pass."""
    xs, ys, _ = screen(V, W, H)
    V = np.asarray(V, dtype=f32)
    F = np.asarray(F, dtype=np.int64).reshape(-1, 3)
    fid = (z % np.uint64(MAXINT)).astype(np.int64)
    hit = fid != MAXINT - 1
    findices = np.where(hit, fid, 0).astype(np.int32)
    bary = np.zeros((H * W, 3), dtype=f32)
    pix = np.nonzero(hit)[0]
    if pix.size:
        tri = F[fid[pix] - 1]
        x0, y0, x1, y1, x2, y2 = xs[tri[:, 0]], ys[tri[:, 0]], xs[tri[:, 1]], ys[tri[:, 1]], xs[tri[:, 2]], ys[tri[:, 2]]
        with np.errstate(all="ignore"):
            area = (x2 - x0) * (y1 - y0) - (x1 - x0) * (y2 - y0)
            inv = (f64(1.0) / area.astype(f64)).astype(f32)
            px = (pix % W).astype(f32) + f32(0.5)
            py = (pix // W).astype(f32) + f32(0.5)
            a, b, c = _bary(x0, y0, x1, y1, x2, y2, area, inv, px, py)
            a = a / V[tri[:, 0], 3]
            b = b / V[tri[:, 1], 3]
            c = c / V[tri[:, 2], 3]
            w = f32(1.0) / (a + b + c)
            bary[pix] = np.stack([a * w, b * w, c * w], 1)
    return findices.reshape(H, W), bary.reshape(H, W, 3)


def rasterize(V, F, W, H, D=None, trunc=1e-6):
    """custom_rasterizer_kernel.rasterize_image(V, F, D, W, H, trunc, D is not None) on the CPU path."""
    return resolve(V, F, W, H, zbuffer(V, F, W, H, D, trunc))


def interpolate(col, findices, barycentric, tri):
    """custom_rasterizer.interpolate in fp32 with the fixed order ((+0 + b0 c0) + b1 c1) + b2 c2; col[B,V,C]."""
    col = np.asarray(col, dtype=f32)[0]
    fi = np.asarray(findices)
    with np.errstate(all="ignore"):
        f = (fi - fi.dtype.type(1) + (fi == 0).astype(fi.dtype)).astype(np.int64)
    v = np.asarray(tri, dtype=np.int64)[f]                      # [H,W,3]
    b = np.asarray(barycentric, dtype=f32)
    c0, c1, c2 = col[v[..., 0]], col[v[..., 1]], col[v[..., 2]]
    out = f32(0) + b[..., 0:1] * c0 + b[..., 1:2] * c1 + b[..., 2:3] * c2
    return out[None]


def mesh_pos(codes, mvp):
    """Clip-space positions of integer-coded vertices (code / 4096) under a 4x4 float64 matrix, rounded once to fp32."""
    v = np.concatenate([np.asarray(codes, np.float64) / 4096, np.ones((len(codes), 1))], 1)
    return (v @ np.asarray(mvp, np.float64).T).astype(f32)


def golden_cases(path):
    """The cases of tests/golden/ref_custom_rasterizer.npz (see make_golden_custom_rasterizer.py), inputs rebuilt
    exactly: ({name: raster case}, {name: interpolate case}).  A raster case has pos [N,4] fp32, tri [F,3] int32,
    hw, depth (or None) and either findices + bary or digest + covered; an interpolate case has col [1,N,C] fp32,
    src (its raster case), fp32_ids, tri_i64 and either out (fp32) or out_digest."""
    z = np.load(path)
    keys = set(k.split("/")[0] for k in z.files)
    mesh_tri = z["mesh/tri"]
    raster, interp = {}, {}
    for k in sorted(keys - {"mesh"}):
        g = lambda n: z[f"{k}/{n}"] if f"{k}/{n}" in z.files else None  # noqa: E731
        if g("interp_src") is not None:
            col = g("col")
            interp[k] = dict(col=(z["mesh/col_codes"].astype(f32) / 256 if col is None else col.view(f32)),
                             src=str(g("interp_src")), fp32_ids=bool(g("fp32_ids")), tri_i64=bool(g("tri_i64")),
                             out=None if g("out") is None else g("out").view(f32),
                             out_digest=None if g("out_digest") is None else str(g("out_digest")))
            continue
        if g("mvp") is not None:
            pos, tri = mesh_pos(z["mesh/codes"], g("mvp")), mesh_tri
        elif g("uv_pos") is not None:
            uv = z["mesh/uv_codes"].astype(f32) / f32(4096)
            pos = np.concatenate([uv * f32(2) - f32(1), np.zeros_like(uv)], 1)
            pos[:, 3] = 1
            tri = mesh_tri
        else:
            pos, tri = g("pos").view(f32), g("tri")
        raster[k] = dict(pos=pos, tri=tri, hw=tuple(int(v) for v in g("hw")),
                         depth=None if g("depth") is None else g("depth").view(f32),
                         findices=g("findices"), bary=None if g("bary") is None else g("bary").view(f32),
                         digest=None if g("digest") is None else str(g("digest")),
                         covered=None if g("covered") is None else int(g("covered")))
    return raster, interp


def digest(findices, bary):
    """"findices:bary" SHA-256 hex digests of the int32 and fp32 bytes, as the fixture stores them."""
    import hashlib
    return (hashlib.sha256(np.ascontiguousarray(findices, dtype=np.int32).tobytes()).hexdigest() + ":" +
            hashlib.sha256(np.ascontiguousarray(bary, dtype=f32).tobytes()).hexdigest())
