"""numpy oracle of the point rasterizer and points_projection (gs_b200.points; rules in
include/gs_b200_pts.h), written from those rules with no pytorch3d.

- Projection, pixel centres and squared distances are defined in fp32, one rounding per operation, so they are
  restated here in numpy float32 in the header's operation order (numpy rounds every float32 operation and never
  contracts to FMA); `project64` is the same camera in float64, for checking the convention itself.
- Rasterization is brute force: every pixel tests every point of its cloud, and keeps the K smallest (z, packed index).
- The lift and its backward are in float64: each point takes its winner's features (an exact copy), and the backward
  is the adjoint, summed over a pixel's slots.
"""
import numpy as np

f32 = np.float32
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def project(points, R, T, Km, hw):
    """points [P,3], one camera (R [3,3], T [3], Km [3,3], hw = (h, w)) -> (x_ndc, y_ndc, z) float32 arrays [P]."""
    p = np.asarray(points, f32)
    R, T, Km = np.asarray(R, f32), np.asarray(T, f32), np.asarray(Km, f32)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    c = [((R[i, 0] * x + R[i, 1] * y) + R[i, 2] * z) + T[i] for i in range(3)]
    h, w = f32(hw[0]), f32(hw[1])
    s = min(h, w) * f32(0.5)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        u = (Km[0, 0] * c[0]) / c[2] + Km[0, 2]
        v = (Km[1, 1] * c[1]) / c[2] + Km[1, 2]
        return (w * f32(0.5) - u) / s, (h * f32(0.5) - v) / s, c[2]


def project64(points, R, T, Km, hw):
    """The same camera as an OpenCV pinhole in float64: pixel (u, v) -> NDC ((w/2 - u) / s, (h/2 - v) / s)."""
    p = np.asarray(points, np.float64)
    c = p @ np.asarray(R, np.float64).T + np.asarray(T, np.float64)
    Km = np.asarray(Km, np.float64)
    u = Km[0, 0] * c[:, 0] / c[:, 2] + Km[0, 2]
    v = Km[1, 1] * c[:, 1] / c[:, 2] + Km[1, 2]
    h, w = float(hw[0]), float(hw[1])
    s = min(h, w) / 2
    return (w / 2 - u) / s, (h / 2 - v) / s, c[:, 2]


def pix_ndc(i, S1, S2):
    """pytorch3d's non-square NDC centre of pixel i (counted from the +X / +Y end), float32."""
    rng = (f32(S1) * f32(2.0)) / f32(S2) if S1 > S2 else f32(2.0)
    off = rng / f32(2.0)
    return -off + (rng * np.asarray(i, f32) + off) / f32(S1)


def centres(H, W):
    """(x centre per column [W], y centre per row [H]) of the H x W image, row 0 at the top."""
    return pix_ndc(W - 1 - np.arange(W), W, H), pix_ndc(H - 1 - np.arange(H), H, W)


def _keys(z, pidx):
    return (np.asarray(z, f32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | pidx.astype(np.uint64)


def rasterize(clouds, R, T, Km, hw, H, W, radius, K):
    """clouds: list of [P_i, 3] arrays; R [ncam,3,3], T [ncam,3], Km [ncam,3,3], hw [ncam,2] (None = (H, W)), ncam 1
    or len(clouds).  -> idx int32, zbuf float32, dists float32, each [N, H, W, K]."""
    N = len(clouds)
    idx = np.full((N, H, W, K), -1, np.int32)
    zbuf = np.full((N, H, W, K), -1, f32)
    dists = np.full((N, H, W, K), -1, f32)
    r2 = f32(radius) * f32(radius)
    xc, yc = centres(H, W)
    first = 0
    for n, pts in enumerate(clouds):
        pts = np.asarray(pts, f32).reshape(-1, 3)
        c = n if len(R) > 1 else 0
        px, py, pz = project(pts, R[c], T[c], Km[c], (H, W) if hw is None else hw[c])
        pidx = np.arange(first, first + len(pts))
        first += len(pts)
        ok = (pz > 0) & np.isfinite(px) & np.isfinite(py)
        if not ok.any():
            continue
        px, py, pz, pidx = px[ok], py[ok], pz[ok], pidx[ok]
        key = _keys(pz, pidx)
        dx = xc[:, None] - px[None, :]                                   # [W, P]
        dx2 = dx * dx
        for y in range(H):
            dy = yc[y] - py
            d2 = dx2 + (dy * dy)[None, :]
            hit = d2 < r2
            cols = np.nonzero(hit.any(1))[0]
            if cols.size == 0:
                continue
            km = np.where(hit[cols], key[None, :], EMPTY)
            kk = min(K, km.shape[1])
            best = np.sort(np.partition(km, kk - 1, axis=1)[:, :kk], axis=1) if kk < km.shape[1] else np.sort(km, axis=1)
            for j in range(kk):
                sel = best[:, j] != EMPTY
                x = cols[sel]
                b = best[sel, j]
                p = (b & np.uint64(0xFFFFFFFF)).astype(np.int64)
                col = np.searchsorted(pidx, p)
                idx[n, y, x, j] = p
                zbuf[n, y, x, j] = (b >> np.uint64(32)).astype(np.uint32).view(f32)
                dists[n, y, x, j] = d2[x, col]
    return idx, zbuf, dists


def winners(idx, P):
    """winner [P] int64: the largest linear index e of idx [N,H,W,K] with idx.flat[e] = p, -1 when none."""
    flat = idx.reshape(-1)
    win = np.full(P, -1, np.int64)
    e = np.nonzero(flat >= 0)[0]
    np.maximum.at(win, flat[e], e)
    return win


def lift(idx, features, P):
    """features [N,C,H,W] -> out [P, C] float64: each point's winner pixel's features, 0 without one."""
    N, C, H, W = features.shape
    K = idx.shape[3]
    win = winners(idx, P)
    out = np.zeros((P, C), np.float64)
    has = win >= 0
    pix = win[has] // K
    n, y, x = pix // (H * W), (pix // W) % H, pix % W
    out[has] = np.asarray(features, np.float64)[n, :, y, x]
    return out


def lift_backward(idx, grad_out, C, P):
    """grad_out [P, C] -> grad_features [N,C,H,W] float64: each pixel sums grad_out[p] over the slots whose point p it
    won."""
    N, H, W, K = idx.shape
    win = winners(idx, P)
    g = np.asarray(grad_out, np.float64)
    grad = np.zeros((N, H, W, C), np.float64)
    flat = idx.reshape(-1)
    e = np.nonzero(flat >= 0)[0]
    e = e[win[flat[e]] == e]
    np.add.at(grad.reshape(-1, C), e // K, g[flat[e]])
    return grad.transpose(0, 3, 1, 2)


def opencv_camera(c2w, intrinsic):
    """(R, T, Km) of one camera-to-world matrix, through a float64 inverse."""
    w2c = np.linalg.inv(np.asarray(c2w, np.float64))
    return w2c[:3, :3], w2c[:3, 3], np.asarray(intrinsic, np.float64)
