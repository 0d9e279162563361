"""Counts, on the CPU, how many fp64 red sets the composite backward issues for one view of the benchmark's config 1
(D0 cloud, 1920x1080, orbit view 0) with one set per (quadrant, splat) versus one set per (tile, splat).

From the oracle's preprocess it rebuilds the culled tile lists (tight_spans in gs_preprocess.cu) and applies the
composite's per-quadrant test (quad_hit in gs_composite.cu) to the four 8x8 quadrants of every listed tile, in numpy
fp32 (the kernels' approximate lg2 / rcp are replaced by exact ones: the counts can differ in a handful of borderline
pairs).  Quadrants entirely outside the image are not counted: their warps have no pixel and visit nothing.  Both
counts are upper bounds of what the kernel visits, which also stops at each tile's last contributing list position.

    python scripts/dev/count_combine_reds.py [--gaussians 1000000] [--view 0]
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [os.path.join(ROOT, "comfyui-3d-pack_b200"), ROOT]
from oracle import gs_oracle as O  # noqa: E402

f32 = np.float32
L2E = f32(1.4426950408889634)
TILE = 16


def tile_pairs(px, py, A, B, C, o, x0, y0, x1, y1):
    """(splat, tile x, tile y) of the culled lists, as tight_spans() lists them"""
    n = px.size
    w, h = x1 - x0, y1 - y0
    tau = (np.log2(o * f32(255)) * f32(1.001) + f32(0.03)).astype(f32)
    det = (A * C - B * B).astype(f32)
    with np.errstate(all="ignore"):
        ymax = np.sqrt(f32(2) * tau * A / det).astype(f32)
        xmax = np.sqrt(f32(2) * tau * C / det).astype(f32)
        uyr = (-(B * xmax) / C).astype(f32)
    fin = np.isfinite(ymax) & np.isfinite(xmax) & np.isfinite(uyr)
    tight = (w <= 255) & (h <= 8) & (A > 0) & (det > 0) & fin
    dead = (w <= 255) & (h <= 8) & ~(o * f32(255) >= 1)
    tight &= ~dead
    whole = ~tight & ~dead
    S, TX, TY = [], [], []
    k2 = f32(2) * tau * A
    for r in range(8):
        sel = np.nonzero(tight & (h > r))[0]
        a = ((y0[sel] + r) * TILE).astype(f32) - py[sel]
        b = a + f32(TILE - 1)
        lo, hi = np.maximum(a, -ymax[sel]), np.minimum(b, ymax[sel])
        ok = lo <= hi
        yr = np.minimum(np.maximum(uyr[sel], lo), hi)
        yl = np.minimum(np.maximum(-uyr[sel], lo), hi)
        with np.errstate(all="ignore"):
            xr = (-(B[sel] * yr) + np.sqrt(np.maximum(k2[sel] - det[sel] * yr * yr, 0))) / A[sel]
            xl = (-(B[sel] * yl) - np.sqrt(np.maximum(k2[sel] - det[sel] * yl * yl, 0))) / A[sel]
        xr = xr + f32(0.01) + f32(1e-4) * np.abs(xr)
        xl = xl - f32(0.01) - f32(1e-4) * np.abs(xl)
        ta = np.maximum(x0[sel], np.ceil((px[sel] + xl - f32(TILE - 1)) / TILE).astype(np.int64))
        tb = np.minimum(x1[sel] - 1, np.floor((px[sel] + xr) / TILE).astype(np.int64))
        cnt = np.where(ok & (tb >= ta), tb - ta + 1, 0)
        s = np.repeat(sel, cnt)
        off = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        S.append(s); TX.append(np.repeat(ta, cnt) + off); TY.append(np.full(s.size, 0, np.int64) + y0[s] + r)
    for s in np.nonzero(whole & (w > 0) & (h > 0))[0]:
        xs, ys = np.meshgrid(np.arange(x0[s], x1[s]), np.arange(y0[s], y1[s]))
        S.append(np.full(xs.size, s)); TX.append(xs.ravel()); TY.append(ys.ravel())
    return np.concatenate(S), np.concatenate(TX), np.concatenate(TY)


def quad_hit(gx, gy, A, B, C, o, X0, Y0):
    """quad_hit() of gs_composite.cu, vectorised"""
    tau = np.log2(o * f32(255)) * f32(1.001) + f32(0.03)
    ux0, uy0 = X0 - gx, Y0 - gy
    ux1, uy1 = ux0 + f32(7), uy0 + f32(7)
    outx, outy = (ux0 > 0) | (ux1 < 0), (uy0 > 0) | (uy1 < 0)
    q = np.where(outx | outy, f32(3.0e38), f32(0))
    ue = np.where(ux0 > 0, ux0, ux1)
    uy = np.minimum(np.maximum(-B * ue / C, uy0), uy1)
    q = np.where(outx, f32(0.5) * (A * ue * ue + C * uy * uy) + B * ue * uy, q)
    ve = np.where(uy0 > 0, uy0, uy1)
    ux = np.minimum(np.maximum(-B * ve / A, ux0), ux1)
    q = np.where(outy, np.minimum(q, f32(0.5) * (A * ux * ux + C * ve * ve) + B * ux * ve), q)
    pd = (A > 0) & (A * C - B * B > 0)
    return (o * f32(255) >= 1) & (~pd | ~(q > tau))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--view", type=int, default=0)
    ap.add_argument("--views", type=int, default=8, help="views of the orbit ring (bench.py config 1: 8)")
    args = ap.parse_args()
    W, H = 1920, 1080
    cl = O.make_cloud("D0", args.gaussians, 0, seed=0)
    st = O.minicam_settings(O.orbit_camera(0, 360.0 * args.view / args.views, 1.75), W, H, 49.1, sh_degree=0)
    with torch.no_grad():
        pre = O.preprocess(cl["means3D"], cl["scales"], cl["rotations"], cl["opacities"], cl["shs"], None, None, None, st)
    v = pre["visible"].numpy()
    xy, con = pre["xy"].numpy()[v].astype(f32), pre["conic"].numpy()[v].astype(f32)
    o = pre["opacity"].numpy()[v].astype(f32)
    rmin, rmax = pre["rect_min"].numpy()[v], pre["rect_max"].numpy()[v]
    A, B, C = L2E * con[:, 0], L2E * con[:, 1], L2E * con[:, 2]       # log2-scaled conic of the splat record
    s, tx, ty = tile_pairs(xy[:, 0], xy[:, 1], A, B, C, o, rmin[:, 0], rmin[:, 1], rmax[:, 0], rmax[:, 1])
    hits = np.zeros(s.size, np.int64)
    for q in range(4):
        X0, Y0 = tx * TILE + 8 * (q & 1), ty * TILE + 8 * (q >> 1)
        inside = (X0 < W) & (Y0 < H)
        h = quad_hit(xy[s, 0], xy[s, 1], A[s], B[s], C[s], o[s], X0.astype(f32), Y0.astype(f32)) & inside
        hits += h
    quad_pairs, tile_hit = int(hits.sum()), int((hits > 0).sum())
    print(f"visible splats {int(v.sum())}, culled (tile, splat) pairs {s.size}")
    print(f"(quadrant, splat) pairs passing quad_hit: {quad_pairs}")
    print(f"(tile, splat) pairs with at least one such quadrant: {tile_hit}")
    print(f"quadrant hits per (tile, splat) pair: {quad_pairs / tile_hit:.3f} "
          f"-> {100 * (1 - tile_hit / quad_pairs):.1f} % fewer fp64 red sets")


if __name__ == "__main__":
    main()
