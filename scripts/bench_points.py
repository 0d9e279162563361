"""Times TriplaneGaussian's point projection (gs_b200.points.points_projection: rasterize at K = 1, then lift the
feature map onto the points) at its own sizes against a torch-only brute force of the same rules on the same card,
alternated in one process.

    python scripts/bench_points.py [--reps 20]

Cases (B = 1, a 252 x 252 feature map of 773 channels, radius 0.0075, as TriplaneGaussian's config and
utils/ops.py call it; points uniform in [-0.5, 0.5]^3 seen from distance 2 with a 40 degree field of view):
  proj_2k / proj_16k   the fused forward at 2048 / 16384 points, against torch: project, test every (pixel, point)
                       pair in chunks of pixel rows, take each pixel's nearest (z, index) and write the features with
                       index_put in pixel order
  bwd_16k              the lift's backward to the feature map at 16384 points (ours only)
  raster_16k_k1 / _k8  PointsRasterizer alone at 16384 points, points_per_pixel = 1 / 8 (ours only)
  inverse              the torch.linalg.inv_ex of the camera-to-world matrix that points_projection starts with
Prints the card's name, power limit and clocks, then one JSON line per case: milliseconds (the lower of two alternated
runs, each the median over reps of CUDA events), and for the fused forward the compulsory bytes over our time.
Before timing, the pixels where the torch brute force's idx equals ours are counted and reported."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "comfyui-3d-pack_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

H = W = 252
C = 773
RADIUS = 0.0075


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:               # the measurement stands without it, the report says so
        q = f"nvidia-smi unavailable ({e})"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    ms.sort()
    return ms[len(ms) // 2]


def alternated(ours, theirs, reps, theirs_reps=None):
    t = [[], []]
    for _ in range(2):
        t[0].append(timed(ours, reps))
        if theirs is not None:
            t[1].append(timed(theirs, theirs_reps or reps))
    return min(t[0]), (min(t[1]) if theirs is not None else None)


def inputs(g, Np, dev):
    pts = (torch.rand(1, Np, 3, generator=g, device=dev) - 0.5)
    eye = torch.tensor([1.2, -1.1, 1.1], device=dev)
    eye = eye * (2.0 / eye.norm())
    fwd = -eye / eye.norm()
    right = torch.linalg.cross(fwd, torch.tensor([0.0, 0.0, 1.0], device=dev))
    right = right / right.norm()
    down = torch.linalg.cross(fwd, right)
    c2w = torch.eye(4, device=dev)
    c2w[:3, :3] = torch.stack([right, down, fwd], 1)
    c2w[:3, 3] = eye
    f = 0.5 * H / torch.tan(torch.tensor(20.0).deg2rad()).item()
    K = torch.tensor([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], device=dev)
    feat = torch.randn(1, C, H, W, generator=g, device=dev)
    return pts, c2w[None], K[None], feat


def torch_projection(pts, c2w, K, feat, rows=36):
    """The same rules in torch: every pixel tests every point; nearest (z, index) wins; index_put in pixel order."""
    w2c = torch.linalg.inv_ex(c2w)[0][0]
    p = pts[0]
    c = p @ w2c[:3, :3].T + w2c[:3, 3]
    s = min(H, W) / 2
    u = K[0, 0, 0] * c[:, 0] / c[:, 2] + K[0, 0, 2]
    v = K[0, 1, 1] * c[:, 1] / c[:, 2] + K[0, 1, 2]
    x, y, z = (W / 2 - u) / s, (H / 2 - v) / s, c[:, 2]
    ok = z > 0
    i = torch.arange(max(H, W), device=p.device, dtype=torch.float32)
    xc = (-1.0 + (2.0 * i[:W] + 1.0) / W).flip(0)
    yc = (-1.0 + (2.0 * i[:H] + 1.0) / H).flip(0)
    zkey = torch.where(ok, z, torch.full_like(z, float("inf")))
    idx = torch.empty(H, W, dtype=torch.long, device=p.device)
    for r0 in range(0, H, rows):
        dy = yc[r0:r0 + rows, None, None] - y
        dx = xc[None, :, None] - x
        hit = dx * dx + dy * dy < RADIUS * RADIUS
        zz = torch.where(hit, zkey, torch.full_like(zkey, float("inf")))
        best, arg = zz.min(-1)
        idx[r0:r0 + rows] = torch.where(torch.isfinite(best), arg, torch.full_like(arg, -1))
    vis = idx >= 0
    out = torch.zeros(p.size(0), C, device=p.device)
    out[idx[vis]] = feat[0].permute(1, 2, 0)[vis]
    return idx, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_points.py needs a CUDA device")
    from gs_b200 import points as P
    dev = torch.device("cuda:0")
    print(json.dumps(card()))
    g = torch.Generator(device=dev).manual_seed(0)
    for Np in (2048, 16384):
        pts, c2w, K, feat = inputs(g, Np, dev)
        ours = lambda: P.points_projection(pts, c2w, K, feat, RADIUS, 1)   # noqa: E731
        idx_t, _ = torch_projection(pts, c2w, K, feat)
        w2c = torch.linalg.inv_ex(c2w)[0]
        cams = P.cameras_from_opencv_projection(w2c[:, :3, :3], w2c[:, :3, 3], K, torch.tensor([[H, W]], device=dev))
        fr = P.PointsRasterizer(cams, P.PointsRasterizationSettings((H, W), RADIUS, 1))(P.Pointclouds(pts))
        same = int((fr.idx[0, ..., 0].long() == idx_t).sum())
        t_ours, t_torch = alternated(ours, lambda: torch_projection(pts, c2w, K, feat), a.reps, max(3, a.reps // 4))
        nbytes = Np * 12 + H * W * 4 * 3 + 2 * Np * C * 4       # points; idx written, read twice; features in, out
        print(json.dumps({"case": f"proj_{Np // 1024}k", "points": Np, "ours_ms": round(t_ours, 4),
                          "torch_ms": round(t_torch, 3), "idx_equal_pixels": f"{same}/{H * W}",
                          "compulsory_MB": round(nbytes / 1e6, 1), "GB_per_s": round(nbytes / t_ours / 1e6, 1)}))
    f = feat.clone().requires_grad_(True)
    out = P.points_projection(pts, c2w, K, f, RADIUS, 1)
    go = torch.randn_like(out)
    t_bwd, _ = alternated(lambda: torch.autograd.grad(out, f, go, retain_graph=True), None, a.reps)
    print(json.dumps({"case": "bwd_16k", "points": 16384, "ours_ms": round(t_bwd, 4)}))
    pc = P.Pointclouds(pts)
    for k in (1, 8):
        rk = P.PointsRasterizer(cams, P.PointsRasterizationSettings((H, W), RADIUS, k))
        t_rk, _ = alternated(lambda: rk(pc), None, a.reps)
        print(json.dumps({"case": f"raster_16k_k{k}", "points": 16384, "ours_ms": round(t_rk, 4)}))
    t_inv, _ = alternated(lambda: torch.linalg.inv_ex(c2w), None, a.reps)
    print(json.dumps({"case": "inverse", "ours_ms": round(t_inv, 4)}))


if __name__ == "__main__":
    main()
