"""Times gs_b200's custom_rasterizer against the reference's own CUDA binary (oracle/_ref, default build: what users of
the reference run) and interpolate against the reference's torch expression, at the Hunyuan3D texture pipelines'
sizes.  CUDA events, median of 10 timed calls after 3 warm-up calls; prints one JSON line per case and writes them
all to --out when given.

    python scripts/bench_custom_rasterizer.py [--out results.json]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "comfyui-3d-pack_b200"), ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import custom_rasterizer as cr  # noqa: E402
from oracle import build_ref  # noqa: E402
from test_gpu_custom_rasterizer import screen_filling, sphere, uv_pos, view_pos  # noqa: E402


def timed(fn, reps=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def torch_interpolate(col, findices, barycentric, tri):
    f = findices - 1 + (findices == 0)
    vcol = col[0, tri.long()[f.long()]]
    return torch.sum(barycentric.view(*barycentric.shape, 1) * vcol, axis=-2).view(1, *barycentric.shape[:2], -1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    ref = build_ref.load("default")
    props = torch.cuda.get_device_properties(0)
    rows = []
    xyz40, tri40, uv40 = sphere(40000, seed=1)
    xyz500, tri500, _ = sphere(500000, seed=2)
    smooth40, stri40, _ = sphere(40000, seed=1, noise=0.0)
    smooth500, stri500, _ = sphere(500000, seed=2, noise=0.0)
    sf_pos, sf_tri = screen_filling()
    # the bumpy spheres' per-vertex noise makes slivers with large boxes (4.7k pixels on average at 40k faces: the warp
    # and CTA queues); the smooth spheres' boxes average 284 (40k) and 38 (500k) pixels, as a decimated mesh's would
    cases = [("view 2048^2, 40k faces", view_pos(xyz40, (2048, 2048)), tri40, (2048, 2048)),
             ("view 2048^2, 500k faces", view_pos(xyz500, (2048, 2048)), tri500, (2048, 2048)),
             ("view 2048^2, smooth, 40k faces", view_pos(smooth40, (2048, 2048)), stri40, (2048, 2048)),
             ("view 2048^2, smooth, 500k faces", view_pos(smooth500, (2048, 2048)), stri500, (2048, 2048)),
             ("UV 4096^2, 40k faces", uv_pos(uv40), tri40, (4096, 4096)),
             ("UV 2048^2, 40k faces", uv_pos(uv40), tri40, (2048, 2048)),
             ("screen-filling, 6 faces at 2048^2", sf_pos, sf_tri, (2048, 2048))]
    for name, pos, tri, hw in cases:
        pos, tri = pos.to(dev), tri.to(dev)
        ours = timed(lambda: cr.rasterize(pos[None], tri, hw))
        theirs = timed(lambda: ref.rasterize_image(pos, tri, torch.zeros(0, device=dev), hw[1], hw[0], 1e-6, 0)) \
            if ref is not None else None
        rows.append({"case": "rasterize " + name, "ours_ms": round(ours, 3),
                     "reference_cuda_ms": None if theirs is None else round(theirs, 3)})
        print(json.dumps(rows[-1]), flush=True)
    # interpolate, C = 3, on the 4096^2 UV bake (uv_feature_map's call)
    pos, tri = uv_pos(uv40).to(dev), tri40.to(dev)
    fi, b = cr.rasterize(pos[None], tri, (4096, 4096))
    rast_out = torch.cat((b, fi.unsqueeze(-1)), dim=-1).unsqueeze(0)
    ids, bary = rast_out[0, ..., -1], rast_out[0, ..., :-1]
    col = torch.randn(1, xyz40.shape[0], 3, device=dev)
    ours = timed(lambda: cr.interpolate(col, ids, bary, tri))
    theirs = timed(lambda: torch_interpolate(col, ids, bary, tri))
    rows.append({"case": "interpolate C=3, 4096^2", "ours_ms": round(ours, 3), "torch_expression_ms": round(theirs, 3)})
    print(json.dumps(rows[-1]), flush=True)
    colg = col.clone().requires_grad_(True)
    bg = bary.clone().requires_grad_(True)
    g = torch.randn(1, 4096, 4096, 3, device=dev)
    ours = timed(lambda: torch.autograd.backward(cr.interpolate(colg, ids, bg, tri), g))
    theirs = timed(lambda: torch.autograd.backward(torch_interpolate(colg, ids, bg, tri), g))
    rows.append({"case": "interpolate C=3, 4096^2, forward + backward", "ours_ms": round(ours, 3),
                 "torch_expression_ms": round(theirs, 3)})
    print(json.dumps(rows[-1]), flush=True)
    meta = {"gpu": props.name, "power_limit": os.popen(
        "nvidia-smi --query-gpu=power.limit --format=csv,noheader -i 0 2>/dev/null").read().strip()}
    print(json.dumps(meta))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"meta": meta, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
