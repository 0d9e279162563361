"""Times one FlexiCubes training step's extraction (forward + backward) on the GPU: the CUDA kernels
(gs_b200.isosurface.FlexiCubes) against the torch oracle restatement (oracle/fc_oracle.py) in fp32, alternated in one
process, at the FlexiCubes node's inputs (flexicubes_trainer.py:48-56, 133-135: grid x2, SDF rand - 0.1, zero
weights, deform through tanh, training=True).

    python scripts/bench_flexicubes.py [--res 64 128 256] [--reps 10] [--out report.json]
    python scripts/bench_flexicubes.py --trellis [--res 256] [--reps 10]

Reports per resolution: median and min milliseconds of both, kernel launches per step, and the compulsory bytes
(inputs read once, outputs and gradients written once) over the CUDA time.  The card's name and power limit are
read in the same run.

--trellis times TRELLIS's mesh decode extraction instead (gs_b200.isosurface.TrellisFlexiCubes, C = 6 colours, in
SparseFeatures2Mesh's dense layout from trellis_inputs): forward only with training off, as the image-to-3D pipeline
runs it, and forward + backward with training on, each against the torch oracle restatement in fp32 (geometry from
oracle/fc_oracle.py, colours from tests/test_trellis_flexicubes_cpu.py), with
torch.cuda.max_memory_allocated above the inputs for each path."""
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


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:               # the measurement stands without it, the report says so
        q = f"nvidia-smi unavailable ({e})"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def inputs(fc, res, seed=0):
    x, cubes = fc.construct_voxel_grid(res)
    x *= 2
    g = torch.Generator(device="cuda").manual_seed(seed)
    sdf = torch.rand(x.shape[0], generator=g, device="cuda") - 0.1
    deform = 0.1 * torch.randn(x.shape, generator=g, device="cuda")
    weight = torch.zeros((cubes.shape[0], 21), device="cuda")
    return x, cubes, sdf, deform, weight


def trellis_inputs(res, seed=0, device="cuda", C=6, band=3.0):
    """SparseFeatures2Mesh's extractor inputs (TRELLIS cube2mesh.py:100-136) at resolution res, restated: a seeded
    band of active cubes `band` cells thick around an analytic surface, per-corner features (sdf with the -1/res bias,
    deform, C colours) averaged over the cubes sharing each grid point, dense default sdf 1 and zeros elsewhere, and
    x = point / res - 0.5 + (1 - 1e-8) / (2 res) tanh(deform).  Returns (x [P,3], sdf [P] and colours [P,C] as views
    of the dense [P,4+C] array, weights [F,21], cube_idx [F,8])."""
    from gs_b200.isosurface import voxel_grid
    g = torch.Generator(device=device).manual_seed(seed)
    R1 = res + 1
    a = torch.arange(res, device=device)
    ijk = torch.stack(torch.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
    scale = torch.tensor([1.0, 0.8, 1.1], device=device)
    surf = lambda p: torch.linalg.vector_norm(p * scale, dim=-1) - 0.3 + \
        0.03 * torch.sin(12 * p[..., 0]) * torch.sin(9 * p[..., 1])
    keep = surf((ijk + 0.5) / res - 0.5).abs() < band / res
    cid = torch.nonzero(keep)[:, 0]
    coords = ijk[cid]
    del ijk, keep
    N = coords.shape[0]
    c = torch.arange(8, device=device)
    corners = coords[:, None, :] + torch.stack([c & 1, (c >> 1) & 1, c >> 2], -1)[None]
    pid = ((corners[..., 0] * R1 + corners[..., 1]) * R1 + corners[..., 2]).reshape(-1)
    sdf = surf(corners / res - 0.5) + 0.5 / res * torch.randn((N, 8), generator=g, device=device) - 1.0 / res
    feats = torch.cat([sdf[..., None], torch.randn((N, 8, 3 + C), generator=g, device=device)], -1).reshape(-1, 4 + C)
    P = R1 ** 3
    sums = torch.zeros((P, 4 + C), device=device).index_add_(0, pid, feats)
    cnt = torch.zeros(P, device=device).index_add_(0, pid, torch.ones_like(pid, dtype=torch.float32))
    dense = torch.zeros((P, 4 + C), device=device)
    dense[:, 0] = 1
    hit = cnt > 0
    dense[hit] = sums[hit] / cnt[hit, None]
    del sums, cnt, feats, corners, pid
    weights = torch.zeros((res ** 3, 21), device=device)
    weights[cid] = 0.5 * torch.randn((N, 21), generator=g, device=device)
    p = torch.arange(P, device=device)
    pts = torch.stack([p // (R1 * R1), (p // R1) % R1, p % R1], 1)
    x = pts / res - 0.5 + (1 - 1e-8) / (res * 2) * torch.tanh(dense[:, 1:4])
    return x, dense[:, 0], dense[:, 4:], weights, voxel_grid(res, device)[1]


def trellis_main(args):
    from gs_b200.isosurface import TrellisFlexiCubes
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_trellis_flexicubes_cpu import flexicubes_colours      # the oracle's geometry plus the colours
    fc = TrellisFlexiCubes(device="cuda")
    report = {"card": card(), "rows": []}
    for res in args.res:
        x, s, col, w, cubes = trellis_inputs(res)
        call = lambda s_, w_, c_, tr: fc(voxelgrid_vertices=x, scalar_field=s_, cube_idx=cubes, resolution=res,
                                         beta=w_[:, :12], alpha=w_[:, 12:20], gamma_f=w_[:, 20],
                                         voxelgrid_colors=c_, training=tr)
        orc = lambda s_, w_, c_, tr: flexicubes_colours(x, s_, res, w_[:, :12], w_[:, 12:20], w_[:, 20],
                                                        training=tr, weight_scale=0.99, dtype=torch.float32,
                                                        attrs=c_)
        cuda_fwd = lambda: call(s, w, col, False)
        orc_fwd = lambda: orc(s, w, col, False)

        def both(fn):
            def run():
                s_ = s.detach().clone().requires_grad_(True)
                w_ = w.detach().clone().requires_grad_(True)
                c_ = col.detach().clone().requires_grad_(True)
                out = fn(s_, w_, c_, True)
                vc = out[4] if len(out) == 5 else out[3]
                (out[0].square().sum() + out[2].mean() + vc.square().sum()).backward()
                return out
            return run

        paths = {"forward": {"cuda": cuda_fwd, "oracle": orc_fwd},
                 "forward_backward": {"cuda": both(call), "oracle": both(orc)}}
        for mode, fns in paths.items():
            row = {"res": res, "mode": mode, "points": x.shape[0], "cubes": cubes.shape[0], "C": col.shape[1]}
            grad = mode == "forward_backward"
            for name, fn in fns.items():
                with torch.set_grad_enabled(grad):
                    out = fn()                                   # warm-up and the one-time cube_idx check
                    torch.cuda.synchronize()
                    if name == "cuda":
                        row["vertices"], row["faces"] = out[0].shape[0], out[1].shape[0]
                    del out
                    torch.cuda.empty_cache()
                    base = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    fn()
                    torch.cuda.synchronize()
                    row[f"{name}_peak_MB_above_inputs"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
                    times = []
                    for _ in range(args.reps):
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        torch.cuda.synchronize()
                        a.record()
                        fn()
                        b.record()
                        torch.cuda.synchronize()
                        times.append(a.elapsed_time(b))
                med = sorted(times)[len(times) // 2]
                row[f"{name}_ms_median"], row[f"{name}_ms_min"] = med, min(times)
            row["speedup_median"] = row["oracle_ms_median"] / row["cuda_ms_median"]
            report["rows"].append(row)
            print(json.dumps(row), flush=True)
        del x, s, col, w, cubes
        torch.cuda.empty_cache()
    print(json.dumps(report["card"]))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(report, fh, indent=1)


def step(extract, x, res, sdf, deform, weight):
    sdf = sdf.detach().requires_grad_(True)
    deform = deform.detach().requires_grad_(True)
    weight = weight.detach().requires_grad_(True)
    grid = x + (2 - 1e-8) / (res * 2) * torch.tanh(deform)
    v, f, L = extract(grid, sdf, weight)[:3]
    (v.square().sum() + L.mean()).backward()
    return v.shape[0], f.shape[0], L.shape[0]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--res", type=int, nargs="+", default=None, help="default 64 128 256, or 256 with --trellis")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--trellis", action="store_true", help="TRELLIS's decode extraction with C = 6 colours")
    ap.add_argument("--out", default=None, help="also write the whole report to this JSON file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_flexicubes needs a GPU"
    if args.trellis:
        args.res = args.res or [256]
        return trellis_main(args)
    args.res = args.res or [64, 128, 256]
    from gs_b200 import _lib
    from gs_b200.isosurface import FlexiCubes
    from oracle import fc_oracle as O
    fc = FlexiCubes(device="cuda")
    report = {"card": card(), "rows": []}
    for res in args.res:
        x, cubes, sdf, deform, weight = inputs(fc, res)
        cuda = lambda g, s, w: fc(g, s, cubes, res, beta_fx12=w[:, :12], alpha_fx8=w[:, 12:20], gamma_f=w[:, 20],
                                  training=True)
        orc = lambda g, s, w: O.flexicubes(g, s, res, w[:, :12], w[:, 12:20], w[:, 20], training=True,
                                           weight_scale=0.99, dtype=torch.float32)
        sizes = step(cuda, x, res, sdf, deform, weight)        # warm-up of both, and the one-time cube_fx8 check
        step(orc, x, res, sdf, deform, weight)
        torch.cuda.synchronize()
        n0 = _lib.lib.gs_b200_launch_count()
        step(cuda, x, res, sdf, deform, weight)
        torch.cuda.synchronize()
        launches = _lib.lib.gs_b200_launch_count() - n0
        times = {"cuda": [], "oracle": []}
        for _ in range(args.reps):
            for name, fn in (("cuda", cuda), ("oracle", orc)):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                step(fn, x, res, sdf, deform, weight)
                b.record()
                torch.cuda.synchronize()
                times[name].append(a.elapsed_time(b))
        P, F = x.shape[0], cubes.shape[0]
        V, T, E = sizes
        # compulsory bytes: forward reads x, s, weights and writes verts, faces, L_dev; backward reads them again
        # plus the output gradients, and writes the input gradients
        fwd = P * 16 + F * 84 + V * 12 + T * 24 + E * 4
        bwd = P * 16 + F * 84 + V * 12 + E * 4 + V * 12 + E * 4 + P * 16 + F * 84
        med = lambda t: sorted(t)[len(t) // 2]
        row = {"res": res, "points": P, "cubes": F, "vertices": V, "faces": T, "L_dev": E,
               "cuda_ms_median": med(times["cuda"]), "cuda_ms_min": min(times["cuda"]),
               "oracle_restatement_ms_median": med(times["oracle"]), "oracle_restatement_ms_min": min(times["oracle"]),
               "speedup_median": med(times["oracle"]) / med(times["cuda"]),
               "library_launches_per_step": launches,
               "compulsory_bytes": fwd + bwd, "compulsory_GB_per_s": (fwd + bwd) / (med(times["cuda"]) * 1e-3) / 1e9}
        report["rows"].append(row)
        print(json.dumps(row), flush=True)
        del x, cubes, sdf, deform, weight
        torch.cuda.empty_cache()
    print(json.dumps(report["card"]))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(report, fh, indent=1)


if __name__ == "__main__":
    main()
