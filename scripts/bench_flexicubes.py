"""Times one FlexiCubes training step's extraction (forward + backward) on the GPU: the CUDA kernels
(gs_b200.isosurface.FlexiCubes) against the torch oracle restatement (oracle/fc_oracle.py) in fp32, alternated in one
process, at the FlexiCubes node's inputs (flexicubes_trainer.py:48-56, 133-135: grid x2, SDF rand - 0.1, zero
weights, deform through tanh, training=True).

    python scripts/bench_flexicubes.py [--res 64 128 256] [--reps 10] [--out report.json]

Reports per resolution: median and min milliseconds of both, kernel launches per step, and the compulsory bytes
(inputs read once, outputs and gradients written once) over the CUDA time.  The card's name and power limit are
read in the same run."""
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
    ap.add_argument("--res", type=int, nargs="+", default=[64, 128, 256])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the whole report to this JSON file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_flexicubes needs a GPU"
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
