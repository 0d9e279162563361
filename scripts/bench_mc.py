"""Marching-cubes timing on the GPU: gs_b200.isosurface.marching_cubes (device volume in, device mesh out) and the
`mcubes` numpy shim end to end (cast, upload, mesh, download, dtype casts), at 256^3 and 512^3 on a seeded
Instant-NGP-like density (oracle.mc_oracle.blob_density: anisotropic Gaussian blobs plus noise) at threshold 10,
the density_thresh of marching_cubes_density_to_mesh.

The CPU column is this repository's numpy oracle (oracle/mc_oracle.py), not PyMCubes: PyMCubes is not a dependency,
so nothing here is compared against it.  Prints the card name and power limit, then one JSON line per grid size.
Dev tool; needs a CUDA device."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "comfyui-3d-pack_b200"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import mcubes  # noqa: E402
from gs_b200.isosurface import marching_cubes  # noqa: E402
from oracle import mc_oracle as M  # noqa: E402

HBM_BPS = 3.35e12   # H100 SXM data-sheet HBM3 bandwidth, for the model only


def card():
    idx = torch.cuda.current_device()
    q = subprocess.run(["nvidia-smi", "-i", str(idx), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(idx), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def model_bytes(n_points, nv, nf):
    """Algorithmic bytes of count + 2 scans + write (see csrc/ngp_mcubes.cu)."""
    return 48 * n_points + 12 * nv + 12 * nf


def time_calls(fn, reps):
    fn(); fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts), min(ts)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sizes", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--oracle-sizes", type=int, nargs="*", default=[256],
                    help="sizes at which the CPU numpy oracle is timed once (it takes seconds per call)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_mc.py needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    for n in args.sizes:
        vol = M.blob_density(n, seed=0, device="cuda")
        vol_np = vol.cpu().numpy()
        verts, tris = marching_cubes(vol, 10.0)
        nv, nf = verts.shape[0], tris.shape[0]
        dev_med, dev_min = time_calls(lambda: marching_cubes(vol, 10.0), args.reps)
        shim_med, shim_min = time_calls(lambda: mcubes.marching_cubes(vol_np, 10), max(3, args.reps // 4))
        row = {"grid": n, "vertices": nv, "triangles": nf,
               "device_call_ms_median": round(dev_med, 3), "device_call_ms_min": round(dev_min, 3),
               "numpy_shim_ms_median": round(shim_med, 3), "numpy_shim_ms_min": round(shim_min, 3),
               "model_bytes": model_bytes(n ** 3, nv, nf),
               "model_ms_at_3.35TBps": round(model_bytes(n ** 3, nv, nf) / HBM_BPS * 1e3, 3),
               "achieved_model_GBps_at_median": round(model_bytes(n ** 3, nv, nf) / (dev_med * 1e-3) / 1e9, 1)}
        if n in args.oracle_sizes:
            t0 = time.perf_counter()
            ov, ot = M.marching_cubes(vol_np, 10.0)
            row["cpu_numpy_oracle_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            row["oracle_bit_identical"] = bool(np.array_equal(ov.view(np.uint32), verts.cpu().numpy().view(np.uint32))
                                               and np.array_equal(ot, tris.cpu().numpy()))
        print(json.dumps(row), flush=True)
        del vol, verts, tris
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
