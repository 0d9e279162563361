"""Dual-marching-cubes timing on the GPU: gs_b200.isosurface.DiffDMC (the `diso.DiffDMC` drop-in) forward, and
forward + backward, at 257^3, 385^3 and 513^3 (Hunyuan3D's default octree_resolution 384 and TripoSG's octree_depth 9
give the last two).  Inputs are seeded TripoSG-like fields (oracle.dmc_oracle.triposg_field: sdf = -logits / res
from a union of spheres plus noise), once dense and once with the hierarchical decoders' NaN mask beyond a band
around the surface.  `marching_cubes` is timed on the same grid in the same run as a yardstick; it refuses
non-finite samples, so on the masked grid it meshes a copy with NaN replaced by +1.

Times are CUDA-event medians after warm-up; each call includes its one host read.  Also reported: output bytes,
peak `max_memory_allocated` above the inputs per call, and the modelled bytes over the data-sheet HBM bandwidth.
Prints the card name and power limit, then one JSON line per (size, mask).  Dev tool; needs a CUDA device."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "comfyui-3d-pack_b200"))
import torch  # noqa: E402

from gs_b200.isosurface import DiffDMC, marching_cubes  # noqa: E402
from oracle import dmc_oracle as D  # noqa: E402

HBM_BPS = 3.35e12   # H100 SXM data-sheet HBM3 bandwidth, for the model only


def card():
    idx = torch.cuda.current_device()
    q = subprocess.run(["nvidia-smi", "-i", str(idx), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(idx), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def model_bytes(n, nv, nq):
    """Algorithmic bytes of count + write (see csrc/ngp_dmc.cu): the grid once per pass, 12 B per vertex and 24 B per
    triangle pair."""
    return 2 * 4 * n ** 3 + 12 * nv + 24 * nq


def time_ms(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts), min(ts)


def peak_bytes(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base, out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sizes", type=int, nargs="+", default=[257, 385, 513])
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dmc.py needs a CUDA device")
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card()}))
    dmc = DiffDMC().to(dev)
    for n in args.sizes:
        for masked in (False, True):
            grid = D.triposg_field(n, seed=0, device=dev, nan_band=masked)
            mc_grid = torch.nan_to_num(grid, nan=1.0) if masked else grid
            fwd = lambda: dmc(grid, normalize=False)
            gw = grid.clone().requires_grad_(True)

            def fwd_bwd():
                v, _ = dmc(gw, normalize=False)
                v.sum().backward()
                gw.grad = None

            peak, (v, f) = peak_bytes(fwd)
            nv, nq = v.shape[0], f.shape[0] // 2
            out_bytes = v.numel() * 4 + f.numel() * 4
            peak_fb, _ = peak_bytes(fwd_bwd)
            t_f = time_ms(fwd, args.reps)
            t_fb = time_ms(fwd_bwd, args.reps)
            t_mc = time_ms(lambda: marching_cubes(mc_grid, 0.0), args.reps)
            mv, mt = marching_cubes(mc_grid, 0.0)
            mb = model_bytes(n, nv, nq)
            print(json.dumps({
                "size": n, "nan_band": masked, "nan_fraction": round(float(torch.isnan(grid).float().mean()), 4),
                "vertices": nv, "quads": nq, "output_bytes": out_bytes,
                "fwd_ms_median": round(t_f[0], 4), "fwd_ms_min": round(t_f[1], 4),
                "fwd_bwd_ms_median": round(t_fb[0], 4), "fwd_bwd_ms_min": round(t_fb[1], 4),
                "peak_fwd_bytes_above_inputs": peak, "peak_fwd_bwd_bytes_above_inputs": peak_fb,
                "model_bytes": mb, "model_ms_at_datasheet_hbm": round(mb / HBM_BPS * 1e3, 4),
                "marching_cubes_ms_median": round(t_mc[0], 4), "marching_cubes_vertices": mv.shape[0],
                "marching_cubes_triangles": mt.shape[0]}))
            del grid, mc_grid, gw, v, f
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
