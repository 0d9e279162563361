"""Times gs_b200's SF3D texture baker (rasterize = TextureBaker.rasterize, and one interpolate) against the reference's
own kernels (the oracle/_ref build of slangtorch's generated CUDA, launched as TextureBaker launches it), on the same
inputs, and checks the outputs bit for bit at every timed size.  CUDA events, median of --reps timed calls after
--warm warm-up calls.  Prints the card and its power limit, then one JSON line per case (faces on the whole-texture
path and the queue counts included); writes them all to --out when given.

    python scripts/bench_uvbake.py [--out results.json] [--ref-cap 1.2e12]

The reference tests every texel against every face until the first hit, so its cost is about texels x faces; its arm
is skipped (and the line says so) above --ref-cap texel-face pairs.
"""
import argparse
import importlib.util
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "comfyui-3d-pack_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

from gs_b200 import uv_bake  # noqa: E402
from oracle import build_ref_sf3d  # noqa: E402
from oracle import uvbake_oracle as O  # noqa: E402


def timed(fn, reps, warm):
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


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"unknown ({e!r})"
    return name, q


def golden_cases():
    path = os.path.join(ROOT, "tests", "golden", "ref_sf3d_baker.npz")
    if not os.path.isfile(path):
        return []
    spec = importlib.util.spec_from_file_location("mk", os.path.join(ROOT, "tests", "golden", "make_golden_sf3d_baker.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    z = dict(np.load(path))
    out = []
    for name in mk.MESHES:
        uv, faces, pos, _ = mk.soup(z, name)
        if pos is None:         # stored with its uvs only
            pos = np.random.default_rng(0).standard_normal((uv.shape[0], 3)).astype(np.float32)
        for res in (1024, 2048):
            out.append((f"golden_{name}", uv, faces, pos, res))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--ref-cap", type=float, default=1.2e12)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warm", type=int, default=2)
    args = ap.parse_args()
    name, plimit = card()
    print(json.dumps({"device": name, "power_limit": plimit}), flush=True)
    lib = build_ref_sf3d.load()
    cases = golden_cases()
    rng = np.random.default_rng(0)
    for F in (10 ** 5, 10 ** 6):
        uv, faces = O.soup(F, 1)
        pos = rng.standard_normal((uv.shape[0], 3)).astype(np.float32)
        for res in (1024, 2048, 4096, 8192):
            cases.append((f"soup_{F}", uv, faces, pos, res))
    adv = O.adversarial(0)["slivers"]
    cases.append(("slivers", adv[0], adv[1], rng.standard_normal((adv[0].shape[0], 3)).astype(np.float32), 1024))
    results = []
    for label, uv, faces, pos, res in cases:
        dev = torch.device("cuda:0")
        uv_t, f_t, pos_t = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (uv, faces, pos))
        F = int(f_t.shape[0])
        n = (res // 16) * 16
        out = torch.empty(res, res, 4, device=dev)
        _, (warp, cta, whole) = uv_bake.rasterize_into(uv_t, f_t, out, n, n, counts=True)
        ip = torch.zeros(res, res, 3, device=dev)
        t_bake = timed(lambda: uv_bake.rasterize_into(uv_t, f_t, out, n, n), args.reps, args.warm)
        t_interp = timed(lambda: uv_bake.interpolate_into(pos_t, out, f_t, ip, n, n), args.reps, args.warm)
        row = {"case": label, "faces": F, "res": res, "ours_bake_ms": round(t_bake, 4),
               "ours_interp_ms": round(t_interp, 4), "warp_queue": warp, "cta_queue": cta,
               "whole_texture_faces": whole}
        if lib is None:
            row["reference"] = "skipped: no oracle/_ref SF3D build"
        elif float(res) * res * F > args.ref_cap:
            row["reference"] = f"skipped: {float(res) * res * F:.2e} texel-face pairs > cap {args.ref_cap:.2e}"
        else:
            ref = torch.empty(res, res, 4, device=dev)
            rip = torch.zeros(res, res, 3, device=dev)
            s = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731
            g = res // 16
            bake = lambda: lib.sf3d_ref_bake_uv(uv_t.data_ptr(), uv_t.shape[0], f_t.data_ptr(), F, ref.data_ptr(),  # noqa: E731
                                                res, res, 16, 16, g, g, s())
            interp = lambda: lib.sf3d_ref_interpolate(pos_t.data_ptr(), pos_t.shape[0], f_t.data_ptr(), F,  # noqa: E731
                                                      ref.data_ptr(), rip.data_ptr(), res, res, 16, 16, g, g, s())
            reps, warm = (1, 1) if float(res) * res * F > 1e11 else (args.reps, args.warm)
            t_rb = timed(bake, reps, warm)
            t_ri = timed(interp, args.reps, args.warm)
            out.fill_(-7.25)
            ref.fill_(-7.25)
            uv_bake.rasterize_into(uv_t, f_t, out, n, n)
            bake()
            uv_bake.interpolate_into(pos_t, out, f_t, ip, n, n)
            interp()
            torch.cuda.synchronize()
            row.update({"ref_bake_ms": round(t_rb, 3), "ref_interp_ms": round(t_ri, 4),
                        "bake_speedup": round(t_rb / t_bake, 1),
                        "bits_equal": bool(torch.equal(out.view(torch.int32), ref.view(torch.int32))
                                           and torch.equal(ip.view(torch.int32), rip.view(torch.int32)))})
        print(json.dumps(row), flush=True)
        results.append(row)
        del out, ip
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"device": name, "power_limit": plimit, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
