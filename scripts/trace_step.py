"""Kernel trace of one warmed config-1 step (bench.py's flagship workload) under torch.profiler.

Writes the Chrome trace to <out>/trace_step.pt.trace.json and prints
  - each kernel's summed time and launch count, grouped by stage;
  - the step's wall time on the device (first kernel start to last kernel end);
  - the time inside the step during which no composite kernel runs: the part of the step that binning,
    preprocess, preprocess-backward and host round trips put on the critical path.

    python scripts/trace_step.py [--out DIR] [--gaussians 1000000] [--views 8]

DIR defaults to trace_step/ under the system's temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "comfyui-3d-pack_b200"))

STAGES = [   # (stage, kernel-name substrings)
    ("composite_fwd", ("composite_forward",)),
    ("composite_bwd", ("composite_backward",)),
    ("preprocess", ("preprocess_multi", "preprocess_kernel", "sh_colour")),
    ("preprocess_bwd", ("preprocess_backward",)),
    ("depth/tile sort", ("rs_histogram", "rs_scan_hist", "rs_onesweep")),
    ("scan", ("scan_reduce", "scan_block_sums", "scan_apply")),
    ("emit", ("emit",)),
    ("ranges", ("ranges",)),
    ("memset/copy", ("Memset", "Memcpy", "memset", "memcpy")),
]


def stage_of(name):
    for st, keys in STAGES:
        if any(k in name for k in keys):
            return st
    return "other"


def union_len(iv):
    iv = sorted(iv)
    tot, cur_s, cur_e = 0.0, None, None
    for s, e in iv:
        if cur_e is None or s > cur_e:
            if cur_e is not None:
                tot += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    if cur_e is not None:
        tot += cur_e - cur_s
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "trace_step"))
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--sh-degree", type=int, default=3)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("trace_step.py needs a CUDA device")
    from gs_b200 import camera, optim_step, synthetic
    dev = torch.device("cuda", 0)
    N, W, H, deg, V = args.gaussians, args.width, args.height, args.sh_degree, args.views
    params = optim_step.PackedParams(synthetic.make_cloud("D0", N, deg, seed=0, device=dev))
    vnp = camera.orbit_views(V, W, H, n_total=V, start=0)
    views = optim_step.ViewSet(vnp, W, H, deg, dev)
    g = torch.Generator(device="cpu").manual_seed(1234)
    dl = torch.rand(V, 5, H, W, generator=g) * 2 - 1
    dl[:, 3:] *= 0.1
    dl = dl.to(dev)
    for _ in range(5):
        optim_step.step_device_pipelined(params, views, dl)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        optim_step.step_device_pipelined(params, views, dl)
        torch.cuda.synchronize()
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "trace_step.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = json.load(f)["traceEvents"]
    kern = [e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]
    if not kern:
        raise SystemExit("no device activity in the trace")
    t0 = min(e["ts"] for e in kern)
    t1 = max(e["ts"] + e["dur"] for e in kern)
    by_stage, by_kernel = {}, {}
    for e in kern:
        st = stage_of(e["name"])
        by_stage[st] = by_stage.get(st, 0.0) + e["dur"]
        k = by_kernel.setdefault((st, e["name"][:90]), [0.0, 0])
        k[0] += e["dur"]
        k[1] += 1
    comp = [(e["ts"], e["ts"] + e["dur"]) for e in kern if stage_of(e["name"]).startswith("composite")]
    step_us = t1 - t0
    no_comp_us = step_us - union_len(comp)
    print(f"{'stage':16s} {'kernel':90s} {'calls':>5s} {'ms':>8s}")
    for (st, nm), (us, n) in sorted(by_kernel.items(), key=lambda kv: (kv[0][0], -kv[1][0])):
        print(f"{st:16s} {nm:90s} {n:5d} {us / 1e3:8.3f}")
    print("per stage (summed kernel ms):", json.dumps({k: round(v / 1e3, 3) for k, v in sorted(by_stage.items())}))
    summary = {"step_ms_device": step_us / 1e3, "no_composite_ms": no_comp_us / 1e3,
               "composite_busy_ms": union_len(comp) / 1e3, "kernels": len(kern),
               "gpu": torch.cuda.get_device_name(0)}
    print(json.dumps(summary))
    with open(os.path.join(args.out, "trace_step_summary.json"), "w") as f:
        json.dump({"summary": summary, "stages_ms": {k: v / 1e3 for k, v in by_stage.items()},
                   "kernels": [{"stage": st, "name": nm, "calls": n, "ms": us / 1e3} for (st, nm), (us, n) in by_kernel.items()]},
                  f, indent=1)


if __name__ == "__main__":
    main()
