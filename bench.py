#!/usr/bin/env python
"""Benchmark of the hot path (BASELINE.json metric), one JSON line on stdout (rank 0).

  python bench.py --gpus N --steps K --warmup W            # CUDA arm (H100, sm_90a), 3DGS rasterizer (configs 1 / 2)
  python bench.py --impl reference --steps K --warmup W    # CPU arm: the pure-PyTorch oracle port
  python bench.py --workload ngp   [--impl reference]      # BASELINE config 3 (Instant-NGP), single GPU
  python bench.py --workload mesh  [--impl reference]      # BASELINE config 4 (mesh ops), single GPU

3DGS (default workload): a "step" = rasterizer forward + backward over this rank's orbit views of the N-Gaussian
cloud (1M Gaussians D0, SH degree 3, 1920x1080), gradients summed over views in place.
  N = 1 : config 1 — V = 8 views.
  N > 1 : config 2 — the 200-view ring dealt over the ranks, ceil(200/N) views per rank (25 at N = 8), ONE
          all-reduce of the packed gradient buffer per step, issued from inside the step (parallel.OverlappedGradAllReduce;
          --ar-chunks > 1 cuts it into Gaussian-range chunks behind the last pass: measured, does not pay, DESIGN.md 7);
          the weak-scaling figure with 8 views per rank is measured too and reported as config.weak_8_views_per_rank.
metric = Msplats/s = N_gaussians * (views of all ranks) / t.

--dump-outputs DIR writes what the timed step computed in its last timed step as DIR/<name>.npy (float32 / float64,
at most 64 MiB in all; larger outputs as a fixed, seeded row sample), so that two builds can be compared output for
output: the inputs are seeded, so the same arguments give the same inputs on every run.
"""
import argparse
import atexit
import json
import math
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "comfyui-3d-pack_b200"))
sys.path.insert(0, ROOT)

METRIC = "Msplats/sec fwd+bwd"
UNIT = "Msplats/s"


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--workload", default="gs", choices=["gs", "ngp", "mesh"])
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--views", type=int, default=None, help="views per rank (default: 8 at N=1, ceil(200/N) at N>1)")
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--sh-degree", type=int, default=3)
    ap.add_argument("--cloud", default="D0", choices=["D0", "D1"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--cpu-sample", default="50000,480,270")
    ap.add_argument("--ar-chunks", type=int, default=1, help="Gaussian-range chunks of the overlapped all-reduce")
    ap.add_argument("--triangles", type=int, default=500_000, help="mesh workload: triangle count")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the outputs of the last timed step as DIR/<name>.npy (CUDA arm, rank 0)")
    return ap.parse_args()


DUMP_LIMIT = 64 * 2 ** 20
DUMP_ROWS = 200_000          # Gaussians sampled from the packed gradient buffer (62 floats each at SH degree 3)


def dump_outputs(out_dir, arrays):
    """arrays: name -> tensor / array; floating arrays keep float64 or become float32, integer arrays become float64.
    When they exceed DUMP_LIMIT, every array over 1 MiB is cut to a fixed, seeded sample of its rows (last axis = one
    row), written as <name>.npy with the sampled row numbers in <name>_rows.npy."""
    import numpy as np
    import torch
    conv = {}
    for name, a in arrays.items():
        a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
        conv[name] = np.ascontiguousarray(a, dtype=np.float64 if a.dtype in (np.float64, np.int64, np.int32) else np.float32)
    total = sum(a.nbytes for a in conv.values())
    if total > DUMP_LIMIT:
        large = [k for k, a in conv.items() if a.nbytes > 2 ** 20]
        small = total - sum(conv[k].nbytes for k in large)
        rows = {k: conv[k].reshape(-1, conv[k].shape[-1] if conv[k].ndim > 1 else 1) for k in large}
        frac = (0.95 * DUMP_LIMIT - small) / sum(r.shape[0] * (r.itemsize * r.shape[1] + 8) for r in rows.values())
        rng = np.random.default_rng(0)
        for k, r in rows.items():
            idx = np.sort(rng.choice(r.shape[0], max(1, int(r.shape[0] * frac)), replace=False))
            conv[k], conv[k + "_rows"] = r[idx], idx.astype(np.float64)
    os.makedirs(out_dir, exist_ok=True)
    for name, a in conv.items():
        np.save(os.path.join(out_dir, name + ".npy"), a)


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
        except Exception:  # noqa: BLE001
            pass
    return 3350.0, "H100 SXM data sheet 3.35 TB/s"


def traffic_of(kernel):
    tr = os.path.join(ROOT, "profiles", "dominant_kernel_traffic.json")
    if os.path.exists(tr):
        try:
            return json.load(open(tr)).get(kernel)
        except Exception:  # noqa: BLE001
            pass
    return None


# --------------------------------------------------------------------------------------
# clocks sampler
# --------------------------------------------------------------------------------------
class Clocks:
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index, interval_ms=20):
        self.f = tempfile.NamedTemporaryFile("w+", suffix=".csv", delete=False)
        try:
            self.p = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                       "-i", str(gpu_index), "-lms", str(int(interval_ms))], stdout=self.f, stderr=subprocess.DEVNULL)
        except Exception:  # noqa: BLE001
            self.p = None
        atexit.register(self._end)        # the poller must not outlive bench.py when a measurement raises

    def _end(self):
        if self.p is not None and self.p.poll() is None:
            self.p.kill()
            self.p.wait()
        if os.path.exists(self.f.name):
            os.unlink(self.f.name)

    def stop(self):
        out = {"sm_mhz": None, "sm_max_mhz": None, "reasons": []}
        if self.p is None:
            return out
        self.p.terminate()
        try:
            self.p.wait(timeout=5)
        except Exception:  # noqa: BLE001
            self.p.kill()
        self.f.flush(); self.f.seek(0)
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.f.read().splitlines():
            c = [x.strip() for x in ln.split(",")]
            if len(c) < 9:
                continue
            try:
                sm.append(float(c[1])); mx.append(float(c[2]))
            except ValueError:
                continue
            for nm, v in zip(names, c[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(nm)
        os.unlink(self.f.name)
        if sm:
            sm.sort()
            out = {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": max(mx), "reasons": sorted(reasons), "samples": len(sm)}
        return out


def timed(fn, steps, warmup):
    """ms per call of fn(): `warmup` untimed calls, then `steps` calls between CUDA events (synchronize on both sides)."""
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


# ======================================================================================
# 3DGS rasterizer (configs 1 and 2)
# ======================================================================================
def gs_cpu_sample_run(sample, sh_degree, cloud_kind, steps, warmup):
    """Times oracle fwd+bwd of one view on a bounded sample; returns (Msplats/s, ms/step, cores, desc)."""
    import torch
    from oracle import gs_oracle as O
    n, w, h = sample
    # torch intra-op threading on the per-tile tensors stops scaling (and then collapses) past ~16 threads:
    # 128 threads were 25x SLOWER than 8 on the GPU box's host.  Use at most 16 and report that count.
    cores = min(os.cpu_count() or 1, 16)
    torch.set_num_threads(cores)
    cl = O.make_cloud(cloud_kind, n, sh_degree, seed=0)
    st = O.minicam_settings(O.orbit_camera(0, 0, 1.75), w, h, 49.1, sh_degree=sh_degree)
    g = torch.Generator().manual_seed(0)
    dc = torch.rand(3, h, w, generator=g) * 2 - 1
    dd = (torch.rand(1, h, w, generator=g) * 2 - 1) * 0.1
    da = (torch.rand(1, h, w, generator=g) * 2 - 1) * 0.1
    inp = {k: cl[k] for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    for _ in range(warmup):
        O.rasterize_with_grads(inp, st, dc, dd, da)
    t0 = time.perf_counter()
    for _ in range(steps):
        O.rasterize_with_grads(inp, st, dc, dd, da)
    dt = (time.perf_counter() - t0) / max(steps, 1)
    desc = (f"oracle/gs_oracle.py fwd+bwd, 1 view, {cloud_kind} N={n} SH{sh_degree} {w}x{h}, torch {cores} threads "
            f"(host has {os.cpu_count()} cores), {warmup} warm-up + {steps} timed steps")
    return n / dt / 1e6, dt * 1e3, cores, desc


def run_gs_reference(args):
    sample = tuple(int(x) for x in args.cpu_sample.split(","))
    val, ms, cores, desc = gs_cpu_sample_run(sample, args.sh_degree, args.cloud, args.steps, max(args.warmup, 0))
    return {
        "impl": "reference", "metric": METRIC, "value": val, "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": {"workload": f"3DGS optimisation fwd+bwd, {args.cloud} random-init cloud, bounded CPU sample of config 1",
                   "sample": desc},
        "cpu_baseline": {"value": val, "unit": UNIT, "cores": cores, "kind": "port", "sample": desc},
        "e2e": {"value": val, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
        "note": "reference rasterizer (diff_gaussian_rasterization) is an un-vendored third-party CUDA package, unavailable "
                "offline; this arm times the pure-PyTorch CPU restatement of the same path on the host cores",
    }


def run_gs(args):
    import ctypes as C
    import numpy as np
    import torch
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py (impl b200) needs a CUDA device; there is no CPU fallback")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    from gs_b200 import _lib, camera, optim_step, parallel, synthetic
    from gs_b200 import rasterizer as _R

    N, W, H, deg = args.gaussians, args.width, args.height, args.sh_degree
    M = (deg + 1) ** 2
    RING = 200
    V = args.views if args.views else (8 if world == 1 else math.ceil(RING / world))
    cloud = synthetic.make_cloud(args.cloud, N, deg, seed=0, device=dev)       # replicated on every rank
    params = optim_step.PackedParams(cloud)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def make_views(v_per_rank):
        """this rank's share of the ring, dealt round-robin like parallel.shard_views (rank r: views r, r+world, ...)"""
        if world == 1:
            vnp = camera.orbit_views(v_per_rank, W, H, n_total=v_per_rank, start=0)
        else:
            ring = max(RING, v_per_rank * world)
            idx = [rank + world * k for k in range(v_per_rank)]
            vnp = np.ascontiguousarray(np.concatenate([camera.orbit_views(1, W, H, n_total=ring, start=i % ring) for i in idx], axis=0))
        g = torch.Generator(device="cpu").manual_seed(1234 + rank)
        dl_cpu = torch.rand(v_per_rank, 5, H, W, generator=g) * 2 - 1
        dl_cpu[:, 3:] *= 0.1
        return vnp, optim_step.ViewSet(vnp, W, H, deg, dev), dl_cpu

    def measure(v_per_rank, steps, warmup):
        vnp, views, dl_cpu = make_views(v_per_rank)
        dl = dl_cpu.to(dev)
        ar = parallel.OverlappedGradAllReduce(params.grads, N, M, nchunks=args.ar_chunks)
        state = {}

        def step():
            with ar:
                state["pairs"] = optim_step.step_device_pipelined(params, views, dl)
            ar.wait()
        for _ in range(warmup):
            step()
        barrier()
        l0 = _lib.lib.gs_b200_launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        barrier()
        e0.record()
        for _ in range(steps):
            step()
        e1.record()
        barrier()
        ms_total = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms_total, op=dist.ReduceOp.MAX)
        ms_step = float(ms_total.item()) / steps
        launches = int(_lib.lib.gs_b200_launch_count() - l0)
        return dict(ms_step=ms_step, value=N * v_per_rank * world / (ms_step * 1e-3) / 1e6, launches=launches,
                    pairs=state["pairs"], vnp=vnp, views=views, dl=dl, dl_cpu=dl_cpu)

    # started before warm-up so it is sampling during the timed region.  Multi-rank steps are long (25-100 views), so the
    # recipe's coarser polling gives as many samples per step; on the 8-GPU box the 20 ms polling is the prime suspect for
    # a 25-view step measuring 29.9 ms (poller on) where the 8-view step right after (poller off) scaled (DESIGN 7)
    clocks = Clocks(local, 20 if world == 1 else 100) if rank == 0 else None
    main = measure(V, args.steps, max(args.warmup, 3))
    clk = clocks.stop() if clocks else None
    if args.dump_outputs and rank == 0:
        # the packed gradient buffer of the last timed step (all-reduced when world > 1), sampled at fixed Gaussians
        rows = torch.randperm(N, generator=torch.Generator().manual_seed(0))[:min(N, DUMP_ROWS)].sort().values
        ri = rows.to(dev)
        arrays = {"gaussian_index": rows, "pairs": torch.tensor([main["pairs"]], dtype=torch.int64)}
        o = 0
        for nm, wdt in zip(("means3D", "shs", "opacities", "scales", "rotations", "means2D"), parallel.GROUP_WIDTHS(M)):
            arrays["grad_" + nm] = params.grads[o:o + N * wdt].view(N, wdt).index_select(0, ri)
            o += N * wdt
        dump_outputs(args.dump_outputs, arrays)
    ms_step, value, launches = main["ms_step"], main["value"], main["launches"]
    weak = None
    if world > 1 and V != 8:
        main.pop("dl"); main.pop("dl_cpu")
        torch.cuda.empty_cache()
        prof = measure(8, args.steps, 3)
        weak = {"value": prof["value"], "unit": UNIT, "ms_per_step": prof["ms_step"], "views_per_gpu": 8}
    else:
        prof = main
    views, dl, vnp, dl_cpu = prof["views"], prof["dl"], prof["vnp"], prof["dl_cpu"]
    Vp = views.V

    # ---- per-stage profile pass (events on the launching stream) -> roofline of the dominant kernel.
    # The per-view C entries run the same kernels one view at a time.  Pair count of the package's own tile lists
    # (culling off) = the K of SURVEY 8d's algorithmic-bytes formula; the timed stages run with culling on, like the step.
    mode0 = _R.get_tile_culling()
    _R.set_tile_culling(0)
    pairs_package = optim_step.step_device(params, views, dl)
    _R.set_tile_culling(2 if mode0 >= 1 else 0)
    pairs_culled = optim_step.step_device(params, views, dl)
    _lib.lib.gs_b200_profile_enable(1)
    for _ in range(2):
        optim_step.step_device(params, views, dl)
    torch.cuda.synchronize()
    _R.set_tile_culling(mode0)
    ms = (C.c_float * _lib.NSTAGES)(); calls = (C.c_int32 * _lib.NSTAGES)()
    _lib.check(_lib.lib.gs_b200_profile_read(ms, calls))
    _lib.lib.gs_b200_profile_enable(0)
    stage_ms = {nm: (ms[i] / calls[i] if calls[i] else 0.0) for i, nm in enumerate(_lib.STAGE_NAMES)}
    pairs_view = pairs_package / Vp          # pairs of the package's tile lists: the algorithm's K*N
    pairs_proc = pairs_culled / Vp           # (tile, splat) pairs the kernels actually walk (tile culling on)
    npix = W * H
    c_in = 4 * (3 + 3 + 4 + 1 + 3 * M)

    def alg_bytes(pv):       # algorithmic bytes per launch (SURVEY 8d / DESIGN.md 5) for pv pairs per view
        return {"preprocess": N * c_in + N * 48, "depth_sort": N * 24, "scan": N * 8, "emit": pv * 12, "tile_sort": pv * 24,
                "ranges": pv * 4, "composite_fwd": pv * 44 + npix * 24, "composite_bwd": pv * (44 + 40) + npix * 28,
                "preprocess_bwd": N * (2 * c_in + 12) + N * 40}
    alg, alg_c = alg_bytes(pairs_view), alg_bytes(pairs_proc)
    dom = max(stage_ms, key=lambda k: stage_ms[k])
    peak, peak_src = peaks()
    t_dom = stage_ms[dom] * 1e-3
    ach = alg[dom] / t_dom / 1e9 if t_dom > 0 else 0.0
    ach_c = alg_c[dom] / t_dom / 1e9 if t_dom > 0 else 0.0
    roofline = {"bound": "hbm", "kernel": dom, "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak,
                "traffic": traffic_of(dom), "peak_source": peak_src,
                "algorithmic_bytes_per_launch": alg[dom], "avg_launch_ms": stage_ms[dom],
                "algorithmic_pairs": "package tile lists (K*N of SURVEY 8d, culling off); the kernels walk the culled lists",
                "on_culled_lists": {"achieved": ach_c, "frac": ach_c / peak, "algorithmic_bytes_per_launch": alg_c[dom]},
                "stage_ms_per_view": stage_ms,
                "note": "the composite kernels are instruction-issue bound (records are L2-resident): the HBM fraction is "
                        "reported as asked, the issue-slot utilisation is in profiles/",
                "step_bytes_all_stages": sum(alg.values()) * Vp}

    # ---- e2e: host buffers through the C-ABI step entry, copies inside the timed region
    e2e = None
    if not args.no_e2e:
        cloud_cpu = {k: v.cpu() for k, v in cloud.items()}
        hs = optim_step.HostStep(cloud_cpu, vnp, W, H, deg, dl_cpu)
        gdev = torch.empty(hs.n_grad, dtype=torch.float32, device=dev) if world > 1 else None
        ghost = torch.empty(hs.n_grad, dtype=torch.float32).pin_memory() if world > 1 else None

        def e2e_step():
            if world > 1:
                hs.run_dev_grads(gdev)
                dist.all_reduce(gdev)
                ghost.copy_(gdev, non_blocking=True)
                torch.cuda.synchronize()
            else:
                hs.run()
        for _ in range(3):
            e2e_step()
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            e2e_step()
        e1.record()
        barrier()
        ms_e = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms_e, op=dist.ReduceOp.MAX)
        ms_e2e = float(ms_e.item()) / args.steps
        e2e = {"value": N * Vp * world / (ms_e2e * 1e-3) / 1e6, "unit": UNIT, "ms_per_step": ms_e2e, "views_per_gpu": Vp,
               "h2d_bytes_per_step": hs.h2d_bytes, "d2h_bytes_per_step": hs.d2h_bytes,
               "api": "gs_b200_step_host (pinned host buffers; binning of every view runs while the SH block uploads, upstream gradients stream in behind the compute, gradients go back in range chunks)"}

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return None
    cpu = None
    if not args.no_cpu_baseline and world == 1:      # reported at N=1 only (contract): keeps multi-rank runs short
        sample = tuple(int(x) for x in args.cpu_sample.split(","))
        v, ms_cpu, cores, desc = gs_cpu_sample_run(sample, deg, args.cloud, 3, 1)      # warm-up + 3 steps, like the reference arm
        cpu = {"value": v, "unit": UNIT, "cores": cores, "kind": "port", "sample": desc, "ms_per_step": ms_cpu}
    config = {"workload": (f"3DGS optimisation fwd+bwd: {N} Gaussians ({args.cloud} reference random-init), SH degree {deg}, {W}x{H}, "
                           + (f"config 1: {V}-view orbit (radius 1.75, fovy 49.1)" if world == 1 else
                              f"config 2: 200-view orbit ring dealt over {world} ranks, {V} views per rank per step")),
              "views_per_gpu": V, "gaussians": N, "pairs_per_view": pairs_view, "pairs_per_view_after_tile_culling": pairs_proc,
              "l2": "inputs larger than L2 (236 MB parameters + views x 41 MB upstream gradients per step vs 50 MB L2); no flush needed",
              "parallelism": f"views sharded over {world} rank(s), Gaussians replicated" + (
                  f", one NCCL all-reduce of the 248 MB packed gradient buffer per step, issued from inside the step in "
                  f"{args.ar_chunks} Gaussian-range chunk(s) (gs_b200_set_grad_sink)" if world > 1 else "")}
    if weak:
        config["weak_8_views_per_rank"] = weak
    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3),
        "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
        "data": "synthetic", "config": config,
        "clocks": clk, "e2e": e2e, "gpu_launches": launches, "roofline": roofline, "cpu_baseline": cpu,
    }
    if world > 1:
        dist.destroy_process_group()
    return line


# ======================================================================================
# Instant-NGP (config 3): two L=16 hash grids (base 16 -> finest 512), 1920x1080 rays, fwd+bwd
# ======================================================================================
NGP_METRIC, NGP_UNIT = "Msamples/sec fwd+bwd (Instant-NGP ray-march)", "Msamples/s"


def ngp_cpu_sample_run(steps, warmup, hw=(36, 64), L=16):
    """oracle/ngp_oracle.py: march + visibility pass + 2x encode + 2x MLP + weights + accumulate, fwd+bwd (torch autograd)
    on a bounded ray set — the call sequence of InstantNGP.render_nerf (Instant_NGP.py:101-156)."""
    import numpy as np
    import torch
    from oracle import gs_oracle as GO
    from oracle import ngp_oracle as NO
    cores = min(os.cpu_count() or 1, 16)
    torch.set_num_threads(cores)
    H, W = hw
    torch.manual_seed(0)
    pls = float(np.exp2(np.log2(512 / 16) / (L - 1)))
    offs = NO.grid_offsets(num_levels=L, per_level_scale=pls)
    emb_d = (torch.rand(int(offs[-1]), 2) * 2e-4 - 1e-4).requires_grad_(True)
    emb_c = (torch.rand(int(offs[-1]), 2) * 2e-4 - 1e-4).requires_grad_(True)
    w_d = [(torch.randn(32, 2 * L) * 0.1).requires_grad_(True), (torch.randn(1, 32) * 0.1).requires_grad_(True)]
    w_c = [(torch.randn(32, 2 * L) * 0.1).requires_grad_(True), (torch.randn(3, 32) * 0.1).requires_grad_(True)]
    g = (torch.arange(64).float() + 0.5) / 64 * 2 - 1
    x, y, z = torch.meshgrid(g, g, g, indexing="ij")
    binary = (x * x + y * y + z * z) < 0.25
    aabb = torch.tensor([-1.0, -1, -1, 1, 1, 1])
    ro, rd = NO.get_rays(GO.orbit_camera(0, 30, 1.75), H, W, 49.1)
    ro, rd = ro.reshape(-1, 3), rd.reshape(-1, 3)
    gimg = torch.rand(H * W, 3)
    leaves = [emb_d, emb_c] + w_d + w_c
    enc = lambda p, e: NO.grid_encode(p, e, offs, num_levels=L, per_level_scale=pls)
    mlp = lambda f, w: torch.relu(f @ w[0].T) @ w[1].T

    def step():
        with torch.no_grad():
            ri, t0, t1 = NO.march(ro, rd, binary, aabb, 0.01, 100.0, 5e-3, t_offset=torch.rand(H * W) * 5e-3)
            sig0 = NO.trunc_exp(mlp(enc(ro[ri] + rd[ri] * (t0 + t1)[:, None] / 2.0, emb_d), w_d)).squeeze(-1)
            keep = NO.visibility_mask(t0, t1, sig0, ri, H * W)
            ri, t0, t1 = ri[keep], t0[keep], t1[keep]
        p = ro[ri] + rd[ri] * (t0 + t1)[:, None] / 2.0
        sig = NO.trunc_exp(mlp(enc(p, emb_d), w_d)).squeeze(-1)
        rgb = torch.sigmoid(mlp(enc(p, emb_c), w_c))
        w, _, _ = NO.render_weight_from_density(t0, t1, sig, ri, H * W)
        col = NO.accumulate_along_rays(w, rgb, ri, H * W)
        alp = NO.accumulate_along_rays(w, None, ri, H * W)
        ((col + (1 - alp)) * gimg).sum().backward()
        for q in leaves:
            q.grad = None
        return int(ri.numel())
    S = 0
    for _ in range(warmup):
        S = step()
    t0_ = time.perf_counter()
    for _ in range(steps):
        S = step()
    dt = (time.perf_counter() - t0_) / max(steps, 1)
    desc = (f"oracle/ngp_oracle.py fwd+bwd, {W}x{H} rays ({S} samples), 2 x L={L} grids (finest 512), torch {cores} threads "
            f"(host has {os.cpu_count()} cores), {warmup} warm-up + {steps} timed steps")
    return S / dt / 1e6, dt * 1e3, cores, desc


def run_ngp(args):
    import ctypes as C
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench.py (impl b200) needs a CUDA device; there is no CPU fallback")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(0)
    import nerfacc
    from kiui.gridencoder import GridEncoder
    from kiui.nn import MLP, trunc_exp
    from gs_b200 import _lib, camera
    H, W, L = args.height, args.width, 16
    torch.manual_seed(0)
    enc_d, enc_c = GridEncoder(num_levels=L, desired_resolution=512).to(dev), GridEncoder(num_levels=L, desired_resolution=512).to(dev)
    mlp_d, mlp_c = MLP(2 * L, 1, 32, 2, bias=False).to(dev), MLP(2 * L, 3, 32, 2, bias=False).to(dev)
    est = nerfacc.OccGridEstimator(roi_aabb=torch.tensor([-1.0, -1, -1, 1, 1, 1], device=dev), resolution=64, levels=1).to(dev)
    g = (torch.arange(64, device=dev).float() + 0.5) / 64 * 2 - 1
    x, y, z = torch.meshgrid(g, g, g, indexing="ij")
    est.binaries = ((x * x + y * y + z * z) < 0.25)[None]; est.occs = est.binaries.flatten().float()
    fovy = 49.1
    modules = {"enc_d": enc_d, "enc_c": enc_c, "mlp_d": mlp_d, "mlp_c": mlp_c}
    params = [q for mod in modules.values() for q in mod.parameters()]

    def rays_of(pose):        # InstantNGP.get_rays (Instant_NGP.py:37-70)
        xs_, ys_ = torch.meshgrid(torch.arange(W, device=dev), torch.arange(H, device=dev), indexing="xy")
        focal = H * 0.5 / np.tan(0.5 * np.deg2rad(fovy))
        dirs = torch.nn.functional.pad(torch.stack([(xs_.flatten() - W * 0.5 + 0.5) / focal, (ys_.flatten() - H * 0.5 + 0.5) / focal * -1.0], -1), (0, 1), value=-1.0)
        rd = dirs @ pose[:3, :3].T
        rd = rd / rd.norm(dim=-1, keepdim=True)
        return pose[:3, 3][None].expand_as(rd).contiguous(), rd
    pose_host = torch.from_numpy(camera.orbit_camera(0, 30, 1.75)).pin_memory()
    ro, rd = rays_of(pose_host.to(dev))
    gimg = torch.rand(H * W, 3, device=dev)
    gimg_host = gimg.cpu().pin_memory()
    out_host = torch.empty(H * W, 3).pin_memory()
    loss_host = torch.empty(1).pin_memory()
    st = {}

    def render(ro, rd, target):       # InstantNGP.render_nerf (Instant_NGP.py:101-156) + an image loss, as fit_nerf
        def sigma_fn(t0, t1, ri):
            return trunc_exp(mlp_d(enc_d(ro[ri] + rd[ri] * (t0 + t1)[:, None] / 2.0))).squeeze(-1)
        with torch.no_grad():
            ri, t0, t1 = est.sampling(ro, rd, sigma_fn=sigma_fn, near_plane=0.01, far_plane=100, render_step_size=5e-3, stratified=True, cone_angle=0)
        p = ro[ri] + rd[ri] * (t0 + t1)[:, None] / 2.0
        sig = trunc_exp(mlp_d(enc_d(p))).squeeze(-1)
        rgb = torch.sigmoid(mlp_c(enc_c(p)))
        w, _, _ = nerfacc.render_weight_from_density(t0, t1, sig, ray_indices=ri, n_rays=H * W)
        col = nerfacc.accumulate_along_rays(w, values=rgb, ray_indices=ri, n_rays=H * W)
        alp = nerfacc.accumulate_along_rays(w, values=None, ray_indices=ri, n_rays=H * W)
        img = col + (1 - alp)
        loss = (img * target).sum()
        loss.backward()
        enc_d.grad_total_variation(1e-8)
        st["grads"] = {f"grad_{m}_{n}".replace(".", "_"): q.grad for m, mod in modules.items()
                      for n, q in mod.named_parameters() if q.grad is not None}
        for q in params:
            q.grad = None
        st["samples"], st["p"], st["img"], st["loss"] = ri.numel(), p.detach(), img.detach(), loss.detach()
        return img, loss

    def step():
        render(ro, rd, gimg)

    def e2e_step():               # pose + target image from pinned host memory, rendered image + loss back
        pose = pose_host.to(dev, non_blocking=True)
        target = gimg_host.to(dev, non_blocking=True)
        r_o, r_d = rays_of(pose)
        img, loss = render(r_o, r_d, target)
        out_host.copy_(img.detach(), non_blocking=True)
        loss_host.copy_(loss.detach().reshape(1), non_blocking=True)
        torch.cuda.synchronize()
    l0 = _lib.lib.gs_b200_launch_count()
    clocks = Clocks(0)
    ms_step = timed(step, args.steps, max(args.warmup, 3))
    clk = clocks.stop()
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, {"image": st["img"].view(H, W, 3), "loss": st["loss"].reshape(1),
                                         "samples": torch.tensor([st["samples"]], dtype=torch.int64), **st["grads"]})
    S = st["samples"]
    value = S / ms_step / 1e3
    e2e = None
    if not args.no_e2e:
        ms_e = timed(e2e_step, args.steps, 3)
        e2e = {"value": S / ms_e / 1e3, "unit": NGP_UNIT, "ms_per_step": ms_e, "h2d_bytes_per_step": 64 + H * W * 12,
               "d2h_bytes_per_step": H * W * 12 + 4, "api": "nerfacc / kiui.gridencoder / kiui.nn shims (InstantNGP.render_nerf call sequence)"}
    # ---- dominant kernels, timed alone on the samples of the last step (C ABI, CUDA events on the launching stream)
    p = st["p"].contiguous()
    emb = enc_d.embeddings.detach()
    feats = torch.empty(S, 2 * L, device=dev)
    gfeat = torch.rand(S, 2 * L, device=dev)
    gemb = torch.zeros_like(emb)
    offs = C.c_void_p(enc_d._offsets_np.ctypes.data)
    P_ = lambda t: C.c_void_p(t.data_ptr())
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def k_fwd():
        _lib.check(_lib.lib.ngp_b200_grid_encode_fwd(P_(p), S, P_(emb), offs, L, 1.0, float(enc_d.per_level_scale), int(enc_d.base_resolution), P_(feats), stream))

    def k_bwd():
        _lib.check(_lib.lib.ngp_b200_grid_encode_bwd(P_(p), S, offs, L, 1.0, float(enc_d.per_level_scale), int(enc_d.base_resolution), P_(gfeat), P_(gemb), stream))
    ms_f, ms_b = timed(k_fwd, 5, 2), timed(k_bwd, 5, 2)
    peak, peak_src = peaks()
    gather = S * L * 8 * 2 * 4                      # SURVEY 8d path B: L levels x 8 corners x F=2 x 4 B per sample and encoder
    per_enc = gather + S * (12 + 2 * L * 4)         # + position read + feature row written (fwd) / read (bwd)
    dom, t_dom = ("grid_encode_bwd", ms_b) if ms_b >= ms_f else ("grid_encode_fwd", ms_f)
    ach = per_enc / (t_dom * 1e-3) / 1e9
    table_mib = emb.numel() * 4 / 2 ** 20
    roofline = {"bound": "hbm", "kernel": dom, "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak, "traffic": traffic_of(dom),
                "peak_source": peak_src, "algorithmic_bytes_per_launch": per_enc, "avg_launch_ms": t_dom,
                "kernel_ms": {"grid_encode_fwd": ms_f, "grid_encode_bwd": ms_b},
                "note": f"one encoder, {S} samples; the gathers / scatters are random accesses into a {table_mib:.0f} MiB table "
                        "(H100 L2: 50 MB), so part of the traffic is served by L2; the HBM fraction is reported as asked",
                "step_algorithmic_bytes": S * (2 * L * 8 * 2 * 4 + 12 + 4 + 8) * 2}
    cpu = None
    if not args.no_cpu_baseline:
        v, ms_cpu, cores, desc = ngp_cpu_sample_run(3, 1)
        cpu = {"value": v, "unit": NGP_UNIT, "cores": cores, "kind": "port", "sample": desc, "ms_per_step": ms_cpu}
    return {
        "metric": NGP_METRIC, "value": value, "unit": NGP_UNIT, "n_gpus": 1, "steps": args.steps, "warmup": max(args.warmup, 3),
        "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": f"config 3: Instant-NGP render_nerf fwd+bwd, two L={L} hash grids (base 16 -> finest 512, T=2^19, F=2), "
                               f"two 32-wide MLPs, {W}x{H} rays, occupancy 64^3 (sphere r=0.5), step 5e-3, stratified, + TV gradient",
                   "rays": H * W, "samples_per_step": S, "Mrays_per_s": H * W / ms_step / 1e3,
                   "l2": "per-sample feature tensors (4 x S x 128 B) far larger than L2; no flush needed"},
        "clocks": clk, "e2e": e2e, "gpu_launches": int(_lib.lib.gs_b200_launch_count() - l0), "roofline": roofline, "cpu_baseline": cpu,
    }


def run_ngp_reference(args):
    v, ms, cores, desc = ngp_cpu_sample_run(args.steps, max(args.warmup, 0))
    return {"impl": "reference", "metric": NGP_METRIC, "value": v, "unit": NGP_UNIT, "n_gpus": args.gpus, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic", "config": {"workload": "config 3 (Instant-NGP), bounded CPU sample", "sample": desc},
            "cpu_baseline": {"value": v, "unit": NGP_UNIT, "cores": cores, "kind": "port", "sample": desc},
            "e2e": {"value": v, "unit": NGP_UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}, "gpu_launches": 0,
            "note": "nerfacc / kiui.gridencoder are un-vendored third-party CUDA packages, unavailable offline; this arm times the "
                    "pure-PyTorch CPU restatement (oracle/ngp_oracle.py)"}


# ======================================================================================
# mesh ops (config 4): rasterize -> antialias -> interpolate -> texture -> antialias, fwd+bwd, 8 views 1080p
# ======================================================================================
MESH_METRIC, MESH_UNIT = "Mtri*views/sec fwd+bwd (rasterize/interpolate/texture/antialias)", "Mtri*views/s"


def uv_sphere(n_lon, n_lat, radius=0.5):
    """Latitude-longitude sphere: 2 * n_lon * n_lat triangles (the polar caps are cut at 1e-3 rad, so none is degenerate),
    seam duplicated so uv is continuous.  Returns (verts [V,3] f32, faces [F,3] i32, uv [V,2] f32)."""
    import numpy as np
    import torch
    th = np.linspace(1e-3, np.pi - 1e-3, n_lat + 1)
    ph = np.linspace(0, 2 * np.pi, n_lon + 1)
    T, P = np.meshgrid(th, ph, indexing="ij")
    v = np.stack([radius * np.sin(T) * np.cos(P), radius * np.cos(T), radius * np.sin(T) * np.sin(P)], -1).reshape(-1, 3)
    uv = np.stack([P / (2 * np.pi), T / np.pi], -1).reshape(-1, 2)
    i, j = np.meshgrid(np.arange(n_lat), np.arange(n_lon), indexing="ij")
    a = (i * (n_lon + 1) + j).reshape(-1); b = a + 1; c = a + (n_lon + 1); d = c + 1
    f = np.concatenate([np.stack([a, c, b], -1), np.stack([b, c, d], -1)], 0)
    return torch.from_numpy(v.astype(np.float32)), torch.from_numpy(f.astype(np.int32)), torch.from_numpy(uv.astype(np.float32))


def mesh_cpu_sample_run(steps, warmup, n_lon=32, n_lat=32, hw=(128, 128)):
    import torch
    from oracle import dr_oracle as D
    from oracle import gs_oracle as GO
    cores = min(os.cpu_count() or 1, 16)
    torch.set_num_threads(cores)
    H, W = hw
    v, f, uv = uv_sphere(n_lon, n_lat)
    proj = D.gl_perspective(49.1, W / H)
    pos = D.clip_positions(v, GO.orbit_camera(0, 30.0, 1.75), proj).requires_grad_(True)
    tex = torch.rand(1, 64, 64, 3, requires_grad=True)
    gi = torch.rand(1, H, W, 3)

    def step():
        rast, db = D.rasterize(pos, f, (H, W))
        alpha = D.antialias(torch.clamp(rast[..., -1:], 0, 1), rast, pos, f)
        texc, texc_db = D.interpolate(uv[None], rast, f, rast_db=db, diff_attrs="all")
        alb = D.antialias(D.texture(tex, texc, filter_mode="linear"), rast, pos, f)
        ((alpha * alb) * gi).sum().backward()
        pos.grad = None; tex.grad = None
    for _ in range(warmup):
        step()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    dt = (time.perf_counter() - t0) / max(steps, 1)
    F = f.shape[0]
    desc = (f"oracle/dr_oracle.py rasterize/antialias/interpolate/texture/antialias fwd+bwd, {F} triangles, 1 view {W}x{H}, "
            f"torch {cores} threads (host has {os.cpu_count()} cores), {warmup} warm-up + {steps} timed steps")
    return F / dt / 1e6, dt * 1e3, cores, desc


def run_mesh(args):
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench.py (impl b200) needs a CUDA device; there is no CPU fallback")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(0)
    import nvdiffrast.torch as dr
    from gs_b200 import _lib
    from oracle import dr_oracle as D           # camera / projection helpers only (host side, outside the timed region)
    from oracle import gs_oracle as GO
    H, W, Vn = args.height, args.width, 8
    proj = torch.as_tensor(D.gl_perspective(49.1, W / H), dtype=torch.float32)
    mvps = torch.stack([proj @ torch.linalg.inv(torch.as_tensor(GO.orbit_camera(0, 45.0 * k, 1.75), dtype=torch.float32))
                        for k in range(Vn)])            # [8,4,4] clip <- object
    torch.manual_seed(0)
    gi = torch.rand(Vn, H, W, 3, device=dev)
    tex = torch.rand(1, 1024, 1024, 3, device=dev, requires_grad=True)
    ctx = dr.RasterizeCudaContext()
    last = {}                 # loss and gradients of the latest step()

    def make_step(n_side):
        v_host, f, uv = uv_sphere(n_side, n_side)
        f, uv = f.to(dev), uv.to(dev)
        vh = torch.cat([v_host, torch.ones(v_host.shape[0], 1)], 1).pin_memory()        # [V,4] homogeneous object-space vertices
        mv = mvps.pin_memory()
        gh = torch.empty(v_host.shape[0], 4).pin_memory()
        lh = torch.empty(1).pin_memory()

        def chain(pos, T):
            rast, db = T("rasterize", lambda: dr.rasterize(ctx, pos, f, (H, W)))
            alpha = T("antialias_alpha", lambda: dr.antialias(torch.clamp(rast[..., -1:], 0, 1).contiguous(), rast, pos, f))
            texc, texc_db = T("interpolate", lambda: dr.interpolate(uv[None], rast, f, rast_db=db, diff_attrs="all"))
            alb = T("texture", lambda: dr.texture(tex, texc, uv_da=texc_db, filter_mode="linear"))
            alb = T("antialias_color", lambda: dr.antialias(alb, rast, pos, f))
            loss = ((alpha * alb) * gi).sum()
            T("backward", lambda: loss.backward())
            return loss
        plain = lambda name, fn: fn()
        # DiffRastRenderer clip transform (diff_mesh_renderer.py:91-95)
        pos_dev = (vh.to(dev)[None] @ mvps.to(dev).transpose(1, 2)).contiguous().requires_grad_(True)

        def step():
            loss = chain(pos_dev, plain)
            last.update(loss=loss.detach(), grad_pos=pos_dev.grad, grad_tex=tex.grad)
            pos_dev.grad = None; tex.grad = None

        def e2e_step():      # vertices + view matrices from pinned host memory; loss and vertex gradient back
            vv = vh.to(dev, non_blocking=True).requires_grad_(True)
            mm = mv.to(dev, non_blocking=True)
            pos = (vv[None] @ mm.transpose(1, 2)).contiguous()
            loss = chain(pos, plain)
            gh.copy_(vv.grad, non_blocking=True); lh.copy_(loss.detach().reshape(1), non_blocking=True)
            tex.grad = None
            torch.cuda.synchronize()

        def prof_step(tm):
            def T(name, fn):
                a, b = torch.cuda.Event(True), torch.cuda.Event(True)
                a.record(); r = fn(); b.record(); tm.append((name, a, b)); return r
            chain(pos_dev, T)
            pos_dev.grad = None; tex.grad = None
        return dict(step=step, e2e=e2e_step, prof=prof_step, F=int(f.shape[0]), nV=int(v_host.shape[0]),
                    h2d=vh.numel() * 4 + mv.numel() * 4, d2h=gh.numel() * 4 + 4)

    m = make_step(int(round(math.sqrt(args.triangles / 2))))
    F, nV = m["F"], m["nV"]
    l0 = _lib.lib.gs_b200_launch_count()
    clocks = Clocks(0)
    ms_step = timed(m["step"], args.steps, max(args.warmup, 3))
    clk = clocks.stop()
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, {"loss": last["loss"].reshape(1), "grad_pos": last["grad_pos"], "grad_tex": last["grad_tex"]})
    value = F * Vn / ms_step / 1e3
    e2e = None
    if not args.no_e2e:
        ms_e = timed(m["e2e"], args.steps, 3)
        e2e = {"value": F * Vn / ms_e / 1e3, "unit": MESH_UNIT, "ms_per_step": ms_e, "h2d_bytes_per_step": m["h2d"], "d2h_bytes_per_step": m["d2h"],
               "api": "nvdiffrast.torch shim (DiffRastRenderer.render op chain)"}
    for _ in range(2):
        tm = []
        m["prof"](tm); torch.cuda.synchronize()
    op_ms = {n: a.elapsed_time(b) for n, a, b in tm}
    P = H * W
    # SURVEY 8d path C per view; one op call handles all 8 views
    alg = {"rasterize": Vn * (F * 12 + nV * 16 + P * 32), "interpolate": Vn * (P * (16 + 4 * 2) + P * 32), "texture": Vn * P * (8 + 12 + 12),
           "antialias_alpha": Vn * P * (2 * 4 * 1 + 16), "antialias_color": Vn * P * (2 * 4 * 3 + 16)}
    dom = max(alg, key=lambda k: op_ms[k])
    peak, peak_src = peaks()
    ach = alg[dom] / (op_ms[dom] * 1e-3) / 1e9
    roofline = {"bound": "hbm", "kernel": dom, "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak, "traffic": traffic_of("mesh_" + dom),
                "peak_source": peak_src, "algorithmic_bytes_per_launch": alg[dom], "avg_launch_ms": op_ms[dom], "op_ms": op_ms,
                "note": "op-level CUDA events on torch's current stream (each op = its kernels for all 8 views); the forward ops are the "
                        "candidates for the dominant kernel, the autograd backward as a whole is listed in op_ms",
                "step_algorithmic_bytes": sum(alg.values())}
    # the regime DiffMesh.training actually runs (diff_mesh.py:81-159): few, large triangles
    m2 = make_step(100)
    ms2 = timed(m2["step"], args.steps, 3)
    large = {"triangles": m2["F"], "ms_per_step": ms2, "value": m2["F"] * Vn / ms2 / 1e3, "unit": MESH_UNIT, "Mpixels_per_s": Vn * P / ms2 / 1e3}
    cpu = None
    if not args.no_cpu_baseline:
        vv, ms_cpu, cores, desc = mesh_cpu_sample_run(3, 1)
        cpu = {"value": vv, "unit": MESH_UNIT, "cores": cores, "kind": "port", "sample": desc, "ms_per_step": ms_cpu}
    return {
        "metric": MESH_METRIC, "value": value, "unit": MESH_UNIT, "n_gpus": 1, "steps": args.steps, "warmup": max(args.warmup, 3),
        "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": f"config 4: {F}-triangle lat-long sphere, {Vn} views {W}x{H}: rasterize -> antialias(alpha) -> interpolate(uv, db) -> "
                               "texture(1024^2, linear) -> antialias(colour), forward + backward",
                   "triangles": F, "vertices": nV, "Mpixels_per_s": Vn * P / ms_step / 1e3, "large_triangle_case": large,
                   "l2": "per-view buffers (8 x 33 MB rast + db, 8 x 25 MB colour) larger than L2; no flush needed"},
        "clocks": clk, "e2e": e2e, "gpu_launches": int(_lib.lib.gs_b200_launch_count() - l0), "roofline": roofline, "cpu_baseline": cpu,
    }


def run_mesh_reference(args):
    v, ms, cores, desc = mesh_cpu_sample_run(args.steps, max(args.warmup, 0))
    return {"impl": "reference", "metric": MESH_METRIC, "value": v, "unit": MESH_UNIT, "n_gpus": args.gpus, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic", "config": {"workload": "config 4 (mesh ops), bounded CPU sample", "sample": desc},
            "cpu_baseline": {"value": v, "unit": MESH_UNIT, "cores": cores, "kind": "port", "sample": desc},
            "e2e": {"value": v, "unit": MESH_UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}, "gpu_launches": 0,
            "note": "nvdiffrast is an un-vendored third-party CUDA package, unavailable offline; this arm times the pure-PyTorch CPU "
                    "restatement (oracle/dr_oracle.py)"}


if __name__ == "__main__":
    a = parse()
    rank = int(os.environ.get("RANK", "0"))
    if a.impl == "reference":
        if rank == 0:      # the CPU arm runs on rank 0 alone; other ranks exit 0 without work
            line = {"gs": run_gs_reference, "ngp": run_ngp_reference, "mesh": run_mesh_reference}[a.workload](a)
            print(json.dumps(line))
    else:
        if a.workload != "gs" and int(os.environ.get("WORLD_SIZE", "1")) > 1:
            raise SystemExit("--workload ngp/mesh are single-GPU lines (N>1 would run replicas only)")
        line = {"gs": run_gs, "ngp": run_ngp, "mesh": run_mesh}[a.workload](a)
        if line is not None:
            print(json.dumps(line))
