"""Times the torch_scatter drop-in (gs_b200.scatter) at its callers' shapes against torch's own atomic,
non-deterministic scatter_add_ / scatter_reduce_ on the same inputs, alternated in one process.

    python scripts/bench_scatter.py [--reps 20]

Cases:
  flexicubes   FlexiCubes loss.py mesh_developable_reg's nine scatter_add calls (per corner: fp32 [F,9] dim=-2,
               fp32 [F], int32 [F], each into out) with random faces at a res-128 trainer mesh's size
               (F = 131072 faces, V = F/2), forward + backward of the fp32 ones
  unique3d     one MeshOptimizer.step's scatter_mean (fp32 [2E,3], index [2E,1], into out) and remesh's scatter_max
               calls (three int64 [2E] 1-D, one expanded int64 [E',4] with a full index) at V = 100k (E = 3V)
  triplane     TriplaneGaussian pointnet.py at its configured size: scatter_mean of c.permute [1,512,16384] into
               zeros [1,512,1024], then scatter_max with dim_size 1024, forward + backward
  worst        fp32 scatter_sum of E = 2^22 elements that all hit one slot: one thread folds them in order
Prints the card's name and power limit, then one JSON line per case: our milliseconds per case (the lower of two
alternated runs, each the median over reps of CUDA events around work that includes the one host read per call),
torch's, and the compulsory bytes (src and the distinct index elements read once, out read and written once) over
our time.  Torch's numbers are for its atomic kernels, whose fp32 bits depend on the schedule; its mean counts are
not torch_scatter's, so only times compare."""
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


def case_flexicubes(ts, g):
    F, V = 131072, 65536
    tris = torch.randint(0, V, (F, 3), generator=g, device="cuda")
    contrib = torch.randn(F, 9, generator=g, device="cuda").requires_grad_(True)
    area = torch.rand(F, generator=g, device="cuda").requires_grad_(True)
    ones = torch.ones(F, dtype=torch.int32, device="cuda")

    def ours():
        cov, va = torch.zeros(V, 9, device="cuda"), torch.zeros(V, device="cuda")
        deg = torch.zeros(V, dtype=torch.int32, device="cuda")
        for c in range(3):
            cov = ts.scatter_add(contrib, tris[:, c], dim=-2, out=cov)
            va = ts.scatter_add(area, tris[:, c], dim=-1, out=va)
            deg = ts.scatter_add(ones, tris[:, c], dim=-1, out=deg)
        (cov.sum() + va.sum()).backward()

    def theirs():
        cov, va = torch.zeros(V, 9, device="cuda"), torch.zeros(V, device="cuda")
        deg = torch.zeros(V, dtype=torch.int32, device="cuda")
        for c in range(3):
            cov = cov.scatter_add(0, tris[:, c, None].expand(F, 9), contrib)
            va = va.scatter_add(0, tris[:, c], area)
            deg = deg.scatter_add(0, tris[:, c], ones)
        (cov.sum() + va.sum()).backward()

    fwd = 3 * (F * 9 * 4 + F * 8 + V * 9 * 8 + F * 4 + F * 8 + V * 8 + F * 4 + F * 8 + V * 8)
    bwd = 3 * (F * 9 * 4 + F * 8 + F * 4 + F * 8)
    return ours, theirs, fwd + bwd


def case_unique3d(ts, g):
    V = 100000
    E = 3 * V
    edges = torch.randint(0, V, (E, 2), generator=g, device="cuda")
    smooth = torch.randn(V, 3, generator=g, device="cuda")
    rank = torch.randint(0, 2 ** 40, (E,), generator=g, device="cuda")
    nb = torch.randint(0, V, (E, 4), generator=g, device="cuda")

    def ours():
        es = smooth[edges]
        ns = torch.zeros_like(smooth)
        ts.scatter_mean(src=es.flip(dims=[1]).reshape(E * 2, -1), index=edges.reshape(E * 2, 1), dim=0, out=ns)
        vr = torch.zeros(V, dtype=torch.int64, device="cuda")
        for _ in range(3):
            ts.scatter_max(src=rank[:, None].expand(-1, 2).reshape(-1), index=edges.reshape(-1), dim=0, out=vr)
        ts.scatter_max(src=rank[:, None].expand(-1, 4), index=nb, dim=0, out=torch.zeros(V, 4, dtype=torch.int64, device="cuda"))

    def theirs():
        es = smooth[edges]
        ns = torch.zeros_like(smooth)
        ns.scatter_reduce_(0, edges.reshape(E * 2, 1).expand(-1, 3), es.flip(dims=[1]).reshape(E * 2, -1), "mean",
                           include_self=False)
        vr = torch.zeros(V, dtype=torch.int64, device="cuda")
        for _ in range(3):
            vr.scatter_reduce_(0, edges.reshape(-1), rank[:, None].expand(-1, 2).reshape(-1), "amax")
        torch.zeros(V, 4, dtype=torch.int64, device="cuda").scatter_reduce_(0, nb, rank[:, None].expand(-1, 4), "amax")

    b = 2 * E * 3 * 4 + 2 * E * 8 + V * 3 * 8 + 3 * (2 * E * 8 * 2 + V * 8 * 2) + (E * 8 + E * 4 * 8 + V * 4 * 8 * 2)
    return ours, theirs, b


def case_triplane(ts, g):
    T, C, P = 16384, 512, 1024
    c = torch.randn(1, T, C, generator=g, device="cuda").requires_grad_(True)
    index = torch.randint(0, P, (1, 1, T), generator=g, device="cuda")

    def ours():
        m = ts.scatter_mean(c.permute(0, 2, 1), index, out=c.new_zeros(1, C, P))
        x = ts.scatter_max(c.permute(0, 2, 1), index, dim_size=P)[0]
        (m.sum() + x.sum()).backward()

    def theirs():
        ix = index.expand(1, C, T)
        m = c.new_zeros(1, C, P).scatter_reduce(2, ix, c.permute(0, 2, 1), "mean", include_self=False)
        x = c.new_zeros(1, C, P).scatter_reduce(2, ix, c.permute(0, 2, 1), "amax", include_self=False)
        (m.sum() + x.sum()).backward()

    b = 2 * (T * C * 4 + T * 8 + C * P * 4 * 2) + 2 * (T * C * 4 + C * P * 4)
    return ours, theirs, b


def case_worst(ts, g):
    E = 2 ** 22
    src = torch.randn(E, generator=g, device="cuda")
    index = torch.zeros(E, dtype=torch.int64, device="cuda")

    def ours():
        ts.scatter_sum(src, index, dim=0)

    def theirs():
        torch.zeros(1, device="cuda").scatter_add_(0, index, src)

    return ours, theirs, E * 4 + E * 8 + 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_scatter needs a CUDA device"
    import torch_scatter as ts
    print(json.dumps({"card": card()}))
    for name, make in (("flexicubes", case_flexicubes), ("unique3d", case_unique3d), ("triplane", case_triplane),
                       ("worst", case_worst)):
        g = torch.Generator(device="cuda").manual_seed(0)
        ours, theirs, nbytes = make(ts, g)
        t_ours, t_torch = [], []
        for _ in range(2):                                   # alternate the two within the run
            t_ours.append(timed(ours, a.reps))
            t_torch.append(timed(theirs, a.reps))
        mo, mt = min(t_ours), min(t_torch)
        print(json.dumps({"case": name, "ours_ms": round(mo, 4), "torch_atomic_ms": round(mt, 4),
                          "ours_ms_runs": [round(x, 4) for x in t_ours], "torch_ms_runs": [round(x, 4) for x in t_torch],
                          "compulsory_bytes": nbytes, "ours_GBps": round(nbytes / mo / 1e6, 1)}))


if __name__ == "__main__":
    main()
