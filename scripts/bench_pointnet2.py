"""Times the pointnet2_ops drop-in (gs_b200.pointnet2) at its TriplaneGaussian callers' shapes against torch
formulations of the same operators on the same card, alternated in one process.

    python scripts/bench_pointnet2.py [--reps 20]

Cases:
  fps_16k      furthest_point_sample B=1, N=16384 -> 2048 (fps_subsample's size; the on-chip kernel) against a
               per-step torch loop (distance, minimum, argmax); reported per FPS step as well
  fps_64k      B=1, N=65536 -> 2048: beyond the on-chip capacity (16384 points), the global-memory kernel
  group_64     grouping_operation forward + backward at SkipTransformer's [1,64,4096] x 16 neighbours, against
               torch.gather of the expanded index and index_add_ (atomic) for the backward
  group_3      the same at [1,3,4096] x 16 (the positions)
  interp       three_interpolate forward + backward, [1,128,1024] -> 4096 points, against torch.gather + sum and
               index_add_
  ball         ball_query 16384 points, 2048 queries, radius 0.1, 32 samples (sample_and_group-like), against a torch
               cdist + mask + cumsum formulation
Prints the card's name and power limit, then one JSON line per case: ours and torch's milliseconds (the lower of two
alternated runs, each the median over reps of CUDA events).  Torch's index_add_ is atomic, so its fp32 bits depend on
the schedule; only the times compare."""
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


def alternated(ours, theirs, reps, theirs_reps=None):
    t = [[], []]
    for _ in range(2):
        t[0].append(timed(ours, reps))
        t[1].append(timed(theirs, theirs_reps or reps))
    return min(t[0]), min(t[1])


def torch_fps(xyz, npoint):
    B, N, _ = xyz.shape
    out = torch.zeros(B, npoint, dtype=torch.long, device=xyz.device)
    temp = torch.full((B, N), 1e10, device=xyz.device)
    last = torch.zeros(B, dtype=torch.long, device=xyz.device)
    ar = torch.arange(B, device=xyz.device)
    for s in range(1, npoint):
        d = ((xyz - xyz[ar, last][:, None]) ** 2).sum(-1)
        temp = torch.minimum(temp, d)
        last = temp.argmax(1)
        out[:, s] = last
    return out


def case_fps(U, g, N, reps):
    xyz = torch.rand(1, N, 3, generator=g, device="cuda") * 2 - 1
    npoint = 2048
    ours, theirs = alternated(lambda: U.furthest_point_sample(xyz, npoint), lambda: torch_fps(xyz, npoint), reps,
                              max(3, reps // 5))
    return {"ms": ours, "torch_ms": theirs, "us_per_step": 1e3 * ours / (npoint - 1),
            "torch_us_per_step": 1e3 * theirs / (npoint - 1)}


def case_group(U, g, C, reps):
    N, S = 4096, 16
    f = torch.randn(1, C, N, generator=g, device="cuda", requires_grad=True)
    idx = torch.randint(0, N, (1, N, S), generator=g, device="cuda", dtype=torch.int32)
    go = torch.randn(1, C, N, S, generator=g, device="cuda")
    il = idx.long().view(1, 1, N * S).expand(1, C, N * S)

    def ours():
        f.grad = None
        U.grouping_operation(f, idx).backward(go)

    def theirs():
        out = torch.gather(f.detach(), 2, il).view(1, C, N, S)
        gf = torch.zeros(1, C, N, device="cuda").index_add_(2, il[0, 0], go.view(1, C, N * S))
        return out, gf

    a, b = alternated(ours, theirs, reps)
    return {"ms": a, "torch_ms": b}


def case_interp(U, g, reps):
    B, C, m, n = 1, 128, 1024, 4096
    f = torch.randn(B, C, m, generator=g, device="cuda", requires_grad=True)
    idx = torch.randint(0, m, (B, n, 3), generator=g, device="cuda", dtype=torch.int32)
    w = torch.rand(B, n, 3, generator=g, device="cuda")
    go = torch.randn(B, C, n, generator=g, device="cuda")
    il = idx.long().view(B, 1, n * 3).expand(B, C, n * 3)

    def ours():
        f.grad = None
        U.three_interpolate(f, idx, w).backward(go)

    def theirs():
        out = (torch.gather(f.detach(), 2, il).view(B, C, n, 3) * w[:, None]).sum(-1)
        vals = (go[..., None] * w[:, None]).view(B, C, n * 3)
        gf = torch.zeros(B, C, m, device="cuda").index_add_(2, il[0, 0], vals)
        return out, gf

    a, b = alternated(ours, theirs, reps)
    return {"ms": a, "torch_ms": b}


def case_ball(U, g, reps):
    N, P, S, r = 16384, 2048, 32, 0.1
    xyz = torch.rand(1, N, 3, generator=g, device="cuda") * 2 - 1
    q = xyz[:, :P].contiguous()

    def theirs():
        d2 = torch.cdist(q, xyz) ** 2
        hit = d2 < r * r
        rank = hit.cumsum(-1) - 1
        keep = hit & (rank < S)
        out = torch.zeros(1, P, S, dtype=torch.long, device="cuda")
        pos = torch.nonzero(keep)
        out[pos[:, 0], pos[:, 1], rank[keep]] = pos[:, 2]
        return out

    a, b = alternated(lambda: U.ball_query(r, S, xyz, q), theirs, reps)
    return {"ms": a, "torch_ms": b}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_pointnet2 needs a GPU"
    from pointnet2_ops import pointnet2_utils as U
    print(json.dumps(card()))
    g = torch.Generator(device="cuda").manual_seed(0)
    cases = {"fps_16k": lambda: case_fps(U, g, 16384, args.reps), "fps_64k": lambda: case_fps(U, g, 65536, args.reps),
             "group_64": lambda: case_group(U, g, 64, args.reps), "group_3": lambda: case_group(U, g, 3, args.reps),
             "interp": lambda: case_interp(U, g, args.reps), "ball": lambda: case_ball(U, g, args.reps)}
    for name, fn in cases.items():
        r = fn()
        print(json.dumps({"case": name, **{k: round(v, 4) for k, v in r.items()}}), flush=True)


if __name__ == "__main__":
    main()
