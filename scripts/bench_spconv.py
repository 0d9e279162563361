"""Submanifold sparse conv (spconv drop-in, csrc/sp_conv.cu) on one GPU, at the TRELLIS / Stable3DGen shapes in fp16.

Voxel sets: a sphere shell at 64^3 (surface-sparse, like TRELLIS's structured latents), subdivided to 128^3 and 256^3.
Per shape: map-build time, conv time over CUDA events, useful TFLOP/s = 2*Cin*Cout*(present neighbour pairs) / time
and its share of the H100 SXM's 989 TFLOP/s dense fp16 figure, and the speed-up over spconv's "native" algorithm
restated in torch (per offset: index_select + cuBLAS mm, accumulated in fixed offset order), with the largest
difference between the two outputs relative to the output scale.  Prints one JSON line per shape (and writes them
to --out when given).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "comfyui-3d-pack_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from gs_b200 import spconv as S  # noqa: E402
from oracle import spconv_oracle as O  # noqa: E402

# (name, resolution, Cin, Cout): SLat flow io blocks at 64^3 and 32^3 (the 32^3 set is the 64^3 shell downsampled),
# then the mesh decoder's two subdivision stages
SHAPES = [("flow_64_128_128", 64, 128, 128), ("flow_32_128_1024", 32, 128, 1024), ("flow_32_1024_1024", 32, 1024, 1024),
          ("flow_64_2048_128", 64, 2048, 128), ("flow_64_256_128", 64, 256, 128),
          ("dec_128_768_192", 128, 768, 192), ("dec_128_192_192", 128, 192, 192),
          ("dec_256_192_96", 256, 192, 96), ("dec_256_96_96", 256, 96, 96)]


def voxel_sets(dev):
    s64 = O.sphere_shell(64)
    s32 = torch.unique(torch.from_numpy(s64) // torch.tensor([1, 2, 2, 2], dtype=torch.int32), dim=0).numpy()
    s128 = O.subdivide(s64)
    s256 = O.subdivide(s128)
    return {r: torch.from_numpy(a).to(dev) for r, a in ((32, s32), (64, s64), (128, s128), (256, s256))}


def native(x, w, b, nbr):
    """spconv's native algorithm: per offset gather + mm, added in offset order"""
    out = b.expand(x.shape[0], -1).clone()
    K3 = nbr.shape[1]
    wf = w.reshape(w.shape[0], K3, -1)
    for o in range(K3):
        col = nbr[:, o]
        rows = torch.nonzero(col >= 0).squeeze(1)
        if rows.numel():
            out.index_add_(0, rows, x.index_select(0, col[rows].long()) @ wf[:, o, :].t())
    return out


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_spconv needs a GPU"
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi}))
    sets = voxel_sets(dev)
    rows = []
    for name, res, cin, cout in SHAPES:
        ind = sets[res]
        N = ind.shape[0]
        g = torch.Generator(device=dev).manual_seed(0)
        x = torch.randn(N, cin, device=dev, dtype=torch.float16, generator=g)
        w = (torch.rand(cout, 3, 3, 3, cin, device=dev, generator=g) * 2 - 1).half() / (27 * cin) ** 0.5
        b = (torch.rand(cout, device=dev, generator=g) * 2 - 1).half()
        spatial = (res, res, res)
        map_ms = timed(lambda: S.build_map(ind, spatial, 1, 3), args.reps)
        m = S.build_map(ind, spatial, 1, 3)
        with torch.inference_mode():
            conv_ms = timed(lambda: S.submconv3d(x, w, b, m), args.reps)
            out = S.submconv3d(x, w, b, m)
            nat_ms = timed(lambda: native(x, w, b, m.nbr), max(3, args.reps // 4))
            ref = native(x.float(), w.float(), b.float(), m.nbr)
        pairs = int((m.nbr >= 0).sum())
        tflops = 2.0 * cin * cout * pairs / (conv_ms * 1e-3) / 1e12
        scale = float(ref.abs().max())
        r = {"shape": name, "N": N, "Cin": cin, "Cout": cout, "pairs": pairs, "map_ms": round(map_ms, 4),
             "conv_ms": round(conv_ms, 4), "tflops": round(tflops, 1), "share_of_989": round(tflops / 989, 3),
             "native_ms": round(nat_ms, 4), "speedup_vs_native": round(nat_ms / conv_ms, 2),
             "max_abs_diff_vs_native_fp32": float((out.float() - ref).abs().max()), "out_scale": scale}
        print(json.dumps(r), flush=True)
        rows.append(r)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
