"""Attention forward (flash_attn drop-in, csrc/gs_attn.cu) on one GPU, at the TRELLIS / Stable3DGen / Hunyuan3D 1.0
shapes, head dim 64.

Shapes: fp16 sparse-structure flow self-attention (1 x 4096, H 16) and cross-attention to 1374 image tokens; SLat flow
self- and cross-attention on the 64^3 sphere shell of bench_spconv.py (12 536 rows, one sequence, H 16); the SLat
decoder's 8^3 windows on the same shell shifted by 4 (H 12); bf16 Hunyuan3D 1.0 self-attention (1 x 3079, H 16).
Per shape: time over CUDA events after warm-up, useful TFLOP/s = 4 d H sum(Lq Lk) / time and its share of the H100 SXM's
989 TFLOP/s dense fp16 / bf16 figure, the same inputs through torch's own FlashAttention-2
(torch.ops.aten._flash_attention_forward, varlen), the ratio of the two times, and the largest difference between the
two outputs relative to max |v|.  Prints one JSON line per shape, after a line with the card's name, power limit and
max SM clock (and writes the lines to --out when given).
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

from gs_b200 import attention as A  # noqa: E402
from oracle import spconv_oracle as SO  # noqa: E402

CTX = 1374        # DINOv2-L/14 with registers at 518 px: 37^2 patches + 5 tokens


def shell_windows(shift=4, window=8):
    """row counts of the shell's shifted 8^3 windows, in TRELLIS's windowed-attention order"""
    c = torch.from_numpy(SO.sphere_shell(64)).long()
    w = (c[:, 1:] + shift) // window
    nw = int(w.max()) + 1
    key = ((c[:, 0] * nw + w[:, 0]) * nw + w[:, 1]) * nw + w[:, 2]
    return torch.unique(key, return_counts=True)[1].tolist()


def shapes():
    n_shell = SO.sphere_shell(64).shape[0]
    return [("ss_flow_self", torch.float16, 16, [4096], [4096]),
            ("ss_flow_cross", torch.float16, 16, [4096], [CTX]),
            ("slat_flow_self", torch.float16, 16, [n_shell], [n_shell]),
            ("slat_flow_cross", torch.float16, 16, [n_shell], [CTX]),
            ("slat_dec_swin", torch.float16, 12, shell_windows(), None),
            ("hunyuan_self_bf16", torch.bfloat16, 16, [3079], [3079])]


def cu(lens, dev):
    c = [0]
    for n in lens:
        c.append(c[-1] + n)
    return torch.tensor(c, dtype=torch.int32, device=dev)


def timed(fn, reps):
    for _ in range(3):
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
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_attention needs a GPU"
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    lines = [{"gpu": smi}]
    print(json.dumps(lines[0]), flush=True)
    for name, dtype, H, lq, lk in shapes():
        lk = lk or lq
        g = torch.Generator(device=dev).manual_seed(0)
        q = torch.randn(sum(lq), H, 64, device=dev, generator=g).to(dtype)
        k = torch.randn(sum(lk), H, 64, device=dev, generator=g).to(dtype)
        v = torch.randn(sum(lk), H, 64, device=dev, generator=g).to(dtype)
        cq, ck = cu(lq, dev), cu(lk, dev)
        mq, mk = max(lq), max(lk)
        with torch.inference_mode():
            ours = lambda: A.varlen(q, k, v, cq, ck, mq, mk)  # noqa: E731
            t = timed(ours, args.reps)
            out = ours()
            r = {"shape": name, "dtype": str(dtype).replace("torch.", ""), "H": H, "sequences": len(lq),
                 "rows_q": sum(lq), "rows_k": sum(lk), "ms": round(t, 4)}
            flops = 4.0 * 64 * H * sum(a * b for a, b in zip(lq, lk))
            r["tflops"] = round(flops / (t * 1e-3) / 1e12, 1)
            r["share_of_989"] = round(r["tflops"] / 989, 3)
            try:
                fa2 = lambda: torch.ops.aten._flash_attention_forward(  # noqa: E731
                    q, k, v, cq, ck, mq, mk, 0.0, False, False, scale=64 ** -0.5)[0]
                t2 = timed(fa2, args.reps)
                ref = fa2()
                r["torch_fa2_ms"] = round(t2, 4)
                r["speedup_vs_torch_fa2"] = round(t2 / t, 3)
                r["max_diff_vs_torch_fa2_rel_max_v"] = float((out.float() - ref.float()).abs().max()
                                                             / v.float().abs().max())
            except (RuntimeError, TypeError) as e:
                r["torch_fa2_error"] = str(e).splitlines()[0][:200]
        print(json.dumps(r), flush=True)
        lines.append(r)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
