"""Microbenchmark of the composite backward's fp64 gradient reds in two shapes: lanes = records (ten red instructions,
each to 32 different 96 B records) and lanes = (record, value) (3 records x 10 values per instruction).  See
red_pattern_bench.cu for what is timed.  Compiles the .cu into a temporary directory, runs it on cuda:0 and prints its
JSON lines after one line naming the card, its power limit and its clocks.

    python scripts/dev/red_pattern_bench.py [--ids 1000000] [--visits 4800000] [--launches 20] [--reps 3]
"""
import argparse
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ids", type=int, default=1_000_000)
    ap.add_argument("--visits", type=int, default=4_800_000, help="sets of ten reds per launch")
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "red_pattern_bench")
        subprocess.run([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                        os.path.join(HERE, "red_pattern_bench.cu"), "-o", exe], check=True)
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
        print('{"nvidia_smi": "%s"}' % (smi.stdout.strip() or smi.stderr.strip()), flush=True)
        rc = subprocess.run([exe, str(args.ids), str(args.visits), str(args.launches), str(args.reps)]).returncode
    sys.exit(rc)


if __name__ == "__main__":
    main()
