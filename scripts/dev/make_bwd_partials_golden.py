"""Writes the fixture of tests/test_gpu_bwd_partials.py (the gradients of its unequal-quadrant tile) from the library
built in the tree this script lives in; needs a GPU.  The committed fixture was written by the composite backward that
kept one partial block per ring stage (92.6 KB of shared memory, two CTAs per SM), before the block was shared.

    python scripts/dev/make_bwd_partials_golden.py [OUT.npz]     (default tests/golden/bwd_partials_grads.npz)
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "comfyui-3d-pack_b200"), ROOT]

import numpy as np  # noqa: E402
import torch  # noqa: E402
from test_gpu_bwd_partials import GOLDEN_FILE, run_case  # noqa: E402

out = sys.argv[1] if len(sys.argv) > 1 else GOLDEN_FILE
grads = run_case(torch.device("cuda:0"))
np.savez_compressed(out, **{k: v.numpy() for k, v in grads.items()})
print("wrote", out, {k: tuple(v.shape) for k, v in grads.items()})
