"""Writes the fixture of tests/test_gpu_composite_combine.py (packed-gradient rows of its cancelling case) from the
library built in the tree this script lives in; needs a GPU.  The committed fixture was written by the composite
backward that issued one set of fp64 reds per (quadrant, splat), before the quadrant partials were combined in the CTA.

    python scripts/dev/make_combine_golden.py [OUT.npz]     (default tests/golden/composite_combine_grads.npz)
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "comfyui-3d-pack_b200"), ROOT]

import numpy as np  # noqa: E402
import torch  # noqa: E402
from test_gpu_composite_combine import CANCEL_GOLDEN, cancelling_case, rows_of  # noqa: E402

out = sys.argv[1] if len(sys.argv) > 1 else CANCEL_GOLDEN
rows = rows_of(cancelling_case(torch.device("cuda:0"))())
np.savez_compressed(out, rows=rows.numpy())
print("wrote", out, tuple(rows.shape))
