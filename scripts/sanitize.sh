#!/bin/bash
# compute-sanitizer passes over small GPU cases (memcheck + racecheck); run on a GPU machine.
set -o pipefail
cd "$(dirname "$0")/.."
T='tests/test_gpu_parity.py::test_onesweep_sort_matches_stable_sort tests/test_gpu_parity.py::test_empty_culled_and_offscreen_inputs tests/test_gpu_parity.py::test_colors_precomp_and_cov3d_precomp_paths tests/test_gpu_mesh.py::test_topology_matches_oracle tests/test_gpu_mesh.py::test_texture_wrap_clamp_and_gradients tests/test_gpu_ngp.py::test_weights_accumulate_forward_backward'
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 9 --launch-timeout 0 python -m pytest $T -m gpu -x -q -k "not 3000001 and not 1048576 and not 123457" 2>&1 | tail -15
echo "memcheck rc=$?"
cat > /tmp/race_case.py <<'PY'
import sys, os
ROOT = os.getcwd(); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "comfyui-3d-pack_b200"))
import torch
from gs_b200 import camera, optim_step, synthetic
dev = torch.device("cuda:0")
cloud = synthetic.make_cloud("D1", 3000, 1, seed=0, device=dev)
params = optim_step.PackedParams(cloud)
views = optim_step.ViewSet(camera.orbit_views(2, 96, 64), 96, 64, 1, dev)
dl = torch.rand(2, 5, 64, 96, device=dev)
optim_step.step_device_pipelined(params, views, dl); torch.cuda.synchronize(); print("grads", float(params.grads.abs().sum()))
PY
timeout 900 compute-sanitizer --tool racecheck --error-exitcode 9 python /tmp/race_case.py 2>&1 | tail -8
echo "racecheck rc=$?"
