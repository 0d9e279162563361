#!/bin/bash
# compute-sanitizer over the kernels added late in round 1 (tile culling, in-pipeline loss, grid kNN, run-reduced
# hash-grid scatter, flat Adam); run on a GPU machine.
set -o pipefail
cd "$(dirname "$0")/.."
cat > /tmp/new_case.py <<'PY'
import sys, os
ROOT = os.getcwd(); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "comfyui-3d-pack_b200"))
import numpy as np, torch
from gs_b200 import camera, optim_step, synthetic, trainer, rasterizer as R
dev = torch.device("cuda:0")
W = H = 176
tr = trainer.GaussianTrainer(trainer.TrainParams(num_pts=9000, sh_degree=1, density_start_iter=10 ** 9), device=dev, seed=1)   # 9000 > 8192: grid kNN
views = camera.orbit_views(3, W, H)
ref = torch.rand(3, 3, H, W, device=dev); mask = (torch.rand(3, 1, H, W, device=dev) > 0.5).float()
print("train loss", tr.train_step(views, W, H, ref, mask))                       # culled lists, loss kernels, Adam
rad = torch.empty(3, tr.N, dtype=torch.int32, device=dev)
img = tr.render_views(views, W, H, radii=rad); print("render", float(img.sum()))
l, dl = optim_step.image_loss(img[0].contiguous(), ref[0].contiguous(), mask[0].contiguous(), 0.2, 3.0, 1.0); print("loss", float(l))
R.set_tile_culling(2)
cloud = synthetic.make_cloud("D1", 3000, 1, seed=0, device=dev)
leaves = {k: v.clone().requires_grad_(True) for k, v in cloud.items()}
t = lambda a: torch.from_numpy(a).to(dev)
rs = R.GaussianRasterizationSettings(H, W, float(views[0, 38]), float(views[0, 39]), t(views[0, 35:38].copy()), 1.0, t(views[0, :16].copy()).view(4, 4),
                                    t(views[0, 16:32].copy()).view(4, 4), 1, t(views[0, 32:35].copy()), False, False)
c, r, d, a = R.GaussianRasterizer(rs)(means3D=leaves["means3D"], means2D=torch.zeros(3000, 3, device=dev, requires_grad=True), shs=leaves["shs"],
                                      opacities=leaves["opacities"], scales=leaves["scales"], rotations=leaves["rotations"])
(c.sum() + a.sum()).backward(); print("culled single-view grads", float(leaves["means3D"].grad.abs().sum()))
R.set_tile_culling(1)
from kiui.gridencoder import GridEncoder
enc = GridEncoder(num_levels=8).to(dev)
o = torch.rand(40, 3, device=dev) - 0.5; dd_ = torch.nn.functional.normalize(torch.randn(40, 3, device=dev), dim=1)
x = (o[:, None] + dd_[:, None] * torch.linspace(0, 0.5, 100, device=dev)[None, :, None]).reshape(-1, 3).clamp(-1, 1).contiguous()
out = enc(x); out.backward(torch.rand_like(out)); print("ngp grad", float(enc.embeddings.grad.abs().sum()))
torch.cuda.synchronize()
PY
timeout 1200 compute-sanitizer --tool memcheck --error-exitcode 9 --launch-timeout 0 python /tmp/new_case.py 2>&1 | tail -12
echo "memcheck rc=$?"

# Hunyuan3D's texture-bake rasterizer (cr_raster.cu): every queue of cr_large_kernel (thread, warp, CTA split and
# whole-face CTA), the depth prior, interpolate forward + backward; memcheck and racecheck
cat > /tmp/cr_case.py <<'PY'
import sys, os
ROOT = os.getcwd(); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "comfyui-3d-pack_b200")); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import custom_rasterizer as cr
from test_gpu_custom_rasterizer import large_faces, screen_filling, sphere, view_pos
dev = torch.device("cuda:0")
xyz, tri, _ = sphere(2000, seed=1)
fi, b = cr.rasterize(view_pos(xyz, (96, 80)).to(dev)[None], tri.to(dev), (96, 80))
pos, t = screen_filling()
cr.rasterize(pos.to(dev)[None], t.to(dev), (128, 128), torch.rand(128, 128, device=dev) * 2 - 1, 1)
pos, t, hw = large_faces(1800, (192, 256), 10)
cr.rasterize(pos.to(dev)[None], t.to(dev), hw)
col = torch.randn(1, xyz.shape[0], 3, device=dev, requires_grad=True)
bq = b.clone().requires_grad_(True)
cr.interpolate(col, fi.float(), bq, tri.to(dev)).sum().backward()
torch.cuda.synchronize(); print("cr ok", int((fi != 0).sum()), float(col.grad.abs().sum()))
PY
for tool in memcheck racecheck; do
  timeout 1200 compute-sanitizer --tool $tool --error-exitcode 9 --launch-timeout 0 python /tmp/cr_case.py 2>&1 | tail -6
  echo "cr $tool rc=$?"
done

# StableFast3D's texture baker (uv_bake.cu): every queue (thread, warp, CTA split, CTA whole-face, whole-texture), a
# region with res % 16 != 0, and interpolate with out-of-range ids; memcheck and racecheck
cat > /tmp/ub_case.py <<'PY'
import sys, os
ROOT = os.getcwd(); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "comfyui-3d-pack_b200"))
import numpy as np, torch
from gs_b200 import uv_bake
from oracle import uvbake_oracle as O
dev = torch.device("cuda:0")
t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
for name, (uv, faces, res) in {**O.queue_cases(0), "nonfinite": O.adversarial(0)["nonfinite"]}.items():
    out = torch.zeros(res, res, 4, device=dev)
    uv_bake.rasterize_into(t(uv), t(faces), out, res - 5, res - 9)
    bad = faces.copy(); bad[::5, 1] = -3
    uv_bake.interpolate_into(t(np.random.rand(uv.shape[0], 3).astype(np.float32)), out, t(bad), torch.zeros(res, res, 3, device=dev), res, res)
torch.cuda.synchronize(); print("ub ok")
PY
for tool in memcheck racecheck; do
  timeout 1200 compute-sanitizer --tool $tool --error-exitcode 9 --launch-timeout 0 python /tmp/ub_case.py 2>&1 | tail -6
  echo "ub $tool rc=$?"
done
