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

# pointnet2_ops (pn2_ops.cu): FPS on-chip and global-memory kernels, ball query, three-NN, gather / grouping and
# three-interpolate forward and backward, with out-of-range indices; memcheck and racecheck
cat > /tmp/pn2_case.py <<'PY'
import sys, os
ROOT = os.getcwd(); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "comfyui-3d-pack_b200"))
import torch
from pointnet2_ops import pointnet2_utils as U
dev = torch.device("cuda:0")
g = torch.Generator(device=dev).manual_seed(0)
for N in (1000, 5000, 16384, 17000):
    xyz = torch.rand(2, N, 3, generator=g, device=dev) * 2 - 1
    idx = U.furthest_point_sample(xyz, 64)
print("fps", int(idx.sum()))
xyz = torch.rand(1, 3000, 3, generator=g, device=dev)
print("ball", int(U.ball_query(0.2, 32, xyz, xyz[:, :100].contiguous()).sum()))
d, i = U.three_nn(xyz, xyz[:, :50].contiguous())
f = torch.randn(1, 8, 3000, device=dev, requires_grad=True)
bad = torch.randint(-5, 3005, (1, 200, 16), generator=g, device=dev, dtype=torch.int32)
U.grouping_operation(f, bad).sum().backward()
U.gather_operation(f, bad[:, :, 0].contiguous()).sum().backward()
fi = torch.randn(1, 8, 50, device=dev, requires_grad=True)
U.three_interpolate(fi, i, torch.rand(1, 3000, 3, device=dev)).sum().backward()
torch.cuda.synchronize(); print("pn2 ok", float(f.grad.abs().sum()), float(fi.grad.abs().sum()))
PY
for tool in memcheck racecheck; do
  timeout 1200 compute-sanitizer --tool $tool --error-exitcode 9 --launch-timeout 0 python /tmp/pn2_case.py 2>&1 | tail -6
  echo "pn2 $tool rc=$?"
done

# spconv (sp_conv.cu): neighbour map with duplicates and rows outside the grid, fp16 (vector and element-wise loads)
# and fp32 forward, dgrad with the duplicate fold, wgrad / dbias over several chunks; memcheck and racecheck
cat > /tmp/sp_case.py <<'PY'
import sys, os
ROOT = os.getcwd(); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "comfyui-3d-pack_b200"))
import torch
from gs_b200 import spconv as S
from oracle import spconv_oracle as O
dev = torch.device("cuda:0")
for name, ind, spatial, B in O.edge_sets():
    m = S.build_map(torch.from_numpy(ind).to(dev), spatial, B, 3)
    for dt, cin in ((torch.float16, 40), (torch.float16, 13), (torch.float32, 13)):
        x = torch.randn(len(ind), cin, device=dev, dtype=dt, requires_grad=True)
        w = torch.randn(24, 3, 3, 3, cin, device=dev, dtype=dt, requires_grad=True)
        b = torch.randn(24, device=dev, dtype=dt, requires_grad=True)
        S.submconv3d(x, w, b, m).float().sum().backward()
ind = torch.from_numpy(O.subdivide(O.sphere_shell(24))).to(dev)
x = torch.randn(len(ind), 16, device=dev, requires_grad=True)
w = torch.randn(16, 3, 3, 3, 16, device=dev, requires_grad=True)
S.submconv3d(x, w, None, S.build_map(ind, (48, 48, 48), 1, 3)).sum().backward()
torch.cuda.synchronize(); print("sp ok", float(w.grad.abs().sum()))
PY
for tool in memcheck racecheck; do
  timeout 1200 compute-sanitizer --tool $tool --error-exitcode 9 --launch-timeout 0 python /tmp/sp_case.py 2>&1 | tail -6
  echo "sp $tool rc=$?"
done

# point rasterizer and points_projection (pts_raster.cu): K = 1, 2 and 8, ragged clouds with an empty one, a shared
# camera, points behind and on the camera plane, the lift from strided features and its backward; memcheck and racecheck
cat > /tmp/pts_case.py <<'PY'
import sys, os
ROOT = os.getcwd(); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "comfyui-3d-pack_b200"))
import torch
from gs_b200 import points as P
dev = torch.device("cuda:0")
g = torch.Generator(device=dev).manual_seed(0)
R = torch.eye(3, device=dev)[None].repeat(3, 1, 1); T = torch.tensor([[0.0, 0.0, 2.0]], device=dev).repeat(3, 1)
Km = torch.tensor([[[30.0, 0, 40], [0, 30, 30], [0, 0, 1]]], device=dev).repeat(3, 1, 1)
cams = P.cameras_from_opencv_projection(R, T, Km, torch.tensor([[60, 80]] * 3, device=dev))
clouds = [torch.rand(900, 3, generator=g, device=dev) * 2 - 1, torch.zeros(0, 3, device=dev), torch.rand(50, 3, generator=g, device=dev) * 6 - 3]
for K in (1, 2, 8):
    fr = P.PointsRasterizer(cams, P.PointsRasterizationSettings((60, 80), 0.05, K))(P.Pointclouds(clouds))
    fr1 = P.PointsRasterizer(P.cameras_from_opencv_projection(R[:1], T[:1], Km[:1], torch.tensor([[60, 80]], device=dev)),
                             P.PointsRasterizationSettings((60, 80), 0.05, K))(P.Pointclouds(clouds))
pts = torch.rand(2, 2000, 3, generator=g, device=dev) - 0.5
c2w = torch.eye(4, device=dev)[None].repeat(2, 1, 1); c2w[:, 2, 3] = -2.0
f = torch.randn(2, 40, 7, 60, generator=g, device=dev).permute(0, 3, 2, 1).requires_grad_(True)
Kf = torch.tensor([[[12.0, 0, 20], [0, 12, 3.5], [0, 0, 1]]], device=dev).repeat(2, 1, 1)
for K in (1, 3):
    P.points_projection(pts, c2w, Kf, f, 0.03, K).sum().backward()
torch.cuda.synchronize(); print("pts ok", int((fr.idx >= 0).sum()), float(f.grad.abs().sum()))
PY
for tool in memcheck racecheck; do
  timeout 1200 compute-sanitizer --tool $tool --error-exitcode 9 --launch-timeout 0 python /tmp/pts_case.py 2>&1 | tail -6
  echo "pts $tool rc=$?"
done
