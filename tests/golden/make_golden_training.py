"""Generates tests/golden/ref_training.npz from the REFERENCE's own GaussianModel code, run on the CPU.

    COMFYUI_3D_PACK=/path/to/ComfyUI-3D-Pack python tests/golden/make_golden_training.py

Pins the host-side pieces either side of the rasterizer (SURVEY §8 rows a8, a9, f1, f2, f4) to the reference itself:
  * get_expon_lr_func                        main_3DGS_renderer.py:21-43
  * GaussianModel.densify_and_prune          :641-688, 752-781  (clone / split / prune incl. the Adam-state surgery
                                             :543-639) on a seeded state, with torch.manual_seed fixed so that
                                             torch.normal in densify_and_split draws the same numbers in the test
  * GaussianModel.reset_opacity              :463-466
  * GaussianModel.to_ply row layout + construct_list_of_gs_attributes   :475-484, mesh_processer/mesh_utils.py:333-345
The class body is exec'd from the reference source with device="cuda" -> "cpu"; third-party names it only uses in
other methods are stubbed.  Nothing from the reference is copied into the repo: only the numeric outputs are stored.
"""
import os, re, types
import numpy as np
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ["COMFYUI_3D_PACK"]


def load_reference_model():
    src = open(os.path.join(REF, "MVs_Algorithms/GaussianSplatting/main_3DGS_renderer.py")).read()
    a = src.index("def get_expon_lr_func(")
    b = len(src)                                   # GaussianModel AND GaussianSplattingRenderer
    body = src[a:b].replace(".cuda()", "").replace('device="cuda"', 'device="cpu"').replace("device='cuda'", "device='cpu'")
    mu = open(os.path.join(REF, "mesh_processer/mesh_utils.py")).read()
    m = re.search(r"^def construct_list_of_gs_attributes\(.*?(?=^def )", mu, flags=re.S | re.M)
    captured = {}

    def write_gs_ply(xyz, normals, f_dc, f_rest, opacities, scale, rotation, names):
        captured["rows"] = np.concatenate((xyz, normals, f_dc, f_rest, opacities, scale, rotation), axis=1)
        captured["names"] = list(names)
        return None

    class _TT:                                   # torchtyping.TensorType["N", 4] in annotations
        def __getitem__(self, k):
            return torch.Tensor
    ns = {"torch": torch, "nn": nn, "np": np, "TensorType": _TT(), "PointCloud": object, "Mesh": object,
          "inverse_sigmoid": lambda x: torch.log(x / (1 - x)), "write_gs_ply": write_gs_ply,
          "SH2RGB": None, "RGB2SH": None, "eval_sh": None, "read_gs_ply": None, "K_nearest_neighbors_func": None,
          "math": __import__("math"), "F": torch.nn.functional}
    # names the renderer class needs: the reference's own SH helpers, point-cloud container stubs, a recording rasterizer
    import importlib.util, sys
    spec = importlib.util.spec_from_file_location("ref_sh_utils_t", os.path.join(REF, "shared_utils/sh_utils.py"))
    shu = importlib.util.module_from_spec(spec); spec.loader.exec_module(shu)
    ns.update(SH2RGB=shu.SH2RGB, RGB2SH=shu.RGB2SH, eval_sh=shu.eval_sh)

    class PointCloud:
        def __init__(self, points, colors, normals):
            self.points, self.colors, self.normals = points, colors, normals
    ns.update(PointCloud=PointCloud, Mesh=type("Mesh", (), {}), PlyData=type("PlyData", (), {}))
    knn = types.ModuleType("simple_knn"); knn_c = types.ModuleType("simple_knn._C")

    def distCUDA2(points):                          # third-party (absent): stand-in = exact 3-NN mean squared distance
        from scipy.spatial import cKDTree
        pn = points.numpy().astype(np.float64)
        d, _ = cKDTree(pn).query(pn, k=4)
        return torch.from_numpy((d[:, 1:] ** 2).mean(axis=1).astype(np.float32))
    knn_c.distCUDA2 = distCUDA2; knn._C = knn_c
    sys.modules["simple_knn"] = knn; sys.modules["simple_knn._C"] = knn_c
    dgr = types.ModuleType("diff_gaussian_rasterization")

    class GaussianRasterizationSettings:
        def __init__(self, **kw):
            self.kw = kw

    class GaussianRasterizer:
        def __init__(self, raster_settings):
            captured["settings"] = raster_settings.kw

        def __call__(self, **kw):
            captured["call"] = kw
            n = kw["means3D"].shape[0]
            H, W = captured["settings"]["image_height"], captured["settings"]["image_width"]
            return torch.full((3, H, W), 1.5), torch.arange(n, dtype=torch.int32) % 3, torch.zeros(1, H, W), torch.zeros(1, H, W)
    dgr.GaussianRasterizationSettings = GaussianRasterizationSettings; dgr.GaussianRasterizer = GaussianRasterizer
    sys.modules["diff_gaussian_rasterization"] = dgr
    exec(m.group(0), ns)
    exec(compile(body, "ref_gaussian_model_cpu", "exec"), ns)
    return ns, captured


def main():
    ns, captured = load_reference_model()
    out = {}
    # ---- lr schedule --------------------------------------------------------------------------------------------
    f = ns["get_expon_lr_func"](lr_init=0.00016 * 10.0, lr_final=0.0000016 * 10.0, lr_delay_mult=0.01, max_steps=30000)
    steps = np.array([0, 1, 10, 500, 2999, 15000, 30000, 40000], dtype=np.int64)
    out["lr_steps"] = steps
    out["lr_values"] = np.array([f(int(s)) for s in steps], dtype=np.float64)
    f2 = ns["get_expon_lr_func"](lr_init=1e-2, lr_final=1e-4, lr_delay_steps=100, lr_delay_mult=0.1, max_steps=1000)
    out["lr2_values"] = np.array([f2(int(s)) for s in (0, 50, 100, 1000)], dtype=np.float64)

    # ---- densify_and_prune on a seeded state ---------------------------------------------------------------------
    g = torch.Generator().manual_seed(7)
    N, deg = 600, 1
    M = (deg + 1) ** 2
    gm = ns["GaussianModel"](deg)
    xyz = (torch.rand(N, 3, generator=g) - 0.5)
    state = {
        "xyz": xyz, "f_dc": torch.randn(N, 1, 3, generator=g), "f_rest": torch.randn(N, M - 1, 3, generator=g) * 0.1,
        "scaling": torch.log(torch.rand(N, 3, generator=g) * 0.08 + 1e-3), "rotation": torch.randn(N, 4, generator=g),
        "opacity": torch.randn(N, 1, generator=g) * 2.0}
    state["scaling"][:15] = float(np.log(0.5))          # too big in world space -> pruned
    state["opacity"][40:70] = -8.0                      # sigmoid < 0.005 -> pruned
    gm._xyz = nn.Parameter(state["xyz"].clone()); gm.init_xyz = state["xyz"].clone()
    gm._features_dc = nn.Parameter(state["f_dc"].clone()); gm._features_rest = nn.Parameter(state["f_rest"].clone())
    gm._scaling = nn.Parameter(state["scaling"].clone()); gm._rotation = nn.Parameter(state["rotation"].clone())
    gm._opacity = nn.Parameter(state["opacity"].clone())
    gm.max_radii2D = torch.rand(N, generator=g) * 3.0    # some > max_screen_size = 1 (see the note in the test)
    gm.spatial_lr_scale = 10.0
    args = types.SimpleNamespace(percent_dense=0.01, position_lr_init=0.00016, position_lr_final=0.0000016,
                                 position_lr_delay_mult=0.01, position_lr_max_steps=30000, feature_lr=0.0025,
                                 opacity_lr=0.05, scaling_lr=0.005, rotation_lr=0.001)
    gm.training_setup(args)
    # one optimizer step so that Adam moments exist and are non-trivial
    for grp in gm.optimizer.param_groups:
        p = grp["params"][0]
        p.grad = torch.randn(p.shape, generator=g) * 1e-3
    pre = {k: v.detach().clone() for k, v in (("xyz", gm._xyz), ("f_dc", gm._features_dc), ("f_rest", gm._features_rest),
                                               ("scaling", gm._scaling), ("rotation", gm._rotation), ("opacity", gm._opacity))}
    grads_in = {grp["name"]: grp["params"][0].grad.clone() for grp in gm.optimizer.param_groups}
    gm.optimizer.step()
    post_step = {grp["name"]: grp["params"][0].detach().clone() for grp in gm.optimizer.param_groups}
    m1 = {grp["name"]: gm.optimizer.state[grp["params"][0]]["exp_avg"].clone() for grp in gm.optimizer.param_groups}
    m2 = {grp["name"]: gm.optimizer.state[grp["params"][0]]["exp_avg_sq"].clone() for grp in gm.optimizer.param_groups}
    gm.xyz_gradient_accum = torch.rand(N, 1, generator=g) * 4e-4
    gm.denom = torch.ones(N, 1); gm.denom[100:130] = 0.0           # 0/0 -> NaN -> 0
    for k in pre:                                  # state AFTER the optimizer step = what densification sees
        out["pre_" + k] = post_step[{"xyz": "xyz", "f_dc": "f_dc", "f_rest": "f_rest", "scaling": "scaling", "rotation": "rotation", "opacity": "opacity"}[k]].numpy()
    for k in grads_in:
        out["m1_" + k] = m1[k].numpy(); out["m2_" + k] = m2[k].numpy()
    out["grad_accum"] = gm.xyz_gradient_accum.numpy().copy(); out["denom"] = gm.denom.numpy().copy()
    out["max_radii2D"] = gm.max_radii2D.numpy().copy()
    out["adam_lrs"] = np.array([grp["lr"] for grp in gm.optimizer.param_groups], dtype=np.float64)
    torch.manual_seed(1234)
    gm.densify_and_prune(2e-4, min_opacity=0.005, extent=4, max_screen_size=1)
    out["dens_seed"] = np.int64(1234)
    for k, v in (("xyz", gm._xyz), ("f_dc", gm._features_dc), ("f_rest", gm._features_rest), ("scaling", gm._scaling),
                 ("rotation", gm._rotation), ("opacity", gm._opacity)):
        out["dens_" + k] = v.detach().numpy().copy()
    for grp in gm.optimizer.param_groups:
        st = gm.optimizer.state[grp["params"][0]]
        out["dens_m1_" + grp["name"]] = st["exp_avg"].numpy().copy()
        out["dens_m2_" + grp["name"]] = st["exp_avg_sq"].numpy().copy()
    out["dens_max_radii2D"] = gm.max_radii2D.numpy().copy()
    # ---- reset_opacity ----------------------------------------------------------------------------------------------
    gm.reset_opacity()
    out["reset_opacity"] = gm._opacity.detach().numpy().copy()
    out["reset_m1_opacity"] = gm.optimizer.state[[grp for grp in gm.optimizer.param_groups if grp["name"] == "opacity"][0]["params"][0]]["exp_avg"].numpy().copy()
    # ---- ply rows -----------------------------------------------------------------------------------------------------
    gm.to_ply()
    out["ply_rows"] = captured["rows"].astype(np.float32)
    out["ply_names"] = np.array(captured["names"])
    np.savez_compressed(os.path.join(HERE, "ref_training.npz"), **out)
    host_fixture(ns, captured)
    loop_fixture(ns)
    ngp_fit_fixture()
    print("wrote ref_training.npz:", {k: v.shape for k, v in out.items() if hasattr(v, "shape")})


def loop_fixture(ns):
    """ref_loop.npz: GaussianSplatting3D.training (MVs_Algorithms/GaussianSplatting/main_3DGS.py:129-232) executed from the
    reference source for a few steps on the CPU — its own GaussianModel / renderer / camera controller / loss composition
    / Adam — with the absent third-party pieces served by this repo's checkers: `diff_gaussian_rasterization` by
    oracle/gs_oracle.py (autograd), `pytorch_msssim.MS_SSIM` by gs_b200/losses.py, `kiui.cam.orbit_camera` by the
    oracle's.  Stored: the state before the loop, per step the reference image index / camera record / background the
    loop drew, and the raw parameters after every optimizer step.  tests/test_gpu_trainer.py replays it on the GPU."""
    import sys, random as _random, tqdm as _tqdm
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE))); sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "comfyui-3d-pack_b200"))
    from oracle import gs_oracle as O
    from gs_b200 import losses as L
    log = {"bg": [], "view": [], "proj": [], "campos": [], "tan": [], "idx": []}
    dgr = types.ModuleType("diff_gaussian_rasterization")

    class GaussianRasterizationSettings:
        def __init__(self, **kw):
            self.__dict__.update(kw)

    class GaussianRasterizer:
        def __init__(self, raster_settings):
            self.rs = raster_settings

        def __call__(self, means3D, means2D, shs=None, colors_precomp=None, opacities=None, scales=None, rotations=None, cov3D_precomp=None):
            r = self.rs
            st = O.Settings(image_height=r.image_height, image_width=r.image_width, tanfovx=r.tanfovx, tanfovy=r.tanfovy, bg=r.bg,
                            scale_modifier=r.scale_modifier, viewmatrix=r.viewmatrix, projmatrix=r.projmatrix, sh_degree=r.sh_degree,
                            campos=r.campos)
            log["bg"].append(r.bg.numpy().copy()); log["view"].append(r.viewmatrix.numpy().copy()); log["proj"].append(r.projmatrix.numpy().copy())
            log["campos"].append(r.campos.numpy().copy()); log["tan"].append(np.array([r.tanfovx, r.tanfovy], dtype=np.float32))
            return O.rasterize(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, st)
    dgr.GaussianRasterizationSettings = GaussianRasterizationSettings; dgr.GaussianRasterizer = GaussianRasterizer
    sys.modules["diff_gaussian_rasterization"] = dgr
    # camera utilities from the reference source
    cam_src = open(os.path.join(REF, "shared_utils/camera_utils.py")).read().replace(".cuda()", "").replace("device='cuda'", "device='cpu'")
    cam_src = cam_src.replace("from kiui.cam import orbit_camera", "orbit_camera = None")
    cns = {}
    exec(compile(cam_src, "camera_utils_cpu", "exec"), cns)
    cns["orbit_camera"] = O.orbit_camera
    img_src = open(os.path.join(REF, "shared_utils/image_utils.py")).read()
    m = re.search(r"^def prepare_torch_img\(.*?(?=^def )", img_src, flags=re.S | re.M)
    ins = {"torch": torch, "F": torch.nn.functional}
    exec(m.group(0).replace('device="cuda"', 'device="cpu"'), ins)

    class MS_SSIM:
        def __init__(self, data_range=1, size_average=True, channel=3):
            assert data_range == 1 and size_average and channel == 3

        def __call__(self, X, Y):
            return L.ms_ssim(X, Y)

    class _Rand:                                    # records the view index the loop draws
        def randint(self, a, b):
            i = _random.randint(a, b); log["idx"].append(i); return i

    class _Ev:
        def __init__(self, *a, **k): pass
        def record(self): pass
    comfy = types.SimpleNamespace(utils=types.SimpleNamespace(ProgressBar=lambda n: types.SimpleNamespace(update_absolute=lambda i: None)))
    src = open(os.path.join(REF, "MVs_Algorithms/GaussianSplatting/main_3DGS.py")).read()
    body = src[src.index("class GSParams"):]
    body = body.replace("device='cuda'", "device='cpu'").replace(".cuda()", "")
    body = body.replace("torch.cuda.Event(enable_timing=True)", "_Ev()").replace("torch.cuda.synchronize()", "None")
    mns = {"random": _Rand(), "tqdm": _tqdm, "torch": torch, "F": torch.nn.functional, "MS_SSIM": MS_SSIM, "SSIM": None, "comfy": comfy,
           "GaussianSplattingRenderer": ns["GaussianSplattingRenderer"], "BaseCameraController": cns["BaseCameraController"],
           "MiniCam": cns["MiniCam"], "calculate_fovX": cns["calculate_fovX"], "get_projection_matrix": cns["get_projection_matrix"],
           "prepare_torch_img": ins["prepare_torch_img"], "_Ev": _Ev}
    exec(compile(body, "ref_main_3dgs_cpu", "exec"), mns)
    K, N, deg, Hh, Ww = 5, 300, 1, 176, 176
    _random.seed(5); np.random.seed(0); torch.manual_seed(0)
    gsp = mns["GSParams"](training_iterations=K, batch_size=1, num_pts=N, sh_degree=deg, density_start_iter=10 ** 9)
    T = mns["GaussianSplatting3D"](gs_params=gsp, init_input=None, device="cpu")
    gm = T.renderer.gaussians
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():                           # a trained-like state: anisotropic, coloured, varied opacity
        gm._scaling.add_(torch.randn(N, 3, generator=g) * 0.4 + 0.8)
        gm._rotation.copy_(torch.randn(N, 4, generator=g))
        gm._features_dc.copy_(torch.randn(N, 1, 3, generator=g))
        gm._features_rest.copy_(torch.randn(N, (deg + 1) ** 2 - 1, 3, generator=g) * 0.1)
        gm._opacity.copy_(torch.randn(N, 1, generator=g))
    out = {"N": np.int64(N), "deg": np.int64(deg), "HW": np.array([Hh, Ww]), "K": np.int64(K)}
    for k, v in (("xyz", gm._xyz), ("f_dc", gm._features_dc), ("f_rest", gm._features_rest), ("scaling", gm._scaling),
                 ("rotation", gm._rotation), ("opacity", gm._opacity)):
        out["init_" + k] = v.detach().numpy().copy()
    n_ref = 3
    ref_imgs = [torch.rand(Hh, Ww, 3, generator=g) for _ in range(n_ref)]
    ref_masks = [(torch.rand(Hh, Ww, generator=g) > 0.35).float() for _ in range(n_ref)]
    poses = [(1.75, 10.0 * i - 10.0, 120.0 * i, 0.0, 0.0, 0.0) for i in range(n_ref)]          # radius, elevation, azimuth, centre
    T.prepare_training(ref_imgs, ref_masks, poses, 49.1)
    # the images are the generator's next draws after the state above: the test redraws them from the same stream, the
    # fixture keeps only their sums as a check (storing them would make it larger than 1 MB)
    out["ref_imgs_sum"] = np.float64(T.ref_imgs_torch.double().sum()); out["ref_masks_sum"] = np.float64(T.ref_masks_torch.double().sum())
    snaps = []
    opt = T.optimizer
    orig_step = opt.step

    def step_and_snapshot(*a, **k):
        r = orig_step(*a, **k)
        snaps.append({grp["name"]: grp["params"][0].detach().numpy().copy() for grp in opt.param_groups})
        return r
    opt.step = step_and_snapshot
    T.training()
    assert len(snaps) == K and len(log["idx"]) == K and len(log["bg"]) == K
    out["idx"] = np.array(log["idx"], dtype=np.int64)
    for k in ("bg", "view", "proj", "campos", "tan"):
        out["step_" + k] = np.stack(log[k])
    for kname in ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation"):
        out["after_" + kname] = np.stack([sn[kname] for sn in snaps])
    np.savez_compressed(os.path.join(HERE, "ref_loop.npz"), **out)
    print("wrote ref_loop.npz: idx", out["idx"], "bg", out["step_bg"][:, 0], "max |dxyz|", float(np.abs(out["after_xyz"][-1] - out["init_xyz"]).max()))


def ngp_fit_fixture():
    """ref_ngp_fit.npz: InstantNGP.fit_nerf (MVs_Algorithms/NeRF/Instant_NGP.py:158-205) executed from the reference source
    for two steps on the CPU (training mode: occupancy-grid update, stratified sampling, MSE losses, TV gradient, Adam with
    the reference's learning rates), nerfacc / kiui served by oracle/ngp_oracle.py and drawing their random numbers from
    the global CPU generator in the order the shims do (gs_b200/ngp.py::set_rng).  The hash tables are too large to store:
    parameters are regenerated from the seed, the fixture keeps the MLP weights and a digest of the tables (values at a
    fixed set of touched entries + sums).  tests/test_gpu_ngp.py replays it through the shims on the GPU."""
    import sys, random as _random, tqdm as _tqdm
    from torch import nn
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle import gs_oracle as O, ngp_oracle as NO

    class GridEncoder(nn.Module):
        def __init__(self, num_levels=16):
            super().__init__()
            self.num_levels = num_levels
            self.offsets = NO.grid_offsets(num_levels=num_levels)
            self.embeddings = nn.Parameter(torch.zeros(int(self.offsets[-1]), 2))
            self.output_dim = 2 * num_levels

        def forward(self, xs, bound=1):
            return NO.grid_encode(xs, self.embeddings, self.offsets, bound=float(bound), num_levels=self.num_levels)

        @torch.no_grad()
        def grad_total_variation(self, weight=1e-7, inputs=None, bound=1, B=1000000):
            x = torch.rand(B, 3) * 2 * bound - bound
            self.embeddings.grad += NO.grad_total_variation(x, self.embeddings.detach(), self.offsets, weight, bound=float(bound), num_levels=self.num_levels)

    class MLP(nn.Module):
        def __init__(self, dim_in, dim_out, dim_hidden, num_layers, bias=True):
            super().__init__()
            self.net = nn.ModuleList([nn.Linear(dim_in if l == 0 else dim_hidden, dim_out if l == num_layers - 1 else dim_hidden, bias=bias)
                                      for l in range(num_layers)])

        def forward(self, x):
            for l, lin in enumerate(self.net):
                x = lin(x)
                if l != len(self.net) - 1:
                    x = torch.relu(x)
            return x

    class OccGridEstimator(nn.Module):             # the estimator logic of gs_b200/ngp.py (nerfacc 0.5.3 semantics), marching by the oracle
        def __init__(self, roi_aabb, resolution=64, levels=1):
            super().__init__()
            self.aabb = roi_aabb; R = self.R = resolution
            self.occs = torch.zeros(R ** 3); self.binaries = torch.zeros(1, R, R, R, dtype=torch.bool)
            g = torch.arange(R)
            self.coords = torch.stack(torch.meshgrid(g, g, g, indexing="ij"), dim=-1).reshape(-1, 3)

        @torch.no_grad()
        def update_every_n_steps(self, step, occ_eval_fn, occ_thre=1e-2, ema_decay=0.95, warmup_steps=256, n=16):
            if step % n != 0:
                return
            assert step < warmup_steps
            x = (self.coords + torch.rand(tuple(self.coords.shape), dtype=torch.float32)) / self.R
            lo, hi = self.aabb[:3], self.aabb[3:]
            x = lo + x * (hi - lo)
            occ = occ_eval_fn(x).squeeze(-1)
            self.occs = torch.maximum(self.occs * ema_decay, occ)
            thre = torch.clamp(self.occs[self.occs >= 0].mean(), max=occ_thre)
            self.binaries = (self.occs > thre).view(self.binaries.shape)

        @torch.no_grad()
        def sampling(self, rays_o, rays_d, sigma_fn=None, near_plane=0.0, far_plane=1e10, render_step_size=1e-3, stratified=False, cone_angle=0.0):
            n = rays_o.shape[0]
            t_off = torch.rand((n,), dtype=torch.float32) * render_step_size if stratified else None
            ri, t0, t1 = NO.march(rays_o, rays_d, self.binaries[0], self.aabb, near_plane, far_plane, render_step_size, t_off)
            if sigma_fn is not None and ri.numel():
                sig = sigma_fn(t0, t1, ri)
                m = NO.visibility_mask(t0, t1, sig.detach(), ri, n, 1e-4, min(0.0, float(self.occs.mean())))
                ri, t0, t1 = ri[m], t0[m], t1[m]
            return ri, t0, t1
    mods = {}
    def mod(name, **attrs):
        m = types.ModuleType(name); m.__dict__.update(attrs); sys.modules[name] = m; mods[name] = m; return m
    nerfacc = mod("nerfacc", OccGridEstimator=OccGridEstimator,
        render_weight_from_density=lambda t_starts, t_ends, sigmas, ray_indices=None, n_rays=None: NO.render_weight_from_density(t_starts, t_ends, sigmas, ray_indices, n_rays),
        accumulate_along_rays=lambda weights, values=None, ray_indices=None, n_rays=None: NO.accumulate_along_rays(weights, values, ray_indices, n_rays))
    sn = lambda x, eps=1e-20: x / torch.sqrt(torch.clamp(torch.sum(x * x, -1, keepdim=True), min=eps))
    log = {"idx": []}

    class _Rand:
        def randint(self, a, b):
            i = _random.randint(a, b); log["idx"].append(i); return i
    img_src = open(os.path.join(REF, "shared_utils/image_utils.py")).read()
    m = re.search(r"^def prepare_torch_img\(.*?(?=^def )", img_src, flags=re.S | re.M)
    ins = {"torch": torch, "F": torch.nn.functional}
    exec(m.group(0).replace('device="cuda"', 'device="cpu"'), ins)
    comfy = types.SimpleNamespace(utils=types.SimpleNamespace(ProgressBar=lambda n: types.SimpleNamespace(update_absolute=lambda i: None)))
    src = open(os.path.join(REF, "MVs_Algorithms/NeRF/Instant_NGP.py")).read()
    body = src[src.index("class InstantNGP"):].replace("torch.cuda.synchronize()", "None")
    body = body.replace("from kiui.gridencoder import GridEncoder", "pass")
    mns = {"tqdm": _tqdm, "random": _Rand(), "np": np, "torch": torch, "nn": nn, "F": torch.nn.functional, "nerfacc": nerfacc, "comfy": comfy,
           "SSIM": None, "MS_SSIM": None, "safe_normalize": sn, "orbit_camera": O.orbit_camera, "MLP": MLP, "trunc_exp": NO.trunc_exp,
           "prepare_torch_img": ins["prepare_torch_img"], "GridEncoder": GridEncoder}
    exec(compile(body, "ref_instant_ngp_cpu", "exec"), mns)
    res, seed, K = 16, 777, 2
    model = mns["InstantNGP"](resolution=res, device="cpu")
    torch.manual_seed(seed); _random.seed(11)
    for enc in (model.encoder_density, model.encoder):
        enc.embeddings.data.uniform_(-0.5, 0.5)
    for mlp in (model.mlp_density, model.mlp):
        for lin in mlp.net:
            lin.weight.data.uniform_(-0.4, 0.4)
    init_d = model.encoder_density.embeddings.detach().clone(); init_c = model.encoder.embeddings.detach().clone()
    n_ref = 2
    ref_imgs = [torch.rand(res, res, 3) for _ in range(n_ref)]
    ref_masks = [(torch.rand(res, res) > 0.4).float() for _ in range(n_ref)]
    poses = [(1.75, -10.0 + 25.0 * i, 80.0 * i, 0.0, 0.0, 0.0) for i in range(n_ref)]
    model.prepare_training(ref_imgs, ref_masks, poses, 49.1)
    model.train()
    model.fit_nerf(iters=K, bg_color=1)
    out = {"seed": np.int64(seed), "res": np.int64(res), "K": np.int64(K), "idx": np.array(log["idx"], dtype=np.int64),
           "levels": np.int64(model.encoder.num_levels), "poses": np.array(poses, dtype=np.float32),
           "ref_imgs": torch.stack(ref_imgs).numpy(), "ref_masks": torch.stack(ref_masks).numpy()}
    for name, mlp in (("mlp_density", model.mlp_density), ("mlp_color", model.mlp)):
        for l, lin in enumerate(mlp.net):
            out[f"{name}_w{l}"] = lin.weight.detach().numpy().copy()
    g = torch.Generator().manual_seed(1)
    for name, emb, init in (("emb_density", model.encoder_density.embeddings.detach(), init_d), ("emb_color", model.encoder.embeddings.detach(), init_c)):
        changed = torch.nonzero((emb != init).any(dim=1))[:, 0]
        pick = changed[torch.randperm(changed.numel(), generator=g)[:40000]]
        rnd = torch.randint(0, emb.shape[0], (10000,), generator=g)
        ids = torch.unique(torch.cat([pick, rnd]))
        out[name + "_ids"] = ids.numpy(); out[name + "_vals"] = emb[ids].numpy().copy()
        out[name + "_sum"] = np.float64(emb.double().sum()); out[name + "_abs_delta"] = np.float64((emb - init).double().abs().sum())
        out[name + "_n_changed"] = np.int64(changed.numel())
    out["binaries_count"] = np.int64(int(model.estimator.binaries.sum()))
    np.savez_compressed(os.path.join(HERE, "ref_ngp_fit.npz"), **out)
    print("wrote ref_ngp_fit.npz: idx", out["idx"], "changed entries", int(out["emb_density_n_changed"]), int(out["emb_color_n_changed"]),
          "occupied cells", int(out["binaries_count"]))
    for k in list(mods):
        sys.modules.pop(k, None)


def host_fixture(ns, captured):
    """ref_host.npz: the reference's random initialisation (GaussianSplattingRenderer.initialize(None, n) +
    GaussianModel.create_from_pcd, main_3DGS_renderer.py:798-826, 407-433), its render() host wrapper (:830-949) driven
    with a recording rasterizer, and InstantNGP.get_rays (MVs_Algorithms/NeRF/Instant_NGP.py:37-70)."""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle import gs_oracle as O
    out = {}
    n, deg = 500, 2
    R = ns["GaussianSplattingRenderer"](sh_degree=deg, white_background=False, radius=1)
    np.random.seed(0)
    R.initialize(None, num_pts=n)
    gm = R.gaussians
    out["init_xyz"] = gm.get_xyz.detach().numpy(); out["init_features"] = gm.get_features.detach().numpy()
    out["init_opacity"] = gm.get_opacity.detach().numpy(); out["init_scaling"] = gm.get_scaling.detach().numpy()
    out["init_rotation"] = gm.get_rotation.detach().numpy(); out["init_spatial_lr_scale"] = np.float32(gm.spatial_lr_scale)
    out["init_raw_opacity"] = gm._opacity.detach().numpy(); out["init_raw_scaling"] = gm._scaling.detach().numpy()
    # render() wrapper with the reference's own MiniCam
    cam_src = open(os.path.join(REF, "shared_utils/camera_utils.py")).read().replace(".cuda()", "")
    cam_src = cam_src.replace("from kiui.cam import orbit_camera", "orbit_camera = None")
    cns = {}
    exec(compile(cam_src, "camera_utils_cpu", "exec"), cns)
    W, H, fovy_deg = 200, 120, 49.1
    c2w = O.orbit_camera(15, 70, 1.75)
    fy = np.deg2rad(fovy_deg); fx = 2 * np.arctan(np.tan(fy / 2) * W / H)
    cam = cns["MiniCam"](c2w.copy(), W, H, fy, fx, 0.01, 100.0)
    gm.active_sh_degree = deg
    res = R.render(cam)
    st, call = captured["settings"], captured["call"]
    out["render_c2w"] = c2w; out["render_dims"] = np.array([W, H, fovy_deg], dtype=np.float32)
    for k in ("image_height", "image_width", "tanfovx", "tanfovy", "scale_modifier", "sh_degree", "prefiltered", "debug"):
        out["set_" + k] = np.float64(st[k])
    for k in ("bg", "viewmatrix", "projmatrix", "campos"):
        out["set_" + k] = st[k].numpy()
    out["call_keys"] = np.array(sorted(call.keys()))
    out["call_none"] = np.array(sorted(k for k, v in call.items() if v is None))
    for k in ("means3D", "means2D", "shs", "opacities", "scales", "rotations"):
        out["call_" + k] = call[k].detach().numpy()
    out["call_means2D_requires_grad"] = np.bool_(call["means2D"].requires_grad)
    out["res_image_max"] = np.float32(res["image"].max())           # clamp(0,1) of the stub's 1.5
    out["res_visibility"] = res["visibility_filter"].numpy()
    # mesh path: OrbitCamera.perspective (camera_utils.py:128-145) and the clip transform of DiffRastRenderer.render
    # (MVs_Algorithms/DiffRastMesh/diff_mesh_renderer.py:91-95), executed from the reference source
    oc = cns["OrbitCamera"](1920, 1080, r=2.2, fovy=49.1, near=0.01, far=100)
    out["gl_persp"] = oc.perspective
    dm_src = open(os.path.join(REF, "MVs_Algorithms/DiffRastMesh/diff_mesh_renderer.py")).read()
    lines = [l for l in dm_src.splitlines() if ("pose = torch.from_numpy" in l or "proj = torch.from_numpy" in l or "v_cam = torch.matmul" in l or "v_clip = v_cam @" in l)]
    assert len(lines) == 4, lines
    gv = torch.Generator().manual_seed(5)
    v = torch.rand(64, 3, generator=gv) - 0.5
    pose_m = O.orbit_camera(25, -40, 2.2).astype(np.float32)
    dns = {"torch": torch, "np": np, "F": torch.nn.functional, "v": v, "pose": pose_m, "proj": oc.perspective}
    exec("\n".join(l.strip() for l in lines), dns)
    out["clip_v"] = v.numpy(); out["clip_pose"] = pose_m; out["clip_out"] = dns["v_clip"].numpy()
    # Instant-NGP rays
    ngp_src = open(os.path.join(REF, "MVs_Algorithms/NeRF/Instant_NGP.py")).read()
    m = re.search(r"^    def get_rays\(.*?(?=^    def )", ngp_src, flags=re.S | re.M)
    import textwrap
    rns = {"torch": torch, "np": np, "F": torch.nn.functional,
           "safe_normalize": lambda x, eps=1e-20: x / torch.sqrt(torch.clamp(torch.sum(x * x, -1, keepdim=True), min=eps))}
    exec(textwrap.dedent(m.group(0)), rns)
    pose = torch.from_numpy(O.orbit_camera(-20, 200, 1.75).astype(np.float32))
    ro, rd = rns["get_rays"](None, pose, 36, 50, 49.1)
    out["rays_pose"] = pose.numpy(); out["rays_o"] = ro.numpy(); out["rays_d"] = rd.numpy()
    ngp_fixture(out, O)
    mesh_fixture(out, O)
    flexi_fixture(out, O)
    bake_fixture(out, O)
    np.savez_compressed(os.path.join(HERE, "ref_host.npz"), **out)
    print("wrote ref_host.npz:", sorted(out.keys()))


def mesh_fixture(out, O):
    """DiffRastRenderer.render (MVs_Algorithms/DiffRastMesh/diff_mesh_renderer.py:72-159) executed from the reference
    source with `nvdiffrast.torch` served by oracle/dr_oracle.py: pins the op order and composition of the mesh path
    (clip transform, rasterize, antialias(alpha), interpolate(uv, 'all'), texture('linear') + sigmoid, depth and normal
    interpolation, antialias(colour), background blend) that tests/test_gpu_mesh.py replays against the shim."""
    import sys, importlib.util
    from oracle import dr_oracle as DO
    mods = {}
    def mod(name, **attrs):
        m = types.ModuleType(name); m.__dict__.update(attrs); sys.modules[name] = m; mods[name] = m; return m
    nv = mod("nvdiffrast")
    drt = mod("nvdiffrast.torch", RasterizeCudaContext=lambda *a, **k: object(), RasterizeGLContext=lambda *a, **k: object(),
              rasterize=lambda ctx, pos, tri, resolution: DO.rasterize(pos, tri, tuple(resolution)),
              interpolate=lambda attr, rast, tri, rast_db=None, diff_attrs=None: DO.interpolate(attr, rast, tri, rast_db=rast_db, diff_attrs=diff_attrs),
              texture=lambda tex, uv, uv_da=None, filter_mode="auto": DO.texture(tex, uv, filter_mode="linear"),
              antialias=lambda color, rast, pos, tri: DO.antialias(color, rast, pos, tri))
    nv.torch = drt
    sn = lambda x, eps=1e-20: x / torch.sqrt(torch.clamp(torch.sum(x * x, -1, keepdim=True), min=eps))
    mod("kiui"); mod("kiui.op", inverse_sigmoid=lambda x: torch.log(x / (1 - x)))
    mod("mesh_processer"); mod("mesh_processer.mesh", safe_normalize=sn)
    spec = importlib.util.spec_from_file_location("ref_diff_mesh_renderer", os.path.join(REF, "MVs_Algorithms/DiffRastMesh/diff_mesh_renderer.py"))
    dm = importlib.util.module_from_spec(spec); spec.loader.exec_module(dm)
    v, f, uv = DO.icosphere(2, 0.5)
    g = torch.Generator().manual_seed(11)
    albedo = torch.rand(16, 16, 3, generator=g) * 0.8 + 0.1
    mesh = types.SimpleNamespace(v=v, f=f, vt=uv, ft=f, vn=sn(v), fn=f, albedo=albedo)
    R = dm.DiffRastRenderer(mesh, True)
    Hh, Ww = 40, 48
    pose = O.orbit_camera(20, 35, 1.75).astype(np.float32)
    proj = DO.gl_perspective(49.1, Ww / Hh)
    with torch.no_grad():
        res = R.render(pose, proj, Hh, Ww, ssaa=1, bg_color=1)
    out["mesh_pose"] = pose; out["mesh_proj"] = proj; out["mesh_hw"] = np.array([Hh, Ww]); out["mesh_albedo"] = albedo.numpy()
    for k in ("image", "alpha", "depth", "normal", "viewcos"):
        out["mesh_" + k] = res[k].numpy()
    for k in list(mods):
        sys.modules.pop(k, None)


def bake_fixture(out, O):
    """color_func_to_albedo (mesh_processer/mesh_utils.py:521-568) executed from the reference source: UV-space rasterize
    (uv*2-1, z=0, w=1), interpolate positions and a coverage mask, query a colour function on the covered texels, pad.
    `nvdiffrast.torch` = oracle/dr_oracle.py; `kiui.op.uv_padding` = this repo's shim (gs_b200/texops.py), so the pin is
    on the composition, not on the padding rule (kiui is absent)."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "comfyui-3d-pack_b200"))
    from oracle import dr_oracle as DO
    from gs_b200 import texops
    mods = {}
    def mod(name, **attrs):
        m = types.ModuleType(name); m.__dict__.update(attrs); sys.modules[name] = m; mods[name] = m; return m
    nv = mod("nvdiffrast")
    drt = mod("nvdiffrast.torch", RasterizeCudaContext=lambda *a, **k: object(), RasterizeGLContext=lambda *a, **k: object(),
              rasterize=lambda ctx, pos, tri, resolution: DO.rasterize(pos, tri, tuple(resolution)),
              interpolate=lambda attr, rast, tri, rast_db=None, diff_attrs=None: DO.interpolate(attr, rast, tri, rast_db=rast_db, diff_attrs=diff_attrs))
    nv.torch = drt
    mod("kiui"); mod("kiui.op", uv_padding=texops.uv_padding)
    mu = open(os.path.join(REF, "mesh_processer/mesh_utils.py")).read()
    m = re.search(r"^def color_func_to_albedo\(.*?(?=^@torch|^def )", mu, flags=re.S | re.M)
    fns = {"torch": torch, "np": np}
    exec(m.group(0).replace('device="cuda"', 'device="cpu"'), fns)
    v, f, uv = DO.icosphere(1, 0.5)
    uv = uv * 0.8 + 0.1                                # keep the chart strictly inside the texture
    mesh = types.SimpleNamespace(v=v, f=f, vt=uv, ft=f)
    rgb_fn = lambda xyz: torch.stack([xyz[:, 0] + 0.5, xyz[:, 1] * xyz[:, 2] + 0.5, (xyz ** 2).sum(-1)], dim=1)
    alb = fns["color_func_to_albedo"](mesh, rgb_fn, texture_resolution=48, padding=2, batch_size=1000, device="cpu", force_cuda_rast=True)
    out["bake_albedo"] = alb.numpy(); out["bake_uv_scale"] = np.array([0.8, 0.1], dtype=np.float32)
    for k in list(mods):
        sys.modules.pop(k, None)


def flexi_fixture(out, O):
    """FlexiCubesRenderer.get_orbit_camera + render_mesh (MVs_Algorithms/FlexiCubes/flexicubes_renderer.py:26-74, with
    util.perspective / xfm_points / interpolate / SimpleMesh.auto_normals, FlexiCubes/util.py:25-93) executed from the
    reference source for a BATCH of two views, `nvdiffrast.torch` served by oracle/dr_oracle.py: mask (antialiased),
    normalised depth, per-face normals via the `arange(F)` attribute index trick, vertex normals, white background."""
    import sys, importlib.util
    from oracle import dr_oracle as DO
    mods = {}
    def mod(name, **attrs):
        m = types.ModuleType(name); m.__dict__.update(attrs); sys.modules[name] = m; mods[name] = m; return m
    nv = mod("nvdiffrast")
    drt = mod("nvdiffrast.torch", RasterizeCudaContext=lambda *a, **k: object(), RasterizeGLContext=lambda *a, **k: object(),
              rasterize=lambda ctx, pos, tri, resolution: DO.rasterize(pos, tri, tuple(resolution)),
              interpolate=lambda attr, rast, tri, rast_db=None, diff_attrs=None: DO.interpolate(attr, rast, tri, rast_db=rast_db, diff_attrs=diff_attrs),
              antialias=lambda color, rast, pos, tri: DO.antialias(color, rast, pos, tri))
    nv.torch = drt
    mod("kiui"); mod("kiui.cam", orbit_camera=O.orbit_camera)
    usrc = open(os.path.join(REF, "MVs_Algorithms/FlexiCubes/util.py")).read()
    util = types.ModuleType("FlexiCubes.util")
    exec(compile(usrc, "ref_flexi_util", "exec"), util.__dict__)
    fc = mod("FlexiCubes"); fc.util = util; sys.modules["FlexiCubes.util"] = util; mods["FlexiCubes.util"] = util
    rsrc = open(os.path.join(REF, "MVs_Algorithms/FlexiCubes/flexicubes_renderer.py")).read().replace("device='cuda'", "device='cpu'").replace('device="cuda"', 'device="cpu"')
    rns = {}
    exec(compile(rsrc, "ref_flexi_renderer", "exec"), rns)
    v, f, _ = DO.icosphere(2, 0.8)
    mesh = util.SimpleMesh(v, f.long())
    mesh.auto_normals()
    mesh.v_nrm = util.safe_normalize(v)
    R = rns["FlexiCubesRenderer"](True)
    res = [40, 56]
    cams = [R.get_orbit_camera(azimuth=az, elevation=el, fovy=45, iter_res=res, cam_radius=3.0, device="cpu") for az, el in ((30.0, 10.0), (200.0, -25.0))]
    mv = torch.stack([c[0] for c in cams]).float(); mvp = torch.stack([c[1] for c in cams]).float()
    with torch.no_grad():
        outd = R.render_mesh(mesh, mv, mvp, res, return_types=["mask", "depth", "normal", "vertex_normal"], white_bg=True)
    out["flexi_mv"] = mv.numpy(); out["flexi_mvp"] = mvp.numpy(); out["flexi_res"] = np.array(res)
    for k, t in outd.items():
        out["flexi_" + k] = t.numpy()
    # ---- c4 feeding c2: the reference's own FlexiCubes.__call__ (flexicubes.py:133-216 + tables.py, pure torch) extracts
    # a mesh from a sphere SDF on a 14^3 grid; the reference renderer renders THAT mesh (changing topology is the case
    # FlexiCubesRenderer exists for).  The GPU test feeds the stored mesh to the CUDA shim.
    tsrc = open(os.path.join(REF, "MVs_Algorithms/FlexiCubes/tables.py")).read()
    tables = types.ModuleType("FlexiCubes.tables")
    exec(compile(tsrc, "ref_flexi_tables", "exec"), tables.__dict__)
    sys.modules["FlexiCubes.tables"] = tables; mods["FlexiCubes.tables"] = tables
    fsrc = open(os.path.join(REF, "MVs_Algorithms/FlexiCubes/flexicubes.py")).read().replace("from .tables import *", "from FlexiCubes.tables import *")
    fns = {}
    exec(compile(fsrc, "ref_flexicubes", "exec"), fns)
    fcx = fns["FlexiCubes"](device="cpu")
    gres = 14
    x_nx3, cube_fx8 = fcx.construct_voxel_grid(gres)
    x_nx3 = x_nx3 * 2.0                                                   # grid spans [-1, 1]^3
    g = torch.Generator().manual_seed(11)
    sdf = x_nx3.norm(dim=-1) - 0.62 + 0.03 * torch.randn(x_nx3.shape[0], generator=g)      # a bumpy sphere
    with torch.no_grad():
        ev, ef, _ = fcx(x_nx3, sdf, cube_fx8, gres, training=False)
    emesh = util.SimpleMesh(ev.float(), ef.long())
    emesh.auto_normals()
    emesh.v_nrm = util.safe_normalize(ev.float())
    with torch.no_grad():
        outx = R.render_mesh(emesh, mv, mvp, res, return_types=["mask", "depth", "normal", "vertex_normal"], white_bg=True)
    out["flexi_ex_v"] = ev.float().numpy(); out["flexi_ex_f"] = ef.numpy().astype(np.int32)
    for k, t in outx.items():
        out["flexi_ex_" + k] = t.numpy()
    for k in list(mods):
        sys.modules.pop(k, None)


def ngp_fixture(out, O):
    """InstantNGP.render_nerf (MVs_Algorithms/NeRF/Instant_NGP.py:101-156) executed from the reference source with its
    third-party imports (nerfacc, kiui — absent) served by oracle/ngp_oracle.py: pins the CALL SEQUENCE and composition
    (ray generation, density-driven sampling, sample midpoints, the two field queries, weights, accumulation, background)
    that tests/test_gpu_ngp.py::test_render_nerf_call_sequence_matches_oracle replays.  Parameters are regenerated in the
    test from the stored seed (tables are tens of MB)."""
    import sys
    from torch import nn
    from oracle import ngp_oracle as NO

    class GridEncoder(nn.Module):
        def __init__(self, num_levels=16):
            super().__init__()
            self.num_levels = num_levels
            self.offsets = NO.grid_offsets(num_levels=num_levels)
            self.embeddings = nn.Parameter(torch.zeros(int(self.offsets[-1]), 2))
            self.output_dim = 2 * num_levels

        def forward(self, xs, bound=1):
            return NO.grid_encode(xs, self.embeddings, self.offsets, bound=float(bound), num_levels=self.num_levels)

    class MLP(nn.Module):
        def __init__(self, dim_in, dim_out, dim_hidden, num_layers, bias=True):
            super().__init__()
            self.net = nn.ModuleList([nn.Linear(dim_in if l == 0 else dim_hidden, dim_out if l == num_layers - 1 else dim_hidden, bias=bias)
                                      for l in range(num_layers)])

        def forward(self, x):
            for l, lin in enumerate(self.net):
                x = lin(x)
                if l != len(self.net) - 1:
                    x = torch.relu(x)
            return x

    class OccGridEstimator(nn.Module):
        def __init__(self, roi_aabb, resolution=64, levels=1):
            super().__init__()
            self.aabb = roi_aabb; self.binaries = torch.zeros(1, resolution, resolution, resolution, dtype=torch.bool)

        def sampling(self, rays_o, rays_d, sigma_fn=None, near_plane=0.0, far_plane=1e10, render_step_size=1e-3, stratified=False, cone_angle=0.0):
            assert not stratified and cone_angle == 0
            ri, t0, t1 = NO.march(rays_o, rays_d, self.binaries[0], self.aabb, near_plane, far_plane, render_step_size)
            if sigma_fn is not None and ri.numel():
                sig = sigma_fn(t0, t1, ri)
                m = NO.visibility_mask(t0, t1, sig, ri, rays_o.shape[0], 1e-4, 0.0)
                ri, t0, t1 = ri[m], t0[m], t1[m]
            return ri, t0, t1
    mods = {}
    def mod(name, **attrs):
        m = types.ModuleType(name); m.__dict__.update(attrs); sys.modules[name] = m; mods[name] = m; return m
    mod("nerfacc", OccGridEstimator=OccGridEstimator,
        render_weight_from_density=lambda t_starts, t_ends, sigmas, ray_indices=None, n_rays=None: NO.render_weight_from_density(t_starts, t_ends, sigmas, ray_indices, n_rays),
        accumulate_along_rays=lambda weights, values=None, ray_indices=None, n_rays=None: NO.accumulate_along_rays(weights, values, ray_indices, n_rays))
    mod("comfy"); mod("comfy.utils")
    mod("pytorch_msssim", SSIM=object, MS_SSIM=object)
    mod("kiui"); mod("kiui.op", safe_normalize=lambda x, eps=1e-20: x / torch.sqrt(torch.clamp(torch.sum(x * x, -1, keepdim=True), min=eps)))
    mod("kiui.cam", orbit_camera=O.orbit_camera); mod("kiui.nn", MLP=MLP, trunc_exp=NO.trunc_exp); mod("kiui.gridencoder", GridEncoder=GridEncoder)
    mod("shared_utils"); mod("shared_utils.image_utils", prepare_torch_img=None)
    import importlib.util
    spec = importlib.util.spec_from_file_location("ref_instant_ngp", os.path.join(REF, "MVs_Algorithms/NeRF/Instant_NGP.py"))
    ngp = importlib.util.module_from_spec(spec); spec.loader.exec_module(ngp)
    res, seed = 20, 4321
    model = ngp.InstantNGP(resolution=res, device="cpu")
    model.ref_cam_fovy = 49.1
    model.eval()
    torch.manual_seed(seed)                      # parameter order below is what the test reproduces
    for enc in (model.encoder_density, model.encoder):
        enc.embeddings.data.uniform_(-0.5, 0.5)
    for mlp in (model.mlp_density, model.mlp):
        for lin in mlp.net:
            lin.weight.data.uniform_(-0.4, 0.4)
    R = 64
    gg = (torch.arange(R).float() + 0.5) / R * 2 - 1
    x, y, z = torch.meshgrid(gg, gg, gg, indexing="ij")
    model.estimator.binaries = ((x * x + y * y + z * z) < 0.36)[None]
    pose = O.orbit_camera(10, 140, 1.75).astype(np.float32)
    with torch.no_grad():
        color, alpha = model.render_nerf(pose, bg_color=1)
    out["ngp_seed"] = np.int64(seed); out["ngp_res"] = np.int64(res); out["ngp_pose"] = pose
    out["ngp_color"] = color.numpy(); out["ngp_alpha"] = alpha.numpy()
    out["ngp_levels"] = np.int64(model.encoder.num_levels); out["ngp_mlp_in"] = np.int64(model.encoder.output_dim)
    for k in list(mods):
        sys.modules.pop(k, None)


if __name__ == "__main__":
    main()
