"""Generates tests/golden/*.npz from a checkout of ComfyUI-3D-Pack named by $COMFYUI_3D_PACK:

    COMFYUI_3D_PACK=/path/to/ComfyUI-3D-Pack python tests/golden/make_golden.py

Two kinds of fixtures:
 (1) ref_*.npz  — outputs of the REFERENCE's own pure-PyTorch helpers that sit on the rasterizer path
     (SH basis shared_utils/sh_utils.py:57-112, covariance build main_3DGS_renderer.py:46-113, MiniCam /
     get_projection_matrix shared_utils/camera_utils.py:174-214).  They pin those pieces of the oracle.
     kiui (absent) is stubbed for the import only; the functions exercised do not call into it, except
     orbit_camera, which the reference itself takes from kiui (so it is NOT pinned here).
 (2) oracle_config0.npz — the oracle's own outputs for BASELINE.json config 0 (2k Gaussians, 128x128, SH-0):
     a regression fixture for the oracle and a seeded parity target for the GPU path.  The rasterizer
     arithmetic itself stays "parity unpinned" (no reference implementation of it is available offline).
"""
import os, sys, types, importlib.util
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ["COMFYUI_3D_PACK"]
sys.path.insert(0, ROOT)


def _load(path, name, stubs=()):
    for s in stubs:
        if s not in sys.modules:
            m = types.ModuleType(s); sys.modules[s] = m
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    torch.manual_seed(0)
    rng = np.random.RandomState(0)
    # ---- (1a) SH basis ---------------------------------------------------------------------------
    sh_utils = _load(os.path.join(REF, "shared_utils/sh_utils.py"), "ref_sh_utils")
    n = 64
    dirs = torch.from_numpy(rng.normal(size=(n, 3)).astype(np.float32))
    dirs = dirs / dirs.norm(dim=1, keepdim=True)
    out = {"dirs": dirs.numpy()}
    for deg in range(4):
        sh = torch.from_numpy(rng.normal(size=(n, 3, (deg + 1) ** 2)).astype(np.float32))
        out[f"sh{deg}"] = sh.numpy()
        out[f"rgb{deg}"] = sh_utils.eval_sh(deg, sh, dirs).numpy()
    out["RGB2SH"] = sh_utils.RGB2SH(torch.tensor([0.0, 0.25, 1.0])).numpy()
    out["SH2RGB"] = sh_utils.SH2RGB(torch.tensor([-1.0, 0.0, 2.0])).numpy()
    np.savez(os.path.join(HERE, "ref_sh.npz"), **out)

    # ---- (1b) covariance build (reference code allocates on "cuda": run it with a cpu shim) -----
    kiui = types.ModuleType("kiui"); kiui_cam = types.ModuleType("kiui.cam"); kiui_op = types.ModuleType("kiui.op")
    kiui_cam.orbit_camera = lambda *a, **k: (_ for _ in ()).throw(RuntimeError("stub"))
    kiui_op.inverse_sigmoid = lambda x: torch.log(x / (1 - x))
    sys.modules.update({"kiui": kiui, "kiui.cam": kiui_cam, "kiui.op": kiui_op})
    src = open(os.path.join(REF, "MVs_Algorithms/GaussianSplatting/main_3DGS_renderer.py")).read()
    # take only the three pure helper functions, redirected to the CPU
    import re
    def grab(fn):
        m = re.search(r"^def %s\(.*?(?=^def |\Z)" % fn, src, flags=re.S | re.M)
        return m.group(0).replace('device="cuda"', 'device="cpu"').replace("device='cuda'", "device='cpu'")
    ns = {"torch": torch}
    exec(grab("strip_lowerdiag") + grab("strip_symmetric") + grab("build_rotation") + grab("build_scaling_rotation"), ns)
    s = torch.from_numpy(np.exp(rng.normal(-3, 0.7, size=(n, 3))).astype(np.float32))
    q = torch.from_numpy(rng.normal(size=(n, 4)).astype(np.float32))
    q = q / q.norm(dim=1, keepdim=True)
    mod = 1.3
    L = ns["build_scaling_rotation"](mod * s, q)          # covariance_activation, main_3DGS_renderer.py:220-224
    cov = ns["strip_symmetric"](L @ L.transpose(1, 2))
    np.savez(os.path.join(HERE, "ref_cov3d.npz"), scales=s.numpy(), rotations=q.numpy(), modifier=np.float32(mod), cov=cov.numpy())

    # ---- (1c) camera matrices ---------------------------------------------------------------------
    cam_src = open(os.path.join(REF, "shared_utils/camera_utils.py")).read().replace(".cuda()", "")
    cam_src = cam_src.replace("from kiui.cam import orbit_camera", "orbit_camera = None")
    cns = {}
    exec(compile(cam_src, "camera_utils_cpu", "exec"), cns)
    from oracle import gs_oracle as O
    cams = {}
    for i, (el, az, W, H, fovy) in enumerate([(0, 0, 128, 128, 49.1), (20, 135, 1920, 1080, 49.1), (-35, -60, 200, 120, 60.0)]):
        c2w = O.orbit_camera(el, az, 1.75)
        fy = np.deg2rad(fovy); fx = 2 * np.arctan(np.tan(fy / 2) * W / H)
        mc = cns["MiniCam"](c2w.copy(), W, H, fy, fx, 0.01, 100.0)
        cams[f"c2w{i}"] = c2w; cams[f"dims{i}"] = np.array([W, H, fovy], dtype=np.float32)
        cams[f"wvt{i}"] = mc.world_view_transform.numpy(); cams[f"full{i}"] = mc.full_proj_transform.numpy()
        cams[f"center{i}"] = mc.camera_center.numpy()
        cams[f"proj{i}"] = cns["get_projection_matrix"](0.01, 100.0, fx, fy).numpy()
    np.savez(os.path.join(HERE, "ref_camera.npz"), **cams)

    # ---- (2) oracle outputs for config 0 --------------------------------------------------------
    N, W, H = 2000, 128, 128
    cl = O.make_cloud("D0", N, 0, seed=0)
    st = O.minicam_settings(O.orbit_camera(0, 0, 1.75), W, H, 49.1, sh_degree=0)
    g = torch.Generator().manual_seed(0)
    dc = torch.rand(3, H, W, generator=g) * 2 - 1
    dd = (torch.rand(1, H, W, generator=g) * 2 - 1) * 0.1
    da = (torch.rand(1, H, W, generator=g) * 2 - 1) * 0.1
    names = ("means3D", "shs", "opacities", "scales", "rotations")
    res, grads = O.rasterize_with_grads({k: cl[k] for k in names}, st, dc, dd, da)
    aux = res["aux"]
    np.savez_compressed(
        os.path.join(HERE, "oracle_config0.npz"),
        **{k: cl[k].numpy() for k in names}, dL_dcolor=dc.numpy(), dL_ddepth=dd.numpy(), dL_dalpha=da.numpy(),
        color=res["color"].numpy(), depth=res["depth"].numpy(), alpha=res["alpha"].numpy(), radii=res["radii"].numpy(),
        keys=aux["keys"], point_list=aux["point_list"], ranges=aux["ranges"], n_contrib=aux["n_contrib"].numpy(),
        **{"g_" + k: v.numpy() for k, v in grads.items()})
    print("wrote", sorted(f for f in os.listdir(HERE) if f.endswith(".npz")))


if __name__ == "__main__":
    main()
