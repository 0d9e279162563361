"""GPU parity tests (run on an H100: pytest -m gpu).  Every test goes through the C ABI
(libgs_b200.so via ctypes); the CPU oracle is the checker.

Tolerances (BASELINE.json north_star): rendered RGBA within 1e-4 abs, gradients within 1e-3 relative,
tile/key indices bit-exact."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import gs_oracle as O

pytestmark = pytest.mark.gpu
NAMES = ("means3D", "shs", "opacities", "scales", "rotations")
RGBA_ATOL = 1e-4
GRAD_RTOL = 1e-3


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def R():
    from gs_b200 import rasterizer
    return rasterizer


def _rs(R, st, dev, deg, debug=False):
    return R.GaussianRasterizationSettings(st.image_height, st.image_width, st.tanfovx, st.tanfovy, st.bg.to(dev),
                                           st.scale_modifier, st.viewmatrix.to(dev), st.projmatrix.to(dev), deg,
                                           st.campos.to(dev), False, debug)


def _upstream(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(3, H, W, generator=g) * 2 - 1, (torch.rand(1, H, W, generator=g) * 2 - 1) * 0.1,
            (torch.rand(1, H, W, generator=g) * 2 - 1) * 0.1)


def _grad_close(a, b, what):
    a, b = a.detach().cpu().double(), b.double()
    scale = float(b.abs().max())
    if scale == 0.0:
        assert float(a.abs().max()) < 1e-5, what
        return
    rel = float((a - b).norm() / b.norm())
    assert rel < GRAD_RTOL, f"{what}: relative error {rel}"
    # element-wise: 1e-3 relative with an absolute floor of 1e-5 of the largest component.  Each element is a sum of up
    # to thousands of fp32 atomics whose order changes from run to run (and differs from the oracle's), so its noise
    # scales with the sum of |terms|, not with the (often cancelling) result; a 1e-6 floor failed about once per
    # cold-start run on one element of dL/dscales while the norm-relative check above stayed below 1e-4.
    assert bool(((a - b).abs() <= GRAD_RTOL * b.abs() + 1e-2 * GRAD_RTOL * scale + 1e-6).all()), what


# ---------------- CUB-free onesweep radix sort -----------------------------------------------------------
@pytest.mark.parametrize("n,bits", [(0, 32), (1, 32), (33, 32), (4096, 32), (4097, 13), (123457, 20), (1 << 20, 32), (3_000_001, 13)])
def test_onesweep_sort_matches_stable_sort(R, dev, n, bits):
    g = torch.Generator(device="cpu").manual_seed(n + bits)
    k = torch.randint(0, 2 ** 31 - 1, (n,), generator=g, dtype=torch.int32).to(dev)
    if bits < 32:
        k = k & ((1 << bits) - 1)
    v = torch.arange(n, device=dev, dtype=torch.int32)
    sk, sv = R.sort_pairs_u32(k, v, 0, bits)
    rk, ri = torch.sort(k.to(torch.int64), stable=True)
    assert torch.equal(sk.to(torch.int64), rk) and torch.equal(sv.to(torch.int64), ri)


def test_onesweep_sort_high_bit_keys_and_ties(R, dev):
    # unsigned ordering (bit 31 set) and heavy ties -> stability
    k = torch.tensor([-1, 5, -2147483648, 5, 0, -1, 5], dtype=torch.int32, device=dev)
    v = torch.arange(7, device=dev, dtype=torch.int32)
    sk, sv = R.sort_pairs_u32(k, v)
    ku = k.cpu().numpy().view(np.uint32).astype(np.int64)
    order = np.argsort(ku, kind="stable")
    assert list(sv.cpu().numpy()) == list(order)
    n = 50000
    k = torch.randint(0, 7, (n,), dtype=torch.int32, device=dev)
    sk, sv = R.sort_pairs_u32(k, torch.arange(n, device=dev, dtype=torch.int32), 0, 3)
    rk, ri = torch.sort(k.to(torch.int64), stable=True)
    assert torch.equal(sv.to(torch.int64), ri)


# ---------------- forward + backward parity vs the oracle ----------------------------------------------
CASES = [
    # kind, N, deg, W, H, elev, azim, bg
    ("D0", 2000, 0, 128, 128, 0, 0, (0, 0, 0)),          # BASELINE config 0
    ("D1", 2000, 3, 128, 128, 10, 30, (0, 0, 0)),
    ("D1", 1500, 1, 100, 70, -20, 200, (1, 1, 1)),       # ragged: sizes not multiples of 16, white background
    ("D1", 20000, 2, 200, 120, 5, 75, (0.2, 0.3, 0.4)),
    ("D0", 30000, 3, 320, 180, 0, 45, (0, 0, 0)),
]


@pytest.mark.parametrize("kind,N,deg,W,H,el,az,bg", CASES)
def test_forward_backward_parity(R, dev, kind, N, deg, W, H, el, az, bg):
    cl = O.make_cloud(kind, N, deg, seed=N % 7)
    st = O.minicam_settings(O.orbit_camera(el, az, 1.75), W, H, 49.1, bg=bg, sh_degree=deg)
    dc, dd, da = _upstream(H, W, N)
    out, grads = O.rasterize_with_grads({k: cl[k] for k in NAMES}, st, dc, dd, da)
    aux = out["aux"]
    rs = _rs(R, st, dev, deg, debug=True)
    fs = R.forward_with_state(rs, cl["means3D"].to(dev), cl["opacities"].to(dev), shs=cl["shs"].to(dev),
                              scales=cl["scales"].to(dev), rotations=cl["rotations"].to(dev))
    # integer outputs: bit-exact
    assert torch.equal(fs["radii"].cpu(), out["radii"])
    assert fs["num_rendered"] == aux["keys"].size
    assert np.array_equal(fs["sorted_keys"].cpu().numpy().astype(np.uint64), aux["keys"])
    assert np.array_equal(fs["point_list"].cpu().numpy().astype(np.uint32), aux["point_list"])
    assert np.array_equal(fs["ranges"].cpu().numpy().astype(np.uint32), aux["ranges"])
    assert int((fs["n_contrib"].cpu() != aux["n_contrib"]).sum()) == 0
    # floating outputs
    assert float((fs["color"].cpu() - out["color"]).abs().max()) < RGBA_ATOL
    assert float((fs["alpha"].cpu() - out["alpha"]).abs().max()) < RGBA_ATOL
    assert float((fs["depth"].cpu() - out["depth"]).abs().max()) < RGBA_ATOL * 2
    assert float((fs["final_T"].cpu() - aux["final_T"]).abs().max()) < RGBA_ATOL
    # gradients through the reference-facing interface
    inp = {k: cl[k].to(dev).requires_grad_(True) for k in NAMES}
    m2 = torch.zeros(N, 3, device=dev, requires_grad=True)
    color, radii, depth, alpha = R.GaussianRasterizer(_rs(R, st, dev, deg))(
        means3D=inp["means3D"], means2D=m2, shs=inp["shs"], colors_precomp=None, opacities=inp["opacities"],
        scales=inp["scales"], rotations=inp["rotations"], cov3D_precomp=None)
    ((color * dc.to(dev)).sum() + (depth * dd.to(dev)).sum() + (alpha * da.to(dev)).sum()).backward()
    for k in NAMES:
        _grad_close(inp[k].grad, grads[k], f"{kind} N={N} grad {k}")
    _grad_close(m2.grad, grads["means2D"], "grad means2D")
    assert float(m2.grad[:, 2].abs().max()) == 0.0


def test_golden_fixture_config0(R, dev):
    g = np.load(os.path.join(GOLDEN, "oracle_config0.npz"))
    t = lambda k: torch.from_numpy(g[k]).to(dev)
    st = O.minicam_settings(O.orbit_camera(0, 0, 1.75), 128, 128, 49.1, sh_degree=0)
    rs = _rs(R, st, dev, 0)
    inp = {k: t(k).requires_grad_(True) for k in NAMES}
    m2 = torch.zeros(2000, 3, device=dev, requires_grad=True)
    color, radii, depth, alpha = R.GaussianRasterizer(rs)(
        means3D=inp["means3D"], means2D=m2, shs=inp["shs"], colors_precomp=None, opacities=inp["opacities"],
        scales=inp["scales"], rotations=inp["rotations"], cov3D_precomp=None)
    assert np.array_equal(radii.cpu().numpy(), g["radii"])
    assert np.abs(color.detach().cpu().numpy() - g["color"]).max() < RGBA_ATOL
    assert np.abs(alpha.detach().cpu().numpy() - g["alpha"]).max() < RGBA_ATOL
    ((color * t("dL_dcolor")).sum() + (depth * t("dL_ddepth")).sum() + (alpha * t("dL_dalpha")).sum()).backward()
    for k in NAMES:
        _grad_close(inp[k].grad, torch.from_numpy(g["g_" + k]), f"golden grad {k}")
    fs = R.forward_with_state(rs, t("means3D"), t("opacities"), shs=t("shs"), scales=t("scales"), rotations=t("rotations"))
    assert np.array_equal(fs["sorted_keys"].cpu().numpy().astype(np.uint64), g["keys"])
    assert np.array_equal(fs["point_list"].cpu().numpy().astype(np.uint32), g["point_list"])
    assert np.array_equal(fs["ranges"].cpu().numpy().astype(np.uint32), g["ranges"])


def test_colors_precomp_and_cov3d_precomp_paths(R, dev):
    N, W, H = 3000, 96, 80
    cl = O.make_cloud("D1", N, 0, seed=9)
    st = O.minicam_settings(O.orbit_camera(15, -50, 1.75), W, H, 49.1, bg=(0.5, 0.5, 0.5), scale_modifier=1.2)
    cols = torch.rand(N, 3, generator=torch.Generator().manual_seed(3))
    cov = O.cov3d_from_scale_rot(cl["scales"], cl["rotations"], 1.2)
    dc, dd, da = _upstream(H, W, 5)
    ins = dict(means3D=cl["means3D"], colors_precomp=cols, opacities=cl["opacities"], cov3D_precomp=cov)
    out, grads = O.rasterize_with_grads(ins, st, dc, dd, da)
    inp = {k: v.to(dev).requires_grad_(True) for k, v in ins.items()}
    m2 = torch.zeros(N, 3, device=dev, requires_grad=True)
    color, radii, depth, alpha = R.GaussianRasterizer(_rs(R, st, dev, 0))(
        means3D=inp["means3D"], means2D=m2, shs=None, colors_precomp=inp["colors_precomp"], opacities=inp["opacities"],
        scales=None, rotations=None, cov3D_precomp=inp["cov3D_precomp"])
    assert torch.equal(radii.cpu(), out["radii"])
    assert float((color.detach().cpu() - out["color"]).abs().max()) < RGBA_ATOL
    ((color * dc.to(dev)).sum() + (depth * dd.to(dev)).sum() + (alpha * da.to(dev)).sum()).backward()
    for k in ins:
        _grad_close(inp[k].grad, grads[k], f"precomp grad {k}")


def test_empty_culled_and_offscreen_inputs(R, dev):
    st = O.minicam_settings(O.orbit_camera(0, 0, 1.75), 64, 48, 49.1, bg=(0.1, 0.2, 0.3))
    rs = _rs(R, st, dev, 0)
    z = lambda *s: torch.zeros(*s, device=dev)
    color, radii, depth, alpha = R.GaussianRasterizer(rs)(means3D=z(0, 3), means2D=z(0, 3), opacities=z(0, 1),
                                                         colors_precomp=z(0, 3), scales=z(0, 3), rotations=z(0, 4))
    assert radii.numel() == 0 and float(alpha.abs().max()) == 0
    assert torch.allclose(color[:, 3, 4].cpu(), torch.tensor([0.1, 0.2, 0.3]))
    # all behind the camera / far off-screen: nothing rendered, zero gradients, no crash
    m = torch.tensor([[0, 0, 5.0], [0, 0, 1.75 - 0.1], [50.0, 0, 0]], device=dev, requires_grad=True)
    rot = torch.tensor([[1.0, 0, 0, 0]], device=dev).repeat(3, 1)
    color, radii, depth, alpha = R.GaussianRasterizer(rs)(means3D=m, means2D=z(3, 3), opacities=torch.full((3, 1), 0.5, device=dev),
                                                         colors_precomp=torch.ones(3, 3, device=dev),
                                                         scales=torch.full((3, 3), 0.01, device=dev), rotations=rot)
    assert int(radii.abs().sum()) == 0 and float(alpha.abs().max()) == 0
    color.sum().backward()
    assert float(m.grad.abs().max()) == 0


def test_inference_mode_and_reference_render_wrapper_contract(R, dev):
    """Render-only node path (nodes.py:1130-1163 runs under inference_mode) + the dict built at main_3DGS_renderer.py:942-949."""
    cl = O.make_cloud("D1", 4000, 1, seed=1)
    st = O.minicam_settings(O.orbit_camera(-10, 120, 1.75), 160, 96, 49.1, sh_degree=1)
    rs = _rs(R, st, dev, 1)
    ref, _, _, refa = O.rasterize(cl["means3D"], None, cl["shs"], None, cl["opacities"], cl["scales"], cl["rotations"], None, st)
    with torch.inference_mode():
        img, radii, depth, alpha = R.GaussianRasterizer(raster_settings=rs)(
            means3D=cl["means3D"].to(dev), means2D=torch.zeros(4000, 3, device=dev), shs=cl["shs"].to(dev),
            colors_precomp=None, opacities=cl["opacities"].to(dev), scales=cl["scales"].to(dev),
            rotations=cl["rotations"].to(dev), cov3D_precomp=None)
        img = img.clamp(0, 1)
        vis = radii > 0
    assert img.shape == (3, 96, 160) and depth.shape == (1, 96, 160) and alpha.shape == (1, 96, 160)
    assert radii.dtype == torch.int32 and vis.dtype == torch.bool
    assert float((img.cpu() - ref.clamp(0, 1)).abs().max()) < RGBA_ATOL
    assert float((alpha.cpu() - refa).abs().max()) < RGBA_ATOL


@pytest.mark.parametrize("kind,n", [("ball", 5000), ("ball", 60000), ("clusters", 40000), ("plane", 30000), ("dups", 20000)])
def test_knn_mean_dist2_matches_kdtree(R, dev, kind, n):
    """distCUDA2 replacement: all-pairs kernel below 8192 points, exact grid search above; both against a kd-tree."""
    g = torch.Generator().manual_seed(n)
    if kind == "ball":
        pts = O.make_cloud("D0", n, 0, seed=2)["means3D"]
    elif kind == "clusters":          # very uneven density: 20 tight blobs + a sparse background
        c = torch.rand(20, 3, generator=g) * 4 - 2
        pts = torch.cat([c[torch.randint(0, 20, (n - 500,), generator=g)] + 0.01 * torch.randn(n - 500, 3, generator=g),
                         torch.rand(500, 3, generator=g) * 20 - 10])
    elif kind == "plane":             # zero extent along z
        pts = torch.cat([torch.rand(n, 2, generator=g), torch.zeros(n, 1)], dim=1)
    else:                             # exact duplicates: distance 0 neighbours
        base = torch.rand(n // 4, 3, generator=g)
        pts = base.repeat(4, 1)[torch.randperm(n // 4 * 4, generator=g)]
    pts = pts.float().contiguous()
    got = R.knn_mean_dist2(pts.to(dev)).cpu().numpy()
    ref = O.knn_mean_dist2(pts.numpy())
    assert np.allclose(got, ref, rtol=1e-4, atol=1e-9)


# ---------------- multi-view step entries ---------------------------------------------------------------
def test_multiview_step_entries_agree_with_per_view_path(dev):
    from gs_b200 import camera, optim_step, synthetic
    N, V, W, H, deg = 20000, 5, 256, 144, 2
    cloud = synthetic.make_cloud("D1", N, deg, seed=5, device=dev)
    params = optim_step.PackedParams(cloud)
    vnp = camera.orbit_views(V, W, H)
    views = optim_step.ViewSet(vnp, W, H, deg, dev)
    dl_cpu = torch.rand(V, 5, H, W, generator=torch.Generator().manual_seed(7)) * 2 - 1
    dl = dl_cpu.to(dev)
    ia = torch.empty(V, 5, H, W, device=dev); ib = torch.empty(V, 5, H, W, device=dev)
    from gs_b200 import rasterizer as R
    assert R.get_tile_culling() == 1
    p1 = optim_step.step_device(params, views, dl, ia); g1 = params.grads.clone()   # per-view C entries: package lists
    try:
        for mode in (0, 1):
            R.set_tile_culling(mode)
            for _ in range(3):
                p2 = optim_step.step_device_pipelined(params, views, dl, ib); g2 = params.grads.clone()
                assert torch.equal(ia, ib)                             # images bit-identical with and without culling
                assert (p1 == p2) if mode == 0 else (0 < p2 < p1)
                assert float((g1 - g2).norm() / g1.norm()) < 1e-5      # atomics: summation order differs
            hs = optim_step.HostStep({k: v.cpu() for k, v in cloud.items()}, vnp, W, H, deg, dl_cpu)
            for _ in range(2):
                assert hs.run() == p2
                assert float((hs.grads.to(dev) - g1).norm() / g1.norm()) < 1e-5
    finally:
        R.set_tile_culling(1)
    # forward-only entry: same images, per-view radii equal to the single-view API's
    rad = torch.empty(V, N, dtype=torch.int32, device=dev)
    ic, pc = optim_step.render_views(params, views, radii=rad)
    assert torch.equal(ic, ia) and 0 < pc < p1
    for v in (0, V - 1):
        t = lambda a: torch.from_numpy(a).to(dev)
        rs = R.GaussianRasterizationSettings(H, W, float(vnp[v, 38]), float(vnp[v, 39]), t(vnp[v, 35:38].copy()), 1.0,
                                            t(vnp[v, :16].copy()).view(4, 4), t(vnp[v, 16:32].copy()).view(4, 4), deg,
                                            t(vnp[v, 32:35].copy()), False, False)
        with torch.no_grad():
            col, r1, dep, alp = R.GaussianRasterizer(rs)(means3D=cloud["means3D"], means2D=torch.zeros(N, 3, device=dev), shs=cloud["shs"],
                                                         opacities=cloud["opacities"], scales=cloud["scales"], rotations=cloud["rotations"])
        assert torch.equal(r1, rad[v]) and torch.equal(col, ic[v, :3]) and torch.equal(dep, ic[v, 3:4]) and torch.equal(alp, ic[v, 4:5])
    cam = camera.MiniCam(camera.orbit_camera(0, 0.0, 1.75), W, H, np.deg2rad(49.1),
                         2 * np.arctan(np.tan(np.deg2rad(49.1) / 2) * W / H), 0.01, 100.0, device=dev)
    assert np.allclose(vnp[0, :16], cam.world_view_transform.reshape(-1).cpu().numpy(), atol=1e-6)


@pytest.mark.parametrize("V", [1, 4, 9])
def test_host_buffer_step_bins_ahead_of_the_sh_upload_and_renders_the_same_bits(dev, V):
    """gs_b200_step_host starts projecting / sorting / binning when the geometry parameters are resident and fills the
    colours in when the SH block lands (V <= 8; beyond that it waits for the upload): images bit-identical to the
    device-resident step, gradients to summation order."""
    from gs_b200 import camera, optim_step, synthetic
    N, W, H, deg = 30000, 320, 176, 3
    cloud = synthetic.make_cloud("D1", N, deg, seed=9, device=dev)
    params = optim_step.PackedParams(cloud)
    vnp = camera.orbit_views(V, W, H)
    views = optim_step.ViewSet(vnp, W, H, deg, dev)
    dl_cpu = torch.rand(V, 5, H, W, generator=torch.Generator().manual_seed(3)) * 2 - 1
    img_dev = torch.empty(V, 5, H, W, device=dev)
    pairs = optim_step.step_device_pipelined(params, views, dl_cpu.to(dev), img_dev)
    g_dev = params.grads.clone()
    hs = optim_step.HostStep({k: v.cpu() for k, v in cloud.items()}, vnp, W, H, deg, dl_cpu)
    img_host = torch.empty(V, 5, H, W).pin_memory()
    for _ in range(3):
        img_host.fill_(-1.0)
        assert hs.run(images=img_host) == pairs
        assert torch.equal(img_host, img_dev.cpu())
        assert float((hs.grads.to(dev) - g_dev).norm() / g_dev.norm()) < 1e-5


def test_multiview_entries_chunking_and_empty_views(dev):
    """V = 18 > 16 views (two internal chunks), one view that sees nothing (all Gaussians behind the camera): the
    pipelined, hook, train and render entries agree with the per-view C entries."""
    from gs_b200 import camera, optim_step, synthetic
    N, V, W, H, deg = 3000, 18, 192, 176, 1
    cloud = synthetic.make_cloud("D1", N, deg, seed=9, device=dev)
    params = optim_step.PackedParams(cloud)
    vnp = camera.orbit_views(V, W, H).copy()
    vnp[5, 14] = -50.0                       # view 5: world->view z translation far negative => every z_view <= 0.2
    views = optim_step.ViewSet(vnp, W, H, deg, dev)
    dl = (torch.rand(V, 5, H, W, generator=torch.Generator().manual_seed(3)) * 2 - 1).to(dev)
    ia = torch.empty(V, 5, H, W, device=dev); ib = torch.empty_like(ia); ic = torch.empty_like(ia)
    optim_step.step_device(params, views, dl, ia); g1 = params.grads.clone()
    assert float(ia[5, 4].abs().max()) == 0.0                          # nothing rendered in the empty view
    optim_step.step_device_pipelined(params, views, dl, ib)
    assert torch.equal(ia, ib) and float((params.grads - g1).norm() / g1.norm()) < 1e-5
    rad = torch.empty(V, N, dtype=torch.int32, device=dev)
    optim_step.render_views(params, views, ic, rad)
    assert torch.equal(ia, ic) and int((rad[5] > 0).sum()) == 0 and int((rad[17] > 0).sum()) > 0
    # LGM-style call: precomputed colours instead of SHs (Gen_3D_Modules/LGM/core/gs.py:75-84)
    from gs_b200 import rasterizer as R
    cols = torch.rand(N, 3, generator=torch.Generator().manual_seed(8)).to(dev)
    id_, _ = optim_step.render_views(params, views, colors_precomp=cols)
    for v in (0, 5, 11):
        t = lambda a: torch.from_numpy(a).to(dev)
        rs = R.GaussianRasterizationSettings(H, W, float(vnp[v, 38]), float(vnp[v, 39]), t(vnp[v, 35:38].copy()), 1.0,
                                            t(vnp[v, :16].copy()).view(4, 4), t(vnp[v, 16:32].copy()).view(4, 4), deg,
                                            t(vnp[v, 32:35].copy()), False, False)
        with torch.no_grad():
            col, _, dep, alp = R.GaussianRasterizer(rs)(means3D=cloud["means3D"], means2D=torch.zeros(N, 3, device=dev), colors_precomp=cols,
                                                        opacities=cloud["opacities"], scales=cloud["scales"], rotations=cloud["rotations"])
        assert torch.equal(col, id_[v, :3]) and torch.equal(dep, id_[v, 3:4]) and torch.equal(alp, id_[v, 4:5])
    seen = []
    def fn(v, img, out):
        seen.append(v); out.copy_(dl[v])
    dlh = torch.empty_like(dl)
    optim_step.step_device_loss(params, views, fn, ic, dlh)
    assert seen == list(range(V)) and torch.equal(dlh, dl)
    assert float((params.grads - g1).norm() / g1.norm()) < 1e-5
    # train entry: compare its upstream gradients / loss with the single-view CUDA loss, its parameter gradients
    # with a plain step fed those upstream gradients
    ref = torch.rand(V, 3, H, W, generator=torch.Generator().manual_seed(4)).to(dev)
    msk = (torch.rand(V, 1, H, W, generator=torch.Generator().manual_seed(5)) > 0.3).float().to(dev)
    lv = torch.zeros(V, device=dev); dlt = torch.empty_like(dl)
    optim_step.step_device_train(params, views, ref, msk, 0.2, 3.0, 1.0 / V, ic, dlt, lv)
    gt = params.grads.clone()
    for v in (0, 5, 17):
        l1, d1 = optim_step.image_loss(ia[v].contiguous(), ref[v].contiguous(), msk[v].contiguous(), 0.2, 3.0, 1.0 / V)
        assert abs(float(l1) - float(lv[v])) <= 1e-6 * max(1.0, abs(float(l1)))
        assert float((d1 - dlt[v]).abs().max()) <= 1e-6 * float(d1.abs().max()) + 1e-12
    optim_step.step_device_pipelined(params, views, dlt)
    assert float((params.grads - gt).norm() / gt.norm()) < 1e-5


# ---------------- tile culling (optional tight tile lists) -----------------------------------------------
@pytest.mark.parametrize("kind,N,deg,W,H", [("D1", 3000, 2, 200, 120), ("D0", 50000, 3, 640, 360), ("big", 400, 0, 320, 200)])
def test_tile_culling_is_a_sublist_with_identical_images(R, dev, kind, N, deg, W, H):
    """Mode 2 drops (tile, splat) pairs that cannot reach alpha >= 1/255 in the tile: the culled list must be an
    order-preserving sub-list of the package's list per tile, and the images must not change by a single bit."""
    from gs_b200 import camera, synthetic
    if kind == "big":       # large, anisotropic splats (squares taller than 8 tiles fall back to the full square)
        g = torch.Generator().manual_seed(3)
        cloud = {"means3D": (torch.rand(N, 3, generator=g) - 0.5), "shs": torch.rand(N, 1, 3, generator=g),
                 "opacities": torch.rand(N, 1, generator=g) ** 3,
                 "scales": torch.exp(torch.rand(N, 3, generator=g) * 4 - 5), "rotations": torch.randn(N, 4, generator=g)}
        cloud = {k: v.to(dev).contiguous() for k, v in cloud.items()}
    else:
        cloud = synthetic.make_cloud(kind, N, deg, seed=11, device=dev)
    vnp = camera.orbit_views(3, W, H)
    t = lambda a: torch.from_numpy(a).to(dev)
    for v in range(3):
        rs = R.GaussianRasterizationSettings(H, W, float(vnp[v, 38]), float(vnp[v, 39]), t(vnp[v, 35:38].copy()), 1.0,
                                            t(vnp[v, :16].copy()).view(4, 4), t(vnp[v, 16:32].copy()).view(4, 4), deg,
                                            t(vnp[v, 32:35].copy()), False, False)
        out = {}
        try:
            for mode in (0, 2):
                R.set_tile_culling(mode)
                leaves = {k: x.clone().requires_grad_(True) for k, x in cloud.items()}
                fs = R.forward_with_state(rs, leaves["means3D"].detach(), leaves["opacities"].detach(), shs=leaves["shs"].detach(),
                                          scales=leaves["scales"].detach(), rotations=leaves["rotations"].detach())
                m2d = torch.zeros(N, 3, device=dev, requires_grad=True)
                color, radii, depth, alpha = R.GaussianRasterizer(rs)(
                    means3D=leaves["means3D"], means2D=m2d, shs=leaves["shs"], opacities=leaves["opacities"],
                    scales=leaves["scales"], rotations=leaves["rotations"])
                up = _upstream(H, W, 5)
                (color * up[0].to(dev)).sum().add((depth * up[1].to(dev)).sum()).add((alpha * up[2].to(dev)).sum()).backward()
                out[mode] = (fs, color.detach(), depth.detach(), alpha.detach(), radii,
                             [leaves[k].grad.clone() for k in NAMES] + [m2d.grad.clone()])
        finally:
            R.set_tile_culling(1)
        f0, f2 = out[0][0], out[2][0]
        for i in (1, 2, 3, 4):
            assert torch.equal(out[0][i], out[2][i])
        assert torch.equal(f0["color"], f2["color"]) and torch.equal(f0["final_T"], f2["final_T"])
        assert f2["num_rendered"] <= f0["num_rendered"]
        if kind != "big":
            assert f2["num_rendered"] < f0["num_rendered"]
        # per-tile sub-list check: walk both lists with two pointers
        r0, r2 = f0["ranges"].cpu().numpy().astype(np.int64), f2["ranges"].cpu().numpy().astype(np.int64)
        l0, l2 = f0["point_list"].cpu().numpy(), f2["point_list"].cpu().numpy()
        for tile in range(r0.shape[0]):
            a = l0[r0[tile, 0]:r0[tile, 1]]; b = l2[r2[tile, 0]:r2[tile, 1]]
            if b.size == 0:
                continue
            pos = np.flatnonzero(np.isin(a, b))
            assert pos.size == b.size and np.array_equal(a[pos], b), f"tile {tile}"
        for ga, gb, nm in zip(out[0][5], out[2][5], NAMES + ("means2D",)):
            # same terms, different atomic summation order (rotation/scale grads are sums of cancelling terms)
            # (D0 is isotropic: its rotation gradient is pure rounding noise around zero -> absolute floor)
            # The "big" cloud (screen-filling anisotropic splats, thousands of atomics per Gaussian, heavy cancellation)
            # shows the same ~1e-4..1e-3 run-to-run noise with culling off (scripts/dev/cull_check.py).
            tol = 5e-3 if kind == "big" else GRAD_RTOL
            assert float((ga - gb).norm()) <= tol * float(ga.norm()) + 1e-6, nm


# ---------------- full-size properties (BASELINE config 1: 1M Gaussians, 1080p) -----------------------
def test_full_size_properties_config1(dev):
    from gs_b200 import camera, optim_step, synthetic
    from gs_b200 import rasterizer as R
    N, W, H, deg = 1_000_000, 1920, 1080, 3
    cloud = synthetic.make_cloud("D0", N, deg, seed=0, device=dev)
    vnp = camera.orbit_views(1, W, H)
    t = lambda a: torch.from_numpy(a).to(dev)
    rs = R.GaussianRasterizationSettings(H, W, float(vnp[0, 38]), float(vnp[0, 39]), t(vnp[0, 35:38].copy()), 1.0,
                                        t(vnp[0, :16].copy()).view(4, 4), t(vnp[0, 16:32].copy()).view(4, 4), deg,
                                        t(vnp[0, 32:35].copy()), False, False)
    fs = R.forward_with_state(rs, cloud["means3D"], cloud["opacities"], shs=cloud["shs"], scales=cloud["scales"],
                              rotations=cloud["rotations"])
    P = fs["num_rendered"]
    assert P > N                                                   # K > 1 pairs per Gaussian at this density
    keys = fs["sorted_keys"]
    assert bool((keys[1:] >= keys[:-1]).all())                     # sortedness of the 64-bit keys
    # equal keys keep Gaussian-index order (stability)
    eq = keys[1:] == keys[:-1]
    pl = fs["point_list"].to(torch.int64)
    assert bool((pl[1:][eq] > pl[:-1][eq]).all())
    r = fs["ranges"].to(torch.int64)
    assert int((r[:, 1] - r[:, 0]).sum()) == P                    # ranges partition the list
    tiles = (keys >> 32)
    nz = r[:, 1] > r[:, 0]
    assert bool((tiles[r[nz, 0]] == torch.nonzero(nz).squeeze(1)).all())
    # every Gaussian's pair count equals its rect area: histogram of point_list == tiles implied by radii>0
    cnt = torch.bincount(pl, minlength=N)
    assert bool(((cnt > 0) == (fs["radii"] > 0)).all())
    # transmittance bookkeeping and bounds
    assert float((fs["alpha"][0] + fs["final_T"] - 1).abs().max()) < 1e-4
    assert bool((fs["n_contrib"].to(torch.int64) <= (r[:, 1] - r[:, 0]).max()).all())
    assert float(fs["color"].min()) >= 0 and bool(torch.isfinite(fs["color"]).all())
    # permutation invariance: shuffling the Gaussians leaves the image unchanged (depth ties aside)
    perm = torch.randperm(N, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    fs2 = R.forward_with_state(rs, cloud["means3D"][perm].contiguous(), cloud["opacities"][perm].contiguous(),
                               shs=cloud["shs"][perm].contiguous(), scales=cloud["scales"][perm].contiguous(),
                               rotations=cloud["rotations"][perm].contiguous())
    assert fs2["num_rendered"] == P
    assert float((fs2["color"] - fs["color"]).abs().max()) < 1e-4
    # backward is linear in the upstream gradient: grads(2 dL) == 2 grads(dL)
    params = optim_step.PackedParams(cloud)
    views = optim_step.ViewSet(vnp, W, H, deg, dev)
    dl = (torch.rand(1, 5, H, W, device=dev, generator=torch.Generator(device=dev).manual_seed(1)) * 2 - 1)
    optim_step.step_device_pipelined(params, views, dl); g1 = params.grads.clone()
    optim_step.step_device_pipelined(params, views, 2 * dl); g2 = params.grads.clone()
    assert bool(torch.isfinite(g1).all())
    assert float((g2 - 2 * g1).norm() / (2 * g1).norm()) < 1e-5


# ---------------- oracle parity AT the size the headline number is quoted on (config 1) ------------------------
def _oracle_settings_from_view(rec, W, H, deg):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    return O.Settings(H, W, float(rec[38]), float(rec[39]), t(rec[35:38]), 1.0, t(rec[0:16]).view(4, 4),
                      t(rec[16:32]).view(4, 4), deg, t(rec[32:35]))


@pytest.mark.parametrize("view_ids", [(0,), (3, 6)])
def test_config1_full_frame_keys_and_sampled_tile_composite_match_the_oracle(dev, R, view_ids):
    """BASELINE config 1 (1M Gaussians D0, SH 3, 1920x1080, the bench's orbit views).  Whole frame: radii, the sorted
    64-bit keys, point_list and ranges bit-exact against the oracle's preprocess + 64-bit stable sort.  64 sampled
    tiles including the densest: RGBA within 1e-4, n_contrib exact, and — with the upstream gradient restricted to
    those tiles — all parameter gradients within 1e-3, with tile culling OFF (the package's lists) and ON (the lists
    the benchmarked step walks)."""
    from gs_b200 import camera, synthetic
    N, W, H, deg = 1_000_000, 1920, 1080, 3
    # the oracle's per-tile tensor ops collapse with one thread per core of a 128-core host (bench.py measured 25x slower
    # than 8 threads): cap the intra-op threads for this test
    threads0 = torch.get_num_threads()
    torch.set_num_threads(min(threads0, 16))
    cloud = synthetic.make_cloud("D0", N, deg, seed=0, device=dev)
    cpu = {k: v.cpu() for k, v in cloud.items()}
    vnp = camera.orbit_views(8, W, H)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    mode0 = R.get_tile_culling()
    stats = []
    try:
        for v in view_ids:
            rec = vnp[v]
            st = _oracle_settings_from_view(rec, W, H, deg)
            rs = R.GaussianRasterizationSettings(H, W, float(rec[38]), float(rec[39]), t(rec[35:38]), 1.0, t(rec[0:16]).view(4, 4),
                                                t(rec[16:32]).view(4, 4), deg, t(rec[32:35]), False, False)
            # ---- oracle: whole-frame integer state
            leaf = {k: cpu[k].clone().requires_grad_(True) for k in NAMES}
            m2 = torch.zeros(N, 3, requires_grad=True)
            pre = O.preprocess(leaf["means3D"], leaf["scales"], leaf["rotations"], leaf["opacities"], leaf["shs"], None, None, m2, st)
            keys, vals = O.duplicate_with_keys_vectorised(pre)
            skeys, svals = O.sort_pairs(keys, vals)
            ranges = O.identify_tile_ranges(skeys, gx * gy)
            # ---- GPU, the package's tile lists (culling off)
            R.set_tile_culling(0)
            fs = R.forward_with_state(rs, cloud["means3D"], cloud["opacities"], shs=cloud["shs"], scales=cloud["scales"],
                                      rotations=cloud["rotations"])
            rad_bad = int((fs["radii"].cpu() != pre["radii"]).sum())
            stats.append(dict(view=v, what="radii", differ=rad_bad, pairs_gpu=int(fs["num_rendered"]), pairs_oracle=int(skeys.size)))
            assert rad_bad == 0, f"view {v}: {rad_bad} radii differ"
            assert fs["num_rendered"] == skeys.size
            assert np.array_equal(fs["sorted_keys"].cpu().numpy().view(np.uint64), skeys)
            assert np.array_equal(fs["point_list"].cpu().numpy().view(np.uint32), svals)
            assert np.array_equal(fs["ranges"].cpu().numpy().view(np.uint32), ranges)
            # ---- sampled tiles: the 8 densest + 56 seeded random non-empty ones
            length = (ranges[:, 1].astype(np.int64) - ranges[:, 0].astype(np.int64))
            dense = np.argsort(-length)[:8]
            nonempty = np.setdiff1d(np.flatnonzero(length > 0), dense)
            rng = np.random.RandomState(100 + v)
            tiles = sorted(set(dense.tolist()) | set(rng.choice(nonempty, 56, replace=False).tolist()))
            assert len(tiles) == 64
            color, depth, alpha, n_contrib, final_T = O.composite(pre, svals, ranges, st, tiles=tiles)
            mask = torch.zeros(H, W, dtype=torch.bool)
            for tl in tiles:
                yy, xx = O._tile_pixels(tl, gx, W, H, torch.float32)
                mask[yy, xx] = True
            dc, dd, da = _upstream(H, W, 7 + v)
            dc, dd, da = dc * mask, dd * mask, da * mask
            loss = (color * dc).sum() + (depth * dd).sum() + (alpha * da).sum()
            og = torch.autograd.grad(loss, [leaf[k] for k in NAMES] + [m2])
            for cull in (0, 2):
                R.set_tile_culling(cull)
                inp = {k: cloud[k].detach().clone().requires_grad_(True) for k in NAMES}
                g2 = torch.zeros(N, 3, device=dev, requires_grad=True)
                c, radii, d, a = R.GaussianRasterizer(rs)(means3D=inp["means3D"], means2D=g2, shs=inp["shs"], colors_precomp=None,
                                                          opacities=inp["opacities"], scales=inp["scales"],
                                                          rotations=inp["rotations"], cov3D_precomp=None)
                # Every pixel takes ~10^3 discrete decisions (alpha >= 1/255, T(1-alpha) < 1e-4) on values that differ from
                # the oracle's by an ulp or two (ex2.approx vs exp): over 16k pixels x ~10^3 splats a handful of pixels may
                # land on the other side of a threshold and then differ by up to alpha*T ~ 4e-3.  All but at most 4 pixels
                # per view must meet 1e-4; the outliers are bounded by one threshold splat (1e-2).
                for nm, gpu, ref in (("color", c, color), ("depth", d, depth), ("alpha", a, alpha)):
                    e = (gpu.detach().cpu() - ref.detach())[:, mask].abs().amax(dim=0)
                    bad = int((e >= RGBA_ATOL).sum())
                    stats.append(dict(view=v, cull=cull, what=nm, max_err=float(e.max()), pixels=int(e.numel()), over_1e4=bad))
                    assert bad <= 4 and float(e.max()) < 1e-2, f"view {v} cull {cull} {nm}: {bad} pixels over 1e-4, max {float(e.max())}"
                ((c * dc.to(dev)).sum() + (d * dd.to(dev)).sum() + (a * da.to(dev)).sum()).backward()
                for k, ref in zip(NAMES + ("means2D",), og):
                    got = (g2 if k == "means2D" else inp[k]).grad
                    if k == "rotations":      # D0 is isotropic: dL/drotation is rounding noise around zero on both sides
                        assert float(got.abs().max()) <= 1e-3 * float(inp["scales"].grad.abs().max()) + 1e-6
                        continue
                    rel = float((got.cpu().double() - ref.double()).norm() / ref.double().norm())
                    stats.append(dict(view=v, cull=cull, what="grad_" + k, rel=rel))
                    assert rel < GRAD_RTOL, f"view {v} cull {cull} grad {k}: {rel}"
            # n_contrib (list positions of the package's lists): exact on the sampled tiles
            R.set_tile_culling(0)
            nc_bad = int((fs["n_contrib"].cpu()[mask] != n_contrib[mask]).sum())
            stats.append(dict(view=v, what="n_contrib", pixels=int(mask.sum()), differ=nc_bad))
            assert nc_bad <= 4, f"view {v}: n_contrib differs on {nc_bad} pixels"
            del fs
    finally:
        R.set_tile_culling(mode0)
        torch.set_num_threads(threads0)
        out_dir = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
        if os.path.isdir(out_dir):
            import json
            with open(os.path.join(out_dir, "config1_parity_stats_%s.json" % "_".join(map(str, view_ids))), "w") as f:
                json.dump(stats, f, indent=1)


# ---------------- other callers of the rasterizer boundary (SURVEY 8f-3) ---------------------------------------------------
def test_triplane_gaussian_double_render_inside_an_fp32_autocast_region(dev, R):
    """TriplaneGaussian (Gen_3D_Modules/TriplaneGaussian/models/renderer.py:261-305) calls the rasterizer twice per view
    inside `torch.autocast(device_type, dtype=torch.float32)` nested in the model's fp16 autocast: once with colours
    (colors_precomp when cfg.use_rgb), once for the mask with colors_precomp = ones, bg = 0 and sh_degree 0.  Both
    calls must return fp32 4-tuples that match the oracle, the mask render equals the alpha output, and gradients flow."""
    N, W, H = 4000, 96, 80
    cl = O.make_cloud("D1", N, 0, seed=21)
    st = O.minicam_settings(O.orbit_camera(5, 65, 1.75), W, H, 49.1, sh_degree=0, bg=(0.3, 0.2, 0.1))
    cols = torch.rand(N, 3, generator=torch.Generator().manual_seed(1))
    ref_c, _, ref_d, ref_a = O.rasterize(cl["means3D"], None, None, cols, cl["opacities"], cl["scales"], cl["rotations"], None, st)
    inp = {k: cl[k].to(dev).requires_grad_(True) for k in ("means3D", "opacities", "scales", "rotations")}
    colsd = cols.to(dev).requires_grad_(True)
    m2 = torch.zeros(N, 3, device=dev, requires_grad=True)
    with torch.autocast("cuda", dtype=torch.float16):
        junk = torch.mm(torch.ones(4, 4, device=dev), torch.ones(4, 4, device=dev))      # the surrounding model runs in fp16
        assert junk.dtype == torch.float16
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            with torch.autocast(device_type="cuda", dtype=torch.float32):
                img, radii, depth, alpha = R.GaussianRasterizer(_rs(R, st, dev, 0))(
                    means3D=inp["means3D"], means2D=m2, shs=None, colors_precomp=colsd, opacities=inp["opacities"],
                    scales=inp["scales"], rotations=inp["rotations"], cov3D_precomp=None)
            st0 = O.minicam_settings(O.orbit_camera(5, 65, 1.75), W, H, 49.1, sh_degree=0, bg=(0.0, 0.0, 0.0))
            with torch.autocast(device_type="cuda", dtype=torch.float32):
                mask, radii2, depth2, alpha2 = R.GaussianRasterizer(_rs(R, st0, dev, 0))(
                    means3D=inp["means3D"], means2D=m2, colors_precomp=torch.ones_like(inp["means3D"]), opacities=inp["opacities"],
                    scales=inp["scales"], rotations=inp["rotations"], cov3D_precomp=None)
    for t in (img, depth, alpha, mask):
        assert t.dtype == torch.float32
    assert float((img.detach().cpu() - ref_c).abs().max()) < RGBA_ATOL
    assert float((depth.detach().cpu() - ref_d).abs().max()) < RGBA_ATOL and float((alpha.detach().cpu() - ref_a).abs().max()) < RGBA_ATOL
    assert torch.equal(radii, radii2)
    assert float((mask - alpha2.expand_as(mask)).abs().max()) < 1e-6                    # ones through the blend = coverage
    (img.sum() + mask.sum()).backward()
    assert all(bool(torch.isfinite(v.grad).all()) and float(v.grad.abs().sum()) > 0 for v in inp.values())


def test_trellis_supersampled_render_then_antialiased_downsample(dev, R):
    """TRELLIS (Gen_3D_Modules/TRELLIS/trellis/renderers/gaussian_render.py:211-230): render at resolution * ssaa with
    overridden colours, then F.interpolate(..., mode='bilinear', antialias=True) down to `resolution`."""
    import torch.nn.functional as F
    N, res, ssaa = 5000, 48, 2
    cl = O.make_cloud("D1", N, 0, seed=33)
    st = O.minicam_settings(O.orbit_camera(-10, 200, 1.75), res * ssaa, res * ssaa, 40.0, sh_degree=0, bg=(1.0, 1.0, 1.0))
    cols = torch.rand(N, 3, generator=torch.Generator().manual_seed(2))
    ref_c, _, _, _ = O.rasterize(cl["means3D"], None, None, cols, cl["opacities"], cl["scales"], cl["rotations"], None, st)
    ref = F.interpolate(ref_c[None], size=(res, res), mode="bilinear", align_corners=False, antialias=True).squeeze()
    img, radii, depth, alpha = R.GaussianRasterizer(_rs(R, st, dev, 0))(
        means3D=cl["means3D"].to(dev), means2D=torch.zeros(N, 3, device=dev), shs=None, colors_precomp=cols.to(dev),
        opacities=cl["opacities"].to(dev), scales=cl["scales"].to(dev), rotations=cl["rotations"].to(dev), cov3D_precomp=None)
    got = F.interpolate(img[None], size=(res, res), mode="bilinear", align_corners=False, antialias=True).squeeze()
    assert got.shape == (3, res, res) and float((got.cpu() - ref).abs().max()) < RGBA_ATOL


def test_in_place_parameter_update_before_backward_is_detected(dev, R):
    """The autograd node saves its tensor inputs with save_for_backward: an optimizer.step()-style in-place update between
    forward and a retained backward raises autograd's version error instead of returning gradients that pair the new
    parameters with the old binning state."""
    N, W, H = 500, 48, 48
    cl = O.make_cloud("D1", N, 0, seed=9)
    st = O.minicam_settings(O.orbit_camera(0, 0, 1.75), W, H, 49.1, sh_degree=0)
    inp = {k: cl[k].to(dev).requires_grad_(True) for k in NAMES}
    img, _, _, _ = R.GaussianRasterizer(_rs(R, st, dev, 0))(means3D=inp["means3D"], means2D=torch.zeros(N, 3, device=dev), shs=inp["shs"],
                                                             colors_precomp=None, opacities=inp["opacities"], scales=inp["scales"],
                                                             rotations=inp["rotations"], cov3D_precomp=None)
    with torch.no_grad():
        inp["means3D"].add_(0.01)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        img.sum().backward()
