"""GPU tests of the optimisation-step kernels and the native trainer (rows a6/a8/a9, SURVEY §8f):
fused activation, fused chain-rule+Adam vs torch.optim.Adam, densification statistics and rules, a short fit."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import ROOT  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def test_activate_matches_reference_activations(dev):
    from gs_b200 import _lib
    N = 5000
    g = torch.Generator(device="cpu").manual_seed(0)
    ro, rs, rr = torch.randn(N, 1, generator=g).to(dev), torch.randn(N, 3, generator=g).to(dev), torch.randn(N, 4, generator=g).to(dev)
    o, s, r = torch.empty_like(ro), torch.empty_like(rs), torch.empty_like(rr)
    _lib.check(_lib.lib.gs_b200_activate(N, _ptr(ro), _ptr(rs), _ptr(rr), _ptr(o), _ptr(s), _ptr(r), None))
    assert torch.allclose(o, torch.sigmoid(ro), atol=1e-6) and torch.allclose(s, torch.exp(rs), rtol=1e-6)
    assert torch.allclose(r, torch.nn.functional.normalize(rr), atol=1e-6)


@pytest.mark.parametrize("M", [1, 4, 9])
def test_fused_adam_matches_torch_adam_through_activations(dev, M):
    """training_setup (main_3DGS_renderer.py:435-453): six groups, eps=1e-15; gradients arrive wrt ACTIVATED values.
    M = 1 and 9 (rows of 3 and 27 floats) make the 128-bit SH pass straddle Gaussian rows: the dc / rest learning rates
    must follow the coefficient, not the position inside the float4."""
    from gs_b200 import _lib
    N = 3000
    g = torch.Generator(device="cpu").manual_seed(1)
    sizes = [3 * N, 3 * M * N, N, 3 * N, 4 * N]
    raw = torch.randn(sum(sizes), generator=g).to(dev) * 0.5
    m1 = torch.zeros_like(raw); m2 = torch.zeros_like(raw)
    lrs = np.array([1.6e-3, 2.5e-3, 1.25e-4, 0.05, 0.005, 0.001], dtype=np.float32)

    def split(buf):
        o = 0; out = []
        for s, shp in zip(sizes, [(N, 3), (N, M, 3), (N, 1), (N, 3), (N, 4)]):
            out.append(buf[o:o + s].view(*shp)); o += s
        return out
    xyz, shs, op, sc, ro = [t.clone().requires_grad_(True) for t in split(raw)]
    dc = shs.detach()[:, :1].clone().requires_grad_(True); rest = shs.detach()[:, 1:].clone().requires_grad_(True)
    opt = torch.optim.Adam([{"params": [xyz], "lr": float(lrs[0])}, {"params": [dc], "lr": float(lrs[1])}, {"params": [rest], "lr": float(lrs[2])},
                            {"params": [op], "lr": float(lrs[3])}, {"params": [sc], "lr": float(lrs[4])}, {"params": [ro], "lr": float(lrs[5])}],
                           lr=0.0, eps=1e-15)
    for step in range(1, 4):
        gact = torch.randn(sum(sizes), generator=g).to(dev)            # dL/d(activated) packed
        gx, gs_, go, gsc, gr = split(gact)
        opt.zero_grad()
        act = (xyz * gx).sum() + (torch.cat([dc, rest], 1) * gs_).sum() + (torch.sigmoid(op) * go).sum() + \
              (torch.exp(sc) * gsc).sum() + (torch.nn.functional.normalize(ro) * gr).sum()
        act.backward(); opt.step()
        _lib.check(_lib.lib.gs_b200_adam_step(N, M, C.c_void_p(lrs.ctypes.data), 0.9, 0.999, 1e-15, step, 1.0, _ptr(gact), _ptr(raw),
                                              _ptr(m1), _ptr(m2), None))
        ref = torch.cat([xyz.detach().reshape(-1), torch.cat([dc, rest], 1).detach().reshape(-1), op.detach().reshape(-1),
                         sc.detach().reshape(-1), ro.detach().reshape(-1)])
        assert float((raw - ref).abs().max()) < 2e-5, step


def test_densify_stats(dev):
    from gs_b200 import _lib
    N = 1000
    g2 = torch.randn(N, 3, device=dev); radii = torch.randint(-1, 5, (N,), dtype=torch.int32, device=dev)
    acc = torch.rand(N, device=dev); den = torch.rand(N, device=dev).round(); mr = torch.rand(N, device=dev) * 3
    a0, d0, m0 = acc.clone(), den.clone(), mr.clone()
    _lib.check(_lib.lib.gs_b200_densify_stats(N, _ptr(g2), _ptr(radii), _ptr(acc), _ptr(den), _ptr(mr), None))
    vis = radii > 0
    assert torch.allclose(acc, torch.where(vis, a0 + g2[:, :2].norm(dim=1), a0), atol=1e-6)
    assert torch.equal(den, torch.where(vis, d0 + 1, d0)) and torch.equal(mr, torch.where(vis, torch.maximum(m0, radii.float()), m0))


def test_densify_and_prune_rules(dev):
    """Clone / split / prune decisions follow main_3DGS_renderer.py:641-668,752-781 on a seeded state."""
    from gs_b200 import trainer
    tr = trainer.GaussianTrainer(trainer.TrainParams(num_pts=2000, sh_degree=1), device=dev, seed=3)
    N = tr.N
    g = torch.Generator(device="cpu").manual_seed(0)
    tr.grad_accum.copy_(torch.rand(N, generator=g).to(dev) * 4e-4); tr.denom.fill_(1.0); tr.denom[:50] = 0.0       # NaN grads -> 0
    tr.v["scaling"].copy_(torch.log(torch.rand(N, 3, generator=g).to(dev) * 0.08 + 1e-3))                          # some > 0.01*4, some > 0.4? no
    tr.v["scaling"][:20] = float(np.log(0.5))                                                                        # too big in world space -> pruned
    tr.v["opacity"][100:140] = -8.0                                                                                  # opacity < 0.005 -> pruned
    tr.max_radii2D[200:230] = 5.0                                                                                    # big on screen: NOT pruned (inert rule)
    grads = tr.grad_accum / tr.denom; grads[grads.isnan()] = 0
    scal = torch.exp(tr.v["scaling"]).max(1).values
    big = scal > 0.01 * 4.0
    n_clone = int(((grads >= 2e-4) & ~big).sum()); n_split = int(((grads >= 2e-4) & big).sum())
    opac = torch.sigmoid(tr.v["opacity"]).squeeze(1)
    # (max_radii2D is reset before the reference's prune() reads it -> the screen-size rule is inert; test_golden_training.py)
    pruned_old = ((grads >= 2e-4) & big) | (opac < 0.005) | (scal > 0.4)
    xyz_before = tr.v["xyz"].clone(); m1_before = tr._views(tr.m1, N)["xyz"].clone()
    info = tr.densify_and_prune(2e-4, 0.005, 4.0, 1.0, generator=None)
    assert info["cloned"] == n_clone and info["split"] == n_split and info["pruned"] == int(pruned_old.sum())
    kept = int((~pruned_old).sum())
    assert tr.N <= kept + n_clone + 2 * n_split and tr.N >= kept
    assert torch.equal(tr.v["xyz"][:kept], xyz_before[~pruned_old])                  # survivors keep order and values
    assert float(tr._views(tr.m1, tr.N)["xyz"][kept:].abs().max()) == 0.0            # new points start with zero Adam state
    assert float(tr.grad_accum.abs().max()) == 0 and tr.radii.numel() == tr.N
    tr.reset_opacity()
    assert float(torch.sigmoid(tr.v["opacity"]).max()) <= 0.01 + 1e-6


def test_short_fit_reduces_loss(dev):
    """End-to-end: render a target from a 'ground-truth' cloud, fit a fresh random cloud for a few steps."""
    from gs_b200 import camera, trainer
    W = H = 192
    V = 4
    views = camera.orbit_views(V, W, H)
    gt = trainer.GaussianTrainer(trainer.TrainParams(num_pts=3000, sh_degree=1), device=dev, seed=7)
    gt.v["shs"][:, 0, :] = torch.rand(gt.N, 3, device=dev) * 2 - 0.5
    gt.v["opacity"].fill_(1.5)
    gt.v["scaling"].add_(0.7)
    target = gt.render_views(views, W, H)
    ref_img = target[:, :3].clamp(0, 1).contiguous(); ref_mask = (target[:, 4:5] > 0.5).float()
    tr = trainer.GaussianTrainer(trainer.TrainParams(num_pts=3000, sh_degree=1, density_start_iter=10 ** 9), device=dev, seed=11)
    ls = [tr.train_step(views, W, H, ref_img, ref_mask) for _ in range(40)]
    assert all(np.isfinite(ls)) and ls[-1] < 0.8 * ls[0], (ls[0], ls[-1])
    from gs_b200 import losses
    l_torch = tr.train_step(views, W, H, ref_img, ref_mask, loss_fn=lambda i, a, r, m: losses.training_loss(i, a, r, m, 0.2, 3.0))
    assert np.isfinite(l_torch) and l_torch < 1.2 * ls[-1]
    assert tr.step_count == 41 and bool(torch.isfinite(tr.raw).all())


def test_pipelined_loss_step_equals_two_pass_step(dev):
    """forward -> loss -> backward inside the pipeline (gs_b200_step_device_hook) gives the same images, loss and
    gradients as: forward all views (gs_b200_render_views), torch loss on the batch, gs_b200_step_device."""
    from gs_b200 import camera, losses, optim_step, trainer
    W, H, V = 208, 176, 5
    views = camera.orbit_views(V, W, H)
    tr = trainer.GaussianTrainer(trainer.TrainParams(num_pts=4000, sh_degree=2), device=dev, seed=5)
    tr.v["shs"][:, 0, :] = torch.rand(tr.N, 3, device=dev)
    tr.v["opacity"].fill_(0.5)
    g = torch.Generator().manual_seed(1)
    ref_img = torch.rand(V, 3, H, W, generator=g).to(dev); ref_mask = (torch.rand(V, 1, H, W, generator=g) > 0.4).float().to(dev)
    radii = torch.empty(V, tr.N, dtype=torch.int32, device=dev)
    imgs_a = tr.render_views(views, W, H, radii=radii).clone()
    x = imgs_a.clone().requires_grad_(True)
    loss = losses.training_loss(x[:, :3].clamp(0, 1), x[:, 4:5], ref_img, ref_mask, 0.2, 3.0)
    loss.backward()
    optim_step.step_device_pipelined(tr._cloud(), tr._viewset(views, W, H), x.grad.contiguous())
    g_a = tr.grads.clone()
    per_view = torch.zeros(V, device=dev)

    def fn(v, img, dl):
        y = img.detach().clone().requires_grad_(True)
        l = losses.training_loss(y[None, :3].clamp(0, 1), y[None, 4:5], ref_img[v:v + 1], ref_mask[v:v + 1], 0.2, 3.0) / V
        l.backward(); dl.copy_(y.grad); per_view[v] = l.detach()
    imgs_b = tr.forward_backward(views, W, H, fn)
    assert torch.equal(imgs_a, imgs_b)
    assert abs(float(per_view.sum()) - float(loss)) < 1e-5 * max(1.0, abs(float(loss)))
    assert float((tr.grads - g_a).norm() / g_a.norm()) < 1e-4
    assert torch.equal(tr.radii, radii[V - 1]) and int((radii > 0).sum()) > 0
    # native path: the same loss as CUDA kernels inside the pipeline
    imgs_c = torch.empty_like(imgs_a); dl_c = torch.empty_like(imgs_a); lv = torch.zeros(V, device=dev)
    tr.activate()
    optim_step.step_device_train(tr._cloud(), tr._viewset(views, W, H), ref_img, ref_mask, 0.2, 3.0, 1.0 / V, imgs_c, dl_c, lv)
    assert torch.equal(imgs_c, imgs_a)
    assert abs(float(lv.sum()) - float(loss)) < 1e-5 * max(1.0, abs(float(loss)))
    assert float((dl_c - x.grad).abs().max()) <= 2e-4 * float(x.grad.abs().max())
    assert float((tr.grads - g_a).norm() / g_a.norm()) < 1e-3
    # a failing hook surfaces as the original Python exception, and the library stays usable
    def bad(v, img, dl):
        raise KeyError("boom")
    with pytest.raises(KeyError):
        tr.forward_backward(views, W, H, bad)
    # a hook that re-enters the step entries is refused (per-thread pipeline state), not silently corrupted
    def reenter(v, img, dl):
        tr.render_views(views, W, H)
    with pytest.raises(RuntimeError, match="re-entrant"):
        tr.forward_backward(views, W, H, reenter)
    assert torch.equal(tr.render_views(views, W, H), imgs_a)


@pytest.mark.parametrize("H,W,ls", [(176, 200, 0.2), (270, 480, 0.2), (163, 161, 1.0), (64, 48, 0.0)])
def test_cuda_image_loss_matches_torch(dev, H, W, ls):
    """gs_b200_image_loss (L1 + alpha MSE + MS-SSIM and the gradient) against the torch restatement + autograd."""
    from gs_b200 import losses, optim_step
    g = torch.Generator().manual_seed(H * 1000 + W)
    ref = torch.rand(3, H, W, generator=g).to(dev)
    img = torch.cat([ref.cpu() + 0.25 * torch.randn(3, H, W, generator=g), torch.rand(1, H, W, generator=g), torch.rand(1, H, W, generator=g)]).to(dev)
    img[:3, :8] = -0.2; img[:3, 8:16] = 1.3                     # rows outside [0,1]: clamp blocks their gradient
    mask = torch.rand(1, H, W, generator=g).to(dev); mask[:, :, : W // 3] = 1.0; mask[:, H // 2:, W // 2:] = 0.0
    x = img.clone().requires_grad_(True)
    lt = losses.training_loss(x[None, :3].clamp(0, 1), x[None, 4:5], ref[None], mask[None], ls, 3.0) * 0.37
    lt.backward()
    lc, dl = optim_step.image_loss(img.contiguous(), ref.contiguous(), mask.contiguous(), ls, 3.0, 0.37)
    assert abs(float(lc) - float(lt)) <= 1e-5 * max(1.0, abs(float(lt)))
    assert float(dl[3].abs().max()) == 0.0
    for c, name in ((slice(0, 3), "rgb"), (slice(4, 5), "alpha")):
        ref_g = x.grad[c]
        assert float((dl[c] - ref_g).abs().max()) <= 2e-4 * float(ref_g.abs().max()) + 1e-12, name
    if ls > 0:
        with pytest.raises(RuntimeError):
            optim_step.image_loss(img[:, :100, :100].contiguous(), ref[:, :100, :100].contiguous(), mask[:, :100, :100].contiguous(), ls)


def test_training_loop_with_densification(dev):
    from gs_b200 import camera, trainer
    W = H = 176
    V = 3
    views = camera.orbit_views(V, W, H)
    gt = trainer.GaussianTrainer(trainer.TrainParams(num_pts=2000, sh_degree=1), device=dev, seed=7)
    gt.v["shs"][:, 0, :] = torch.rand(gt.N, 3, device=dev) * 2 - 0.5
    gt.v["opacity"].fill_(1.5); gt.v["scaling"].add_(0.7)
    target = gt.render_views(views, W, H)
    ref_img = target[:, :3].clamp(0, 1).contiguous(); ref_mask = (target[:, 4:5] > 0.5).float()
    tr = trainer.GaussianTrainer(trainer.TrainParams(num_pts=2000, sh_degree=1, density_start_iter=5, densification_interval=10,
                                                     densify_grad_threshold=1e-6, opacity_reset_interval=10 ** 9), device=dev, seed=11)
    n0 = tr.N
    ls = [tr.train_step(views, W, H, ref_img, ref_mask) for _ in range(25)]
    assert all(np.isfinite(ls))
    assert tr.N != n0                                     # statistics were collected (radii > 0) and acted upon
    assert bool(torch.isfinite(tr.raw).all()) and tr.radii.numel() == tr.N


def test_training_steps_reproduce_the_reference_loop(dev):
    """End to end: GaussianSplatting3D.training (main_3DGS.py:129-232) was executed from the reference source on the CPU for
    five steps (its own GaussianModel, renderer wrapper, camera controller, loss composition and Adam; rasterizer = the
    oracle, MS-SSIM = gs_b200/losses.py; tests/golden/make_golden_training.py -> ref_loop.npz).  Replaying the same view /
    background draws through GaussianTrainer.train_step — CUDA rasterizer forward/backward, CUDA loss, fused Adam — must land
    on the same raw parameters after every optimizer step (measured: <= 9e-6 absolute after five steps)."""
    import os
    from conftest import GOLDEN
    from gs_b200 import trainer
    G = np.load(os.path.join(GOLDEN, "ref_loop.npz"))
    N, deg, K = int(G["N"]), int(G["deg"]), int(G["K"]); H, W = int(G["HW"][0]), int(G["HW"][1])
    tr = trainer.GaussianTrainer(trainer.TrainParams(num_pts=N, sh_degree=deg, density_start_iter=10 ** 9), device=dev, seed=0)
    t = lambda k: torch.from_numpy(G[k]).to(dev)
    tr.v["xyz"].copy_(t("init_xyz")); tr.v["shs"].copy_(torch.cat([t("init_f_dc"), t("init_f_rest")], 1))
    tr.v["opacity"].copy_(t("init_opacity")); tr.v["scaling"].copy_(t("init_scaling")); tr.v["rotation"].copy_(t("init_rotation"))
    tr.m1.zero_(); tr.m2.zero_(); tr.step_count = 0
    # the fixture's reference images / masks are the next draws of its generator (seed 3) after the trained-like state
    g = torch.Generator().manual_seed(3)
    for shape in ((N, 3), (N, 4), (N, 1, 3), (N, (deg + 1) ** 2 - 1, 3), (N, 1)):
        torch.randn(*shape, generator=g)
    ref_imgs = torch.stack([torch.rand(H, W, 3, generator=g) for _ in range(3)]).permute(0, 3, 1, 2).contiguous()
    ref_masks = torch.stack([(torch.rand(H, W, generator=g) > 0.35).float() for _ in range(3)])[:, None].contiguous()
    assert float(ref_imgs.double().sum()) == float(G["ref_imgs_sum"]) and float(ref_masks.double().sum()) == float(G["ref_masks_sum"])
    ref_imgs, ref_masks = ref_imgs.to(dev), ref_masks.to(dev)
    moved = 0.0
    for s in range(K):
        i = int(G["idx"][s])
        rec = np.zeros((1, 40), dtype=np.float32)
        rec[0, :16] = G["step_view"][s].reshape(-1); rec[0, 16:32] = G["step_proj"][s].reshape(-1)
        rec[0, 32:35] = G["step_campos"][s]; rec[0, 35:38] = G["step_bg"][s]; rec[0, 38:40] = G["step_tan"][s]
        loss = tr.train_step(rec, W, H, ref_imgs[i:i + 1].contiguous(), ref_masks[i:i + 1].contiguous())
        assert np.isfinite(loss)
        ref = {"xyz": G["after_xyz"][s], "shs": np.concatenate([G["after_f_dc"][s], G["after_f_rest"][s]], 1),
               "opacity": G["after_opacity"][s], "scaling": G["after_scaling"][s], "rotation": G["after_rotation"][s]}
        lrs = {"xyz": 1.6e-3, "shs": 0.0025, "opacity": 0.05, "scaling": 0.005, "rotation": 0.001}
        for k, r in ref.items():
            d = np.abs(tr.v[k].cpu().numpy() - r)
            # Measured: every element within 9e-6.  Adam turns the SIGN of a gradient into a step of size lr, so an element
            # whose gradient is pure summation noise (atomics order) could legitimately differ by 2 lr per step; tolerate
            # at most 0.1 % such elements, bounded by that worst case, so the test cannot flake on one of them.
            assert float((d > 5e-5).mean()) <= 1e-3 and float(d.max()) <= 2.0 * lrs[k] * (s + 1) + 5e-5, (s, k, float(d.max()))
        moved = max(moved, float(np.abs(G["after_opacity"][s] - G["init_opacity"]).max()))
    assert moved > 0.05                     # the parameters really moved (opacity lr 0.05 per step), this is not 0 == 0


def test_cuda_densification_reproduces_the_reference_model_fixture_and_is_fast(dev):
    """gs_b200_densify_plan / _apply (stream compaction in the packed layout) against tests/golden/ref_training.npz — the
    state the REFERENCE's GaussianModel.densify_and_prune (main_3DGS_renderer.py:543-688,752-781) left behind on the same
    inputs, with the same torch.normal draws: parameters, both Adam moments, row order, zeroed statistics.  Then the
    cost at config-1 scale: a densification of 1M Gaussians (compaction of 3 x 59 floats per row) makes no device
    allocation when the result fits the capacity and waits for the device once (the read of the counts)."""
    import os
    import warnings
    from conftest import GOLDEN
    from gs_b200 import trainer
    G = np.load(os.path.join(GOLDEN, "ref_training.npz"), allow_pickle=False)
    N, deg = G["pre_xyz"].shape[0], 1
    tr = trainer.GaussianTrainer.__new__(trainer.GaussianTrainer)
    tr.p = trainer.TrainParams(sh_degree=deg); tr.device = dev; tr.M = (deg + 1) ** 2; tr.step_count = 0
    tr._alloc(N)
    t = lambda k: torch.from_numpy(G[k]).to(dev)
    tr.v["xyz"].copy_(t("pre_xyz")); tr.v["opacity"].copy_(t("pre_opacity")); tr.v["scaling"].copy_(t("pre_scaling")); tr.v["rotation"].copy_(t("pre_rotation"))
    tr.v["shs"].copy_(torch.cat([t("pre_f_dc"), t("pre_f_rest")], dim=1))
    m1, m2 = tr._views(tr.m1, N), tr._views(tr.m2, N)
    for k in ("xyz", "opacity", "scaling", "rotation"):
        m1[k].copy_(t("m1_" + k)); m2[k].copy_(t("m2_" + k))
    m1["shs"].copy_(torch.cat([t("m1_f_dc"), t("m1_f_rest")], dim=1)); m2["shs"].copy_(torch.cat([t("m2_f_dc"), t("m2_f_rest")], dim=1))
    tr.grad_accum.copy_(t("grad_accum").squeeze(1)); tr.denom.copy_(t("denom").squeeze(1)); tr.max_radii2D.copy_(t("max_radii2D"))
    # the reference drew torch.normal(mean=0, std=stds) for [2 x split parents, 3]: the same standard-normal stream, unscaled
    g = tr.grad_accum / tr.denom; g[g.isnan()] = 0
    n_split = int(((g >= 2e-4) & (torch.exp(tr.v["scaling"]).max(1).values > 0.01 * 4.0)).sum())
    torch.manual_seed(int(G["dens_seed"]))
    z = torch.empty(2 * n_split, 3).normal_()
    info = tr.densify_and_prune(2e-4, 0.005, 4.0, 1.0, normal_samples=z)
    assert tr.N == G["dens_xyz"].shape[0] == info["n"] and info["n_before"] == N and info["split"] == n_split
    ref_shs = np.concatenate([G["dens_f_dc"], G["dens_f_rest"]], axis=1)
    for mine, ref in (("xyz", G["dens_xyz"]), ("opacity", G["dens_opacity"]), ("scaling", G["dens_scaling"]), ("rotation", G["dens_rotation"]), ("shs", ref_shs)):
        assert np.allclose(tr.v[mine].cpu().numpy(), ref, rtol=1e-5, atol=1e-6), mine
    m1, m2 = tr._views(tr.m1, tr.N), tr._views(tr.m2, tr.N)
    for k in ("xyz", "opacity", "scaling", "rotation"):
        assert np.array_equal(m1[k].cpu().numpy(), G["dens_m1_" + k]) and np.array_equal(m2[k].cpu().numpy(), G["dens_m2_" + k]), k
    assert np.array_equal(m1["shs"].cpu().numpy(), np.concatenate([G["dens_m1_f_dc"], G["dens_m1_f_rest"]], axis=1))
    assert float(tr.grad_accum.abs().max()) == 0 and float(tr.denom.abs().max()) == 0 and float(tr.max_radii2D.abs().max()) == 0
    # ---- config-1 scale: 1M Gaussians, SH degree 3
    big = trainer.GaussianTrainer(trainer.TrainParams(num_pts=1_000_000, sh_degree=3), device=dev, seed=0)
    gen = torch.Generator(device="cpu").manual_seed(0)
    acc = (torch.rand(big.N, generator=gen) * 4e-4).to(dev)
    big._alloc_grow(int(1.6 * big.N)); big._bind(big.N, zero=False)          # head room, as after the first growth
    big._densify_workspace()                                                  # plan arrays live with the capacity
    for it in range(3):
        n0 = big.N
        big.grad_accum.copy_(acc[:n0] if acc.numel() >= n0 else torch.rand(n0, device=dev) * 4e-4); big.denom.fill_(1.0)
        big.v["opacity"][: n0 // 20] = -8.0                                    # 5 % pruned
        cap0 = big._cap
        torch.cuda.synchronize()
        allocs0 = torch.cuda.memory_stats(dev)["allocation.all.allocated"]
        with warnings.catch_warnings(record=True) as syncs:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                info = big.densify_and_prune(2e-4, 0.005, 4.0, 1.0)
            finally:
                torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
        assert info["cloned"] > 1000 and info["pruned"] >= n0 // 20 and big.N == info["n"]
        # the host waits for the device once (the 40-byte read of the counts)
        n_sync = sum("called a synchronizing CUDA operation" in str(w.message) for w in syncs)
        assert n_sync <= 1, [str(w.message) for w in syncs]
        if big._cap == cap0:                      # no capacity growth in this densification: no device allocation at all
            assert torch.cuda.memory_stats(dev)["allocation.all.allocated"] == allocs0
        acc = torch.rand(big.N, generator=gen).to(dev) * 4e-4
