"""The composite backward adds the four quadrant partials of each (tile, splat) inside the CTA, in fp64 and in a fixed
warp order, before one set of fp64 reds per (tile, splat) into SplatGrad.  These tests pin what that must keep: the
sums are the per-quadrant sums (to fp64 rounding), and two runs give the same gradients."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import gs_oracle as O

pytestmark = pytest.mark.gpu
NAMES = ("means3D", "shs", "opacities", "scales", "rotations")
GRAD_RTOL = 1e-3
CANCEL_GOLDEN = os.path.join(GOLDEN, "composite_combine_grads.npz")
N_CANCEL, W_CANCEL, H_CANCEL, V_CANCEL, DEG_CANCEL, ROWS_CANCEL = 200_000, 1920, 1080, 2, 0, 4096


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def cancelling_case(dev):
    """D0 cloud (isotropic scales, identity rotations: every rotation gradient is a sum of cancelling terms), two orbit
    views at 1080p, seeded upstream gradients.  Returns a function that runs the step and returns the packed
    gradients."""
    from gs_b200 import camera, optim_step, synthetic
    cloud = synthetic.make_cloud("D0", N_CANCEL, DEG_CANCEL, seed=11, device=dev)
    params = optim_step.PackedParams(cloud)
    views = optim_step.ViewSet(camera.orbit_views(V_CANCEL, W_CANCEL, H_CANCEL), W_CANCEL, H_CANCEL, DEG_CANCEL, dev)
    g = torch.Generator().manual_seed(12)
    dl = torch.rand(V_CANCEL, 5, H_CANCEL, W_CANCEL, generator=g) * 2 - 1
    dl[:, 3:] *= 0.1
    dl = dl.to(dev)

    def run():
        optim_step.step_device(params, views, dl)
        torch.cuda.synchronize()
        return params.grads.clone()
    return run


def rows_of(grads):
    """[ROWS_CANCEL, 17] packed-gradient rows (means3D, shs, opacity, scales, rotations, means2D) of seeded Gaussians"""
    n, m = N_CANCEL, (DEG_CANCEL + 1) ** 2
    idx = torch.randperm(n, generator=torch.Generator().manual_seed(13))[:ROWS_CANCEL].sort().values.to(grads.device)
    out, o = [], 0
    for w in (3, 3 * m, 1, 3, 4, 3):
        out.append(grads[o:o + w * n].view(n, w)[idx]); o += w * n
    return torch.cat(out, dim=1).cpu()


def _within_one_ulp(a, b):
    """bit-identical, or one fp32 ulp apart at the larger magnitude (an fp64 sum that landed on a rounding boundary)"""
    m = torch.maximum(a.abs(), b.abs())
    ulp = torch.nextafter(m, torch.full_like(m, float("inf"))) - m
    return (a == b) | ((a - b).abs() <= ulp)


def test_cancelling_gradients_repeat_and_equal_the_per_quadrant_sums(dev):
    """Two runs of the step on the same inputs give the same packed gradients, element by element, up to one fp32 ulp;
    and the rows of 4096 seeded Gaussians equal, to the same bar, the fixture written by the build that issued one set
    of fp64 reds per (quadrant, splat) (scripts/dev/make_combine_golden.py).  The rotation gradients are pure
    cancellation, so one extra fp32 rounding of a partial moves them by many ulps of their own size.  Checked once by
    hand on an H100: a build that adds the quadrant partials in fp32 instead of fp64 fails the fixture comparison
    (13,048 of 69,632 elements beyond one ulp)."""
    run = cancelling_case(dev)
    g1, g2 = run(), run()
    same = _within_one_ulp(g1, g2)
    assert bool(same.all()), f"{int((~same).sum())} of {same.numel()} gradient elements differ between two runs"
    ref = torch.from_numpy(np.load(CANCEL_GOLDEN)["rows"])
    got = rows_of(g1)
    assert bool(got[:, 10:14].abs().max() > 0), "rotation gradients are all zero: the case lost its cancelling sums"
    ok = _within_one_ulp(got, ref)
    assert bool(ok.all()), f"{int((~ok).sum())} of {ok.numel()} fixture elements differ by more than one ulp"


# ---------------- tile-heavy case against the per-pixel oracle ---------------------------------------------
def _tile_heavy_cloud(seed=21):
    """A few hundred large anisotropic splats (each covers all four quadrants of many tiles) plus small ones whose
    footprints straddle tile and quadrant edges."""
    g = torch.Generator().manual_seed(seed)
    nl, ns, deg = 300, 200, 1
    n = nl + ns
    means = (torch.rand(n, 3, generator=g) - 0.5) * 0.7
    log_s = torch.empty(n, 3)
    log_s[:nl] = torch.empty(nl, 3).uniform_(np.log(0.03), np.log(0.12), generator=g)
    log_s[nl:] = torch.empty(ns, 3).uniform_(np.log(0.004), np.log(0.012), generator=g)
    rots = torch.nn.functional.normalize(torch.randn(n, 4, generator=g), dim=1)
    opac = torch.empty(n, 1).uniform_(0.05, 0.6, generator=g)
    shs = (torch.rand(n, (deg + 1) ** 2, 3, generator=g) - 0.5)
    return {"means3D": means.contiguous(), "shs": shs.contiguous(), "opacities": opac, "scales": torch.exp(log_s),
            "rotations": rots.contiguous()}, deg


def _grad_close(a, b, what):
    a, b = a.detach().cpu().double(), b.double()
    scale = float(b.abs().max())
    assert scale > 0.0, what
    rel = float((a - b).norm() / b.norm())
    assert rel < GRAD_RTOL, f"{what}: relative error {rel}"
    assert bool(((a - b).abs() <= GRAD_RTOL * b.abs() + 1e-2 * GRAD_RTOL * scale + 1e-6).all()), what


def test_tile_heavy_case_matches_the_oracle(dev):
    from gs_b200 import rasterizer as R
    cl, deg = _tile_heavy_cloud()
    W, H = 256, 192
    st = O.minicam_settings(O.orbit_camera(10, 30, 1.75), W, H, 49.1, bg=(0.1, 0.2, 0.3), sh_degree=deg)
    g = torch.Generator().manual_seed(22)
    dc = torch.rand(3, H, W, generator=g) * 2 - 1
    dd = (torch.rand(1, H, W, generator=g) * 2 - 1) * 0.1
    da = (torch.rand(1, H, W, generator=g) * 2 - 1) * 0.1
    out, grads = O.rasterize_with_grads({k: cl[k] for k in NAMES}, st, dc, dd, da)
    radii = out["radii"]
    assert int(out["aux"]["keys"].size) >= 10 * int((radii > 0).sum()), "not tile-heavy: too few tiles per splat"
    rs = R.GaussianRasterizationSettings(H, W, st.tanfovx, st.tanfovy, st.bg.to(dev), st.scale_modifier,
                                         st.viewmatrix.to(dev), st.projmatrix.to(dev), deg, st.campos.to(dev), False, False)
    inp = {k: cl[k].to(dev).requires_grad_(True) for k in NAMES}
    m2 = torch.zeros(cl["means3D"].shape[0], 3, device=dev, requires_grad=True)
    color, r, depth, alpha = R.GaussianRasterizer(rs)(
        means3D=inp["means3D"], means2D=m2, shs=inp["shs"], colors_precomp=None, opacities=inp["opacities"],
        scales=inp["scales"], rotations=inp["rotations"], cov3D_precomp=None)
    ((color * dc.to(dev)).sum() + (depth * dd.to(dev)).sum() + (alpha * da.to(dev)).sum()).backward()
    assert torch.equal(r.cpu(), radii)
    assert float((color.detach().cpu() - out["color"]).abs().max()) < 1e-4
    for k in NAMES:
        _grad_close(inp[k].grad, grads[k], f"tile-heavy grad {k}")
    _grad_close(m2.grad, grads["means2D"], "tile-heavy grad means2D")
