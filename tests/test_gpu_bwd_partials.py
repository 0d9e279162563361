"""The composite backward keeps ONE block of per-quadrant fp32 partials in shared memory for both ring stages.  A warp
stores the partials of stage `it` only after the combine of stage it - 1 has read the block, so a warp that runs ahead
of the others waits there.  These tests build a tile whose four quadrants do very different amounts of work, so that the
wait happens, and pin the gradients bit for bit to the fixture written by the build that kept one partial block per
ring stage (scripts/dev/make_bwd_partials_golden.py)."""
import math
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import gs_oracle as O

NAMES = ("means3D", "shs", "opacities", "scales", "rotations")
GOLDEN_FILE = os.path.join(GOLDEN, "bwd_partials_grads.npz")
W = H = 16                 # one 16x16 tile: one CTA, so every SplatGrad sum gets one fp64 red per value, in a fixed order
FOVY, RADIUS, DEG = 49.1, 1.75, 1
BATCH = 128                # records per ring stage of the composite kernels


def unequal_quadrant_cloud(seed=31):
    """Splats placed in pixel units in front of a camera on the +z axis looking at the origin:
    - 4 layers of a 4x4 grid of opaque splats over quadrant (0, 0), in front: its pixels terminate within the first
      stage of the list, so its warp skips every other stage and has its first partials to store in the last one;
    - 150 large faint splats over the whole tile, at depths behind: quadrants (1, 0) and (0, 1) hit few records per stage;
    - 500 small faint splats in quadrant (1, 1), at the same depths: its warp hits almost every record of every stage."""
    g = torch.Generator().manual_seed(seed)
    px, py, dep, sig, op = [], [], [], [], []
    for layer in range(4):
        for gy in range(4):
            for gx in range(4):
                px.append(0.5 + 2 * gx); py.append(0.5 + 2 * gy)
                dep.append(1.0 + 0.01 * layer + 0.001 * (4 * gy + gx)); sig.append(1.5); op.append(0.99)
    for n, lo, span, s_lo, s_hi, o_hi in ((150, -0.5, 16.0, 3.0, 5.0, 0.05), (500, 10.0, 5.0, 0.7, 1.2, 0.06)):
        px += (torch.rand(n, generator=g) * span + lo).tolist()
        py += (torch.rand(n, generator=g) * span + lo).tolist()
        dep += torch.empty(n).uniform_(1.5, 2.0, generator=g).tolist()
        sig += torch.empty(n).uniform_(s_lo, s_hi, generator=g).tolist()
        op += torch.empty(n).uniform_(0.02, o_hi, generator=g).tolist()
    px, py, dep, sig = (torch.tensor(v, dtype=torch.float32) for v in (px, py, dep, sig))
    k = math.tan(math.radians(FOVY) / 2) * dep / (W / 2)          # world units per pixel at each splat's depth
    n = px.numel()
    rots = torch.zeros(n, 4)
    rots[:, 0] = 1.0
    return {"means3D": torch.stack([(px - 7.5) * k, -(py - 7.5) * k, RADIUS - dep], 1).contiguous(),
            "shs": (torch.rand(n, (DEG + 1) ** 2, 3, generator=g) - 0.5).contiguous(),
            "opacities": torch.tensor(op)[:, None].contiguous(), "scales": (sig * k)[:, None].repeat(1, 3).contiguous(),
            "rotations": rots}


def settings():
    return O.minicam_settings(O.orbit_camera(0, 0, RADIUS), W, H, FOVY, bg=(0.1, 0.2, 0.3), sh_degree=DEG)


def upstream():
    g = torch.Generator().manual_seed(32)
    dc = torch.rand(3, H, W, generator=g) * 2 - 1
    dd = (torch.rand(1, H, W, generator=g) * 2 - 1) * 0.1
    da = (torch.rand(1, H, W, generator=g) * 2 - 1) * 0.1
    return dc, dd, da


def run_case(dev):
    """gradients of the six inputs (NAMES, then means2D) through the device rasterizer, on the CPU"""
    from gs_b200 import rasterizer as R
    cl, st = unequal_quadrant_cloud(), settings()
    dc, dd, da = upstream()
    rs = R.GaussianRasterizationSettings(H, W, st.tanfovx, st.tanfovy, st.bg.to(dev), st.scale_modifier,
                                         st.viewmatrix.to(dev), st.projmatrix.to(dev), DEG, st.campos.to(dev), False, False)
    inp = {k: cl[k].to(dev).requires_grad_(True) for k in NAMES}
    m2 = torch.zeros(cl["means3D"].shape[0], 3, device=dev, requires_grad=True)
    color, _, depth, alpha = R.GaussianRasterizer(rs)(
        means3D=inp["means3D"], means2D=m2, shs=inp["shs"], colors_precomp=None, opacities=inp["opacities"],
        scales=inp["scales"], rotations=inp["rotations"], cov3D_precomp=None)
    ((color * dc.to(dev)).sum() + (depth * dd.to(dev)).sum() + (alpha * da.to(dev)).sum()).backward()
    torch.cuda.synchronize()
    out = {k: inp[k].grad.cpu() for k in NAMES}
    out["means2D"] = m2.grad.cpu()
    return out


def test_unequal_quadrant_case_has_the_intended_shape():
    """(CPU, oracle) the premise of the GPU test: one tile, a list of six stages, quadrant (0, 0) done within the first
    stage, each of the other three quadrants walking the whole list."""
    cl, st = unequal_quadrant_cloud(), settings()
    _, radii, _, _, aux = O.rasterize(cl["means3D"], torch.zeros_like(cl["means3D"]), cl["shs"], None, cl["opacities"],
                                      cl["scales"], cl["rotations"], None, st, return_aux=True)
    assert int((radii > 0).sum()) == radii.numel()
    ranges = aux["ranges"]
    assert ranges.shape[0] == 1
    length = int(ranges[0, 1] - ranges[0, 0])
    assert length == radii.numel() and (length + BATCH - 1) // BATCH == 6
    nc = aux["n_contrib"]
    assert int(nc[:8, :8].max()) <= BATCH, "quadrant (0, 0) must finish within the front stage"
    for y0, x0 in ((0, 8), (8, 0), (8, 8)):
        assert int(nc[y0:y0 + 8, x0:x0 + 8].max()) > 5 * BATCH, "the other quadrants must walk all six stages"


@pytest.mark.gpu
def test_unequal_quadrants_give_the_fixture_gradients_bit_for_bit():
    """Two runs give the same bits, equal to the fixture, and close to the oracle (which guards the fixture itself).
    The splats are isotropic, so the oracle's rotation gradient is zero and that one is held to the fixture only."""
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    dev = torch.device("cuda:0")
    g1, g2 = run_case(dev), run_case(dev)
    ref = np.load(GOLDEN_FILE)
    for k in NAMES + ("means2D",):
        assert torch.equal(g1[k], g2[k]), f"grad {k} differs between two runs"
        want = torch.from_numpy(ref[k])
        diff = int((g1[k] != want).sum())
        assert diff == 0, f"grad {k}: {diff} of {want.numel()} elements differ from the fixture"
    cl, st = unequal_quadrant_cloud(), settings()
    _, grads = O.rasterize_with_grads({k: cl[k] for k in NAMES}, st, *upstream())
    for k in ("means3D", "shs", "opacities", "scales", "means2D"):
        a, b = g1[k].double(), grads[k].detach().double()
        rel = float((a - b).norm() / b.norm())
        assert rel < 1e-3, f"grad {k}: relative error {rel} against the oracle"


@pytest.mark.gpu
def test_backward_occupancy():
    """The composite backward's shared memory fits three CTAs per SM, and on an H100 the occupancy calculator reports
    three CTAs per SM for it."""
    import ctypes as C
    from gs_b200 import _lib
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    ctas, smem = C.c_int32(0), C.c_int32(0)
    _lib.check(_lib.lib.gs_b200_composite_bwd_occupancy(C.byref(ctas), C.byref(smem)))
    assert 3 * (smem.value + 1024) <= 228 * 1024, smem.value
    if "H100" in torch.cuda.get_device_name(0):
        assert ctas.value == 3, f"{ctas.value} CTAs per SM"
    else:
        assert ctas.value >= 1
