"""CPU tests of the point rasterizer's oracle (oracle/points_oracle.py) on hand-worked cases, of its camera convention
against an independent float64 pinhole projection, and of gs_b200.points' host-side validation and C ABI.

Most cases use the camera R = I, T = 0, fx = fy = s, (cx, cy) = the image centre, under which a world point
(-a z, -b z, z) lands at NDC (a, b); on a 4 x 4 image the pixel centres sit at +-0.25 and +-0.75, all exact in fp32."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import points_oracle as O

f32 = np.float32


def _cam(H, W, n=1):
    s = min(H, W) / 2
    Km = np.array([[s, 0, W / 2], [0, s, H / 2], [0, 0, 1]], f32)
    return np.repeat(np.eye(3, dtype=f32)[None], n, 0), np.zeros((n, 3), f32), np.repeat(Km[None], n, 0)


def _at(a, b, z=1.0):
    """the world point that the simple camera sends to NDC (a, b) at depth z"""
    return [-a * z, -b * z, z]


def _rast(clouds, H=4, W=4, radius=0.1, K=1):
    R, T, Km = _cam(H, W, len(clouds))
    return O.rasterize([np.array(c, f32).reshape(-1, 3) for c in clouds], R, T, Km, None, H, W, radius, K)


def test_pixel_centres_and_one_point_at_a_centre():
    xc, yc = O.centres(4, 4)
    np.testing.assert_array_equal(xc, f32([0.75, 0.25, -0.25, -0.75]))      # column 0 is the +X (left) end
    np.testing.assert_array_equal(yc, f32([0.75, 0.25, -0.25, -0.75]))      # row 0 is the +Y (top) end
    idx, zbuf, dists = _rast([[_at(0.25, -0.25, 2.0)]])
    want = np.full((1, 4, 4, 1), -1, np.int32)
    want[0, 2, 1, 0] = 0
    np.testing.assert_array_equal(idx, want)
    assert zbuf[0, 2, 1, 0] == 2.0 and dists[0, 2, 1, 0] == 0.0
    assert (zbuf[idx < 0] == -1).all() and (dists[idx < 0] == -1).all()


def test_coverage_is_strict_at_exactly_the_radius():
    p = [_at(0.375, -0.25)]                     # 0.125 from the centre (0.25, -0.25), 0.375 from (0.75, -0.25)
    idx, _, _ = _rast([p], radius=0.125)        # dx*dx = 0.015625 = radius^2 exactly: not covered
    assert (idx == -1).all()
    r = float(np.nextafter(f32(0.125), f32(1)))
    idx, _, dists = _rast([p], radius=r)
    assert np.argwhere(idx >= 0).tolist() == [[0, 2, 1, 0]] and dists[0, 2, 1, 0] == f32(0.015625)


def test_z_ties_go_to_the_smaller_packed_index():
    same = [_at(0.25, 0.25, 3.0)] * 3
    idx, zbuf, _ = _rast([same], K=1)
    assert idx[0, 1, 1, 0] == 0
    idx, zbuf, _ = _rast([same], K=2)
    assert idx[0, 1, 1].tolist() == [0, 1] and zbuf[0, 1, 1].tolist() == [3.0, 3.0]
    nearer_later = [_at(0.25, 0.25, 3.0), _at(0.25, 0.25, 2.0)]
    idx, _, _ = _rast([nearer_later], K=1)
    assert idx[0, 1, 1, 0] == 1


def test_k2_keeps_the_two_nearest_in_z_order():
    pts = [_at(0.25, 0.25, 3.0), _at(0.26, 0.25, 1.0), _at(0.24, 0.24, 2.0)]
    idx, zbuf, dists = _rast([pts], radius=0.05, K=2)
    assert idx[0, 1, 1].tolist() == [1, 2] and zbuf[0, 1, 1].tolist() == [1.0, 2.0]
    assert dists[0, 1, 1, 0] > 0 and dists[0, 1, 1, 1] > 0
    idx3, zbuf3, _ = _rast([pts], radius=0.05, K=3)
    assert idx3[0, 1, 1].tolist() == [1, 2, 0] and zbuf3[0, 1, 1].tolist() == [1.0, 2.0, 3.0]
    one, _, _ = _rast([pts[:1]], radius=0.05, K=2)
    assert one[0, 1, 1].tolist() == [0, -1]


def test_behind_and_on_the_camera_plane_are_never_drawn():
    idx, _, _ = _rast([[[0.25, 0.25, -1.0]]], radius=10.0)        # z < 0
    assert (idx == -1).all()
    idx, _, _ = _rast([[[0.0, 0.0, 0.0], [-0.25, 0.25, 0.0]]], radius=10.0)    # z = 0: 0/0 and x/0
    assert (idx == -1).all()
    idx, _, _ = _rast([[[0.0, 0.0, 0.0], _at(0.25, 0.25, 1e-30)]], radius=10.0)
    assert (idx[..., 0] == 1).all()                               # the smallest positive z still draws


def test_clouds_and_packed_indices():
    idx, _, _ = _rast([[_at(0.25, 0.25)], [], [_at(-0.75, -0.75), _at(0.75, 0.75)]])
    assert np.argwhere(idx[0] >= 0).tolist() == [[1, 1, 0]] and idx[0, 1, 1, 0] == 0
    assert (idx[1] == -1).all()
    assert idx[2, 3, 3, 0] == 1 and idx[2, 0, 0, 0] == 2


def test_non_square_ndc_extents_252x180():
    H, W = 180, 252
    xc, yc = O.centres(H, W)
    assert np.isclose(xc[0], 1.4 - 1.4 / W) and np.isclose(xc[-1], -1.4 + 1.4 / W)     # longer side: [-1.4, 1.4]
    assert np.isclose(yc[0], 1 - 1 / H) and np.isclose(yc[-1], -1 + 1 / H)             # shorter side: [-1, 1]
    assert np.allclose(np.diff(xc), -2 / H, atol=1e-6) and np.allclose(np.diff(yc), -2 / H, atol=1e-6)  # square pixels
    # a point at the pixel-space centre of pixel (row 7, column 200) lands on that pixel only
    R, T, Km = _cam(H, W)
    u, v = 200.5, 7.5
    s = H / 2
    p = np.array([[(u - W / 2) / s, (v - H / 2) / s, 1.0]], f32)
    idx, _, dists = O.rasterize([p], R, T, Km, None, H, W, 0.5 / s, 1)
    assert np.argwhere(idx >= 0).tolist() == [[0, 7, 200, 0]] and dists[0, 7, 200, 0] < 1e-10


def _rotation(rng):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


@pytest.mark.parametrize("hw", [(252, 252), (180, 252), (252, 180)])
def test_camera_against_an_independent_pinhole(hw):
    """cameras_from_opencv_projection's NDC at the principal point and the four image corners: (w/2 - u) / s and
    (h/2 - v) / s with s = min(h, w) / 2, so +X is left, +Y up and the shorter side spans [-1, 1]."""
    rng = np.random.default_rng(1)
    H, W = hw
    R, T = _rotation(rng), rng.normal(size=3)
    fx, fy, cx, cy = 300.0, 280.0, W / 2 + 3.5, H / 2 - 2.25
    Km = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]])
    s = min(H, W) / 2
    uv = [(cx, cy), (0, 0), (W, 0), (0, H), (W, H)]
    z = rng.uniform(1, 4, len(uv))
    cam = np.array([[(u - cx) / fx * d, (v - cy) / fy * d, d] for (u, v), d in zip(uv, z)])
    world = (cam - T) @ R                                          # R^T (c - T)
    want = np.array([[(W / 2 - u) / s, (H / 2 - v) / s] for u, v in uv])
    x, y, zz = O.project(world.astype(f32), R, T, Km, (H, W))
    np.testing.assert_allclose(np.stack([x, y], 1), want, atol=2e-5)
    np.testing.assert_allclose(zz, z, rtol=1e-5)
    x64, y64, _ = O.project64(world, R, T, Km, (H, W))
    np.testing.assert_allclose(np.stack([x64, y64], 1), want, atol=1e-9)
    assert np.isclose(want[1, 0], W / 2 / s) and np.isclose(want[1, 1], H / 2 / s)       # top-left: +X, +Y


def test_lift_takes_the_largest_pixel_index_and_backward_is_its_adjoint():
    idx = np.full((2, 2, 3, 2), -1, np.int32)
    idx[0, 0, 0, 0] = 4
    idx[0, 1, 2, 1] = 4            # larger linear index: wins for point 4
    idx[1, 0, 1, 0] = 1
    idx[1, 0, 1, 1] = 2            # same pixel, both won
    rng = np.random.default_rng(0)
    feat = rng.normal(size=(2, 3, 2, 3)).astype(f32)
    out = O.lift(idx, feat, 6)
    np.testing.assert_array_equal(out[4], feat[0, :, 1, 2])
    np.testing.assert_array_equal(out[1], feat[1, :, 0, 1])
    np.testing.assert_array_equal(out[2], feat[1, :, 0, 1])
    assert (out[[0, 3, 5]] == 0).all()
    g = rng.normal(size=(6, 3))
    grad = O.lift_backward(idx, g, 3, 6)
    want = np.zeros_like(grad)
    want[0, :, 1, 2] = g[4]
    want[1, :, 0, 1] = g[1] + g[2]
    np.testing.assert_array_equal(grad, want)
    # adjoint: <lift(f), g> = <f, lift_backward(g)>
    assert np.isclose((O.lift(idx, feat, 6) * g).sum(), (feat * grad).sum())


def test_settings_and_argument_errors_before_any_gpu_work():
    from gs_b200 import points as P
    cpu = torch.zeros(1, 4, 3)
    with pytest.raises(RuntimeError, match="CPU"):
        P.Pointclouds(cpu)
    with pytest.raises(TypeError, match="float32"):
        P.Pointclouds(cpu.double())
    with pytest.raises(TypeError):
        P.Pointclouds("points")
    with pytest.raises(RuntimeError, match="CPU"):
        P.points_projection(cpu, torch.eye(4)[None], torch.eye(3)[None], torch.zeros(1, 2, 4, 4))
    with pytest.raises(TypeError, match="float32"):
        P.points_projection(cpu.half(), torch.eye(4)[None], torch.eye(3)[None], torch.zeros(1, 2, 4, 4))
    with pytest.raises(RuntimeError, match="CPU"):
        P.cameras_from_opencv_projection(torch.eye(3)[None], torch.zeros(1, 3), torch.eye(3)[None], torch.ones(1, 2))
    with pytest.raises(TypeError, match="floating"):
        P.cameras_from_opencv_projection(torch.eye(3, dtype=torch.int64)[None], torch.zeros(1, 3), torch.eye(3)[None],
                                         torch.ones(1, 2))
    for K in (0, 9):
        with pytest.raises(NotImplementedError, match="points_per_pixel"):
            P.PointsRasterizer(raster_settings=P.PointsRasterizationSettings(8, 0.1, K))(None)
    for size in (0, (4,), (4, -1), 4.0):
        with pytest.raises(ValueError, match="image_size"):
            P.PointsRasterizer(raster_settings=P.PointsRasterizationSettings(size, 0.1, 1))(None)
    with pytest.raises(ValueError, match="radius"):
        P.PointsRasterizer(raster_settings=P.PointsRasterizationSettings(8, -0.1, 1))(None)
    with pytest.raises(NotImplementedError, match="radius"):
        P.PointsRasterizer(raster_settings=P.PointsRasterizationSettings(8, torch.ones(3), 1))(None)
    with pytest.raises(TypeError, match="Pointclouds"):
        P.PointsRasterizer(raster_settings=P.PointsRasterizationSettings(8, 0.1, 1))(cpu)
    for cls in (P.CamerasBase, P.AlphaCompositor, P.NormWeightedCompositor, P.PointsRenderer):
        with pytest.raises(NotImplementedError):
            cls()
    s = P.PointsRasterizationSettings(image_size=(252, 180), radius=0.0075, points_per_pixel=1, bin_size=0)
    assert (s.image_size, s.radius, s.points_per_pixel, s.bin_size, s.max_points_per_bin) == ((252, 180), 0.0075, 1, 0, None)


def test_c_abi_is_bound_from_include():
    """gs_b200_pts_* are bound from include/gs_b200_pts.h: every declared function resolves with one argtype per
    parameter."""
    from gs_b200 import _lib
    from gs_b200 import points as P
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "gs_b200_pts.h")).read(), flags=re.S)
    declared = dict(re.findall(r"\b(gs_b200_pts_\w+)\s*\(([^()]*)\)\s*;", src))
    assert set(declared) == {"gs_b200_pts_scratch_bytes", "gs_b200_pts_rasterize", "gs_b200_pts_lift",
                             "gs_b200_pts_lift_backward"}
    for name, params in declared.items():
        assert len(getattr(_lib.lib, name).argtypes) == params.count(",") + 1, name
    I, L, F, V = ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p
    assert (_lib.lib.gs_b200_pts_rasterize.restype, tuple(_lib.lib.gs_b200_pts_rasterize.argtypes)) == \
        (I, (I, L, I, I, I, F, I) + (V,) * 11)
    assert _lib.lib.gs_b200_pts_scratch_bytes.restype == ctypes.c_size_t and P.MAX_K == 8
    # argument errors come back through gs_b200_last_error, with no GPU work
    assert _lib.lib.gs_b200_pts_scratch_bytes(1, 10, 4, 4, 9) == 0 and "K 9" in _lib.last_error()
    assert _lib.lib.gs_b200_pts_scratch_bytes(0, 10, 4, 4, 1) == 0
    assert _lib.lib.gs_b200_pts_scratch_bytes(2, 10, 4, 4, 3) >= 2 * 16 * 3 * 8 + 10 * 16
    assert _lib.lib.gs_b200_pts_rasterize(1, 4, 4, 4, 1, -1.0, 1, *([None] * 11)) == 1 and "radius" in _lib.last_error()
