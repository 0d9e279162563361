"""CPU tests of the mesh-path oracle (oracle/dr_oracle.py): hand-computable cases, watertightness, texture values,
antialias blend weights, autograd vs fp64 central differences."""
import numpy as np
import pytest
import torch

from conftest import ROOT  # noqa: F401
from oracle import dr_oracle as D
from oracle import gs_oracle as O


def _ndc_tri(pts, z=0.0, w=1.0):
    return torch.tensor([[[x * w, y * w, z * w, w] for x, y in pts]], dtype=torch.float32)


def test_single_triangle_coverage_and_barycentrics():
    # right triangle covering the lower-left half of an 8x8 image (y up: row 0 is the bottom row)
    pos = _ndc_tri([(-1, -1), (1, -1), (-1, 1)], z=0.25)
    tri = torch.tensor([[0, 1, 2]], dtype=torch.int32)
    rast, db = D.rasterize(pos, tri, (8, 8))
    ids = rast[0, ..., 3]
    for y in range(8):
        for x in range(8):
            inside = (x + 0.5) + (y + 0.5) < 8          # pixel centre strictly below the hypotenuse
            assert (ids[y, x] == 1) == inside, (x, y)
    u, v = rast[0, ..., 0], rast[0, ..., 1]
    y, x = 2, 3                                          # centre (3.5,2.5)/8 -> weights of v1 (x) and v2 (y)
    assert abs(float(v[y, x]) - 3.5 / 8) < 1e-6           # v = weight of vertex 1
    assert abs(float(1 - u[y, x] - v[y, x]) - 2.5 / 8) < 1e-6
    assert abs(float(rast[0, y, x, 2]) - 0.25) < 1e-6     # z/w
    assert abs(float(db[0, y, x, 2]) - 1 / 8) < 1e-6      # dv/dX = 1/8 per pixel
    assert abs(float(db[0, y, x, 0]) + 1 / 8) < 1e-6      # du/dX = -1/8


def test_shared_edge_is_watertight_and_exclusive():
    # two triangles forming the full-screen quad, diagonal through pixel centres
    pos = _ndc_tri([(-1, -1), (1, -1), (1, 1), (-1, 1)])
    tri = torch.tensor([[0, 1, 2], [0, 2, 3]], dtype=torch.int32)
    ids = D.rasterize_ids(pos, tri, (8, 8))[0]
    assert bool((ids > 0).all())                          # no holes, also on the diagonal (centres exactly on the edge)
    # same result with the second triangle wound the other way (orientation independent coverage)
    tri2 = torch.tensor([[0, 1, 2], [0, 3, 2]], dtype=torch.int32)
    assert bool((D.rasterize_ids(pos, tri2, (8, 8))[0] > 0).all())


def test_depth_test_and_clip_range():
    near = _ndc_tri([(-1, -1), (1, -1), (-1, 1)], z=-0.5)[0]
    far = _ndc_tri([(-1, -1), (1, -1), (-1, 1)], z=0.5)[0]
    out = _ndc_tri([(-1, -1), (1, -1), (-1, 1)], z=1.5)[0]
    pos = torch.cat([far, near, out])[None]
    tri = torch.tensor([[0, 1, 2], [3, 4, 5], [6, 7, 8]], dtype=torch.int32)
    ids = D.rasterize_ids(pos, tri, (8, 8))[0]
    assert set(ids.unique().tolist()) == {0, 2}           # nearer (z/w=-0.5) wins; z/w=1.5 is clipped
    # ties -> lowest triangle index
    pos2 = torch.cat([far, far])[None]
    ids2 = D.rasterize_ids(pos2, torch.tensor([[3, 4, 5], [0, 1, 2]], dtype=torch.int32), (8, 8))[0]
    assert set(ids2.unique().tolist()) == {0, 1}


def test_vertex_behind_eye_needs_no_clipping():
    # one vertex with w < 0: homogeneous edge functions still give the visible part; must not crash or cover everything
    pos = torch.tensor([[[-0.5, -0.5, 0.0, 1.0], [0.5, -0.5, 0.0, 1.0], [0.0, 2.0, 0.0, -0.5]]])
    tri = torch.tensor([[0, 1, 2]], dtype=torch.int32)
    ids = D.rasterize_ids(pos, tri, (16, 16))[0]
    assert 0 < int((ids > 0).sum()) < 256


def test_interpolate_and_pixel_derivatives():
    pos = _ndc_tri([(-1, -1), (1, -1), (-1, 1)])
    tri = torch.tensor([[0, 1, 2]], dtype=torch.int32)
    rast, db = D.rasterize(pos, tri, (8, 8))
    attr = torch.tensor([[[0.0, 10.0], [1.0, 10.0], [0.0, 20.0]]])     # a0 = NDC-ish x ramp, a1 = 10 + 10*y ramp
    out, da = D.interpolate(attr, rast, tri, rast_db=db, diff_attrs="all")
    assert abs(float(out[0, 2, 3, 0]) - 3.5 / 8) < 1e-6
    assert abs(float(out[0, 2, 3, 1]) - (10 + 10 * 2.5 / 8)) < 1e-5
    assert abs(float(da[0, 2, 3, 0]) - 1 / 8) < 1e-6 and abs(float(da[0, 2, 3, 1])) < 1e-6        # d a0 / dX, dY
    assert abs(float(da[0, 2, 3, 3]) - 10 / 8) < 1e-5                                             # d a1 / dY
    assert float(out[0, 7, 7].abs().max()) == 0.0                                                 # background


def test_texture_bilinear_values_wrap_and_clamp():
    tex = torch.arange(16, dtype=torch.float32).reshape(1, 4, 4, 1)
    uv = torch.tensor([[[[0.125, 0.125], [0.25, 0.125], [0.0, 0.125], [0.375, 0.625]]]])      # texel centres at (i+.5)/4
    out = D.texture(tex, uv)
    assert abs(float(out[0, 0, 0, 0]) - 0.0) < 1e-6               # centre of texel (0,0)
    assert abs(float(out[0, 0, 1, 0]) - 0.5) < 1e-6               # halfway between texel 0 and 1 in x
    assert abs(float(out[0, 0, 2, 0]) - 1.5) < 1e-6               # u=0 wraps: half texel 3 (=3) and texel 0 (=0)
    assert abs(float(out[0, 0, 3, 0]) - (2 * 4 + 1)) < 1e-6       # centre of texel x=1, y=2
    outc = D.texture(tex, uv, boundary_mode="clamp")
    assert abs(float(outc[0, 0, 2, 0]) - 0.0) < 1e-6


def test_antialias_blend_weight_on_a_vertical_edge():
    # quad covering x in [-1, x_e] of a 8x4 image; silhouette edge at pixel coordinate 4.25 -> crosses between
    # pixel centres 3.5 and 4.5 at t = 0.75 measured from the covered pixel -> uncovered pixel gets 0.25
    xe = 4.25 / 8 * 2 - 1
    pos = _ndc_tri([(-1, -1), (xe, -1), (xe, 1), (-1, 1)])
    tri = torch.tensor([[0, 1, 2], [0, 2, 3]], dtype=torch.int32)
    rast, _ = D.rasterize(pos, tri, (4, 8))
    alpha = torch.clamp(rast[..., -1:], 0, 1)
    aa = D.antialias(alpha, rast, pos, tri)
    # (top row: the pixel left of the edge belongs to the OTHER triangle of the quad, which does not own the
    #  silhouette edge -> not antialiased; only the edges of the pixel's own triangle are considered, as in the package)
    assert torch.allclose(aa[0, :, 3, 0], torch.ones(4)) and torch.allclose(aa[0, :3, 4, 0], torch.full((3,), 0.25), atol=1e-6)
    # edge at 3.75: t = 0.25 -> the covered pixel loses 0.25
    xe = 3.75 / 8 * 2 - 1
    pos = _ndc_tri([(-1, -1), (xe, -1), (xe, 1), (-1, 1)])
    rast, _ = D.rasterize(pos, tri, (4, 8))
    aa = D.antialias(torch.clamp(rast[..., -1:], 0, 1), rast, pos, tri)
    assert torch.allclose(aa[0, :3, 3, 0], torch.full((3,), 0.75), atol=1e-6) and float(aa[0, :, 4, 0].abs().max()) == 0
    # the interior diagonal (shared edge) must not be antialiased
    assert torch.allclose(aa[0, :, :3, 0], torch.ones(4, 3))


def test_edge_opposites_closed_mesh_has_no_boundary():
    v, f, _ = D.icosphere(1)
    opp = D.edge_opposites(f)
    assert int((opp < 0).sum()) == 0
    # the partner's opposite vertex is not one of the triangle's own vertices
    assert bool((opp != f.to(torch.int64)).all())


def test_gradients_match_finite_differences_fp64():
    torch.manual_seed(0)
    v, f, uv = D.icosphere(1)
    v = (v.double() * 1.3).contiguous()
    pose = O.orbit_camera(15, 35, 1.75)
    H = W = 24
    proj = D.gl_perspective(49.1, 1.0)
    tex0 = torch.rand(1, 8, 8, 3, dtype=torch.float64)
    gimg = torch.rand(1, H, W, 3, dtype=torch.float64); ga = torch.rand(1, H, W, 1, dtype=torch.float64)

    def render(vv, tex):
        pos = torch.cat([vv, torch.ones_like(vv[:, :1])], dim=1) @ torch.inverse(torch.from_numpy(pose).double()).T
        pos = (pos @ torch.from_numpy(proj).double().T)[None]
        rast, db = D.rasterize(pos, f, (H, W))
        alpha = D.antialias(torch.clamp(rast[..., -1:], 0, 1), rast, pos, f)
        texc, _ = D.interpolate(uv.double()[None], rast, f, rast_db=db, diff_attrs="all")
        col = D.antialias(torch.sigmoid(D.texture(tex, texc)), rast, pos, f)
        return (col * gimg).sum() + (alpha * ga).sum()

    vv = v.clone().requires_grad_(True); tt = tex0.clone().requires_grad_(True)
    loss = render(vv, tt)
    gv, gt = torch.autograd.grad(loss, [vv, tt])
    rng = np.random.RandomState(0)
    checked = 0
    for j in rng.choice(v.numel(), size=10, replace=False):
        eps = 1e-7
        p = v.clone(); m = v.clone(); p.view(-1)[j] += eps; m.view(-1)[j] -= eps
        lp, lm = float(render(p, tex0)), float(render(m, tex0))
        fd = (lp - lm) / (2 * eps)
        an = float(gv.reshape(-1)[j])
        if abs(fd - an) > 1e-3 * max(1.0, abs(fd)):        # a coverage flip inside +-eps makes FD meaningless: re-test smaller
            continue
        checked += 1
    assert checked >= 8
    for j in rng.choice(tex0.numel(), size=6, replace=False):
        eps = 1e-6
        p = tex0.clone(); m = tex0.clone(); p.view(-1)[j] += eps; m.view(-1)[j] -= eps
        fd = (float(render(v, p)) - float(render(v, m))) / (2 * eps)
        assert abs(fd - float(gt.reshape(-1)[j])) <= 1e-5 * max(1.0, abs(fd))


def test_mipmapped_texture_levels_and_limits():
    """'linear-mipmap-linear': zero derivatives -> level 0 = plain bilinear; a footprint of exactly 2^k texels -> level k
    of the box-filtered pyramid; an anisotropic footprint uses its MAJOR axis; the last level of a power-of-two texture is
    the mean texel."""
    g = torch.Generator().manual_seed(0)
    tex = torch.rand(1, 16, 32, 3, generator=g)
    uv = torch.rand(1, 5, 7, 2, generator=g)
    z = torch.zeros(1, 5, 7, 4)
    assert torch.allclose(D.texture(tex, uv, "linear-mipmap-linear", uv_da=z), D.texture(tex, uv, "linear"))
    pyr = D.mip_pyramid(tex)
    assert [tuple(t.shape[1:3]) for t in pyr] == [(16, 32), (8, 16), (4, 8), (2, 4), (1, 2)]
    assert torch.allclose(pyr[-1].mean(dim=(1, 2)), tex.mean(dim=(1, 2)), atol=1e-6)
    for k in (1, 2, 3):
        da = torch.zeros(1, 5, 7, 4)
        da[..., 0] = (2.0 ** k) / 32          # du/dX = 2^k texels of the 32-wide side, nothing along Y
        da[..., 3] = 1.0 / 16                 # dv/dY = 1 texel: the major axis decides
        got = D.texture(tex, uv, "linear-mipmap-linear", uv_da=da)
        assert torch.allclose(got, D.texture(pyr[k], uv, "linear"), atol=1e-6), k
    assert float(D.mip_level(torch.full((1, 1, 1, 4), 100.0), 16, 32, len(pyr)).max()) == len(pyr) - 1      # clamped


# ---------------- scenes with vertices and edges exactly on pixel centres; the windowed evaluation ----------------------
def test_fan_premise_centre_vertex_is_on_the_fp32_pixel_centre():
    from fractions import Fraction
    rng = np.random.default_rng(1)
    for persp in (False, True):
        pos, tri, (px, py) = D.pixel_centre_fan(rng, 64, 64, persp)
        x, y, _, w = pos[0, 0].tolist()
        assert Fraction(x) / Fraction(w) == Fraction(D.pixel_centre(px, 64))
        assert Fraction(y) / Fraction(w) == Fraction(D.pixel_centre(py, 64))
        assert len({tuple(sorted(t)) for t in tri.tolist()}) == tri.shape[0]


@pytest.mark.parametrize("persp", [False, True])
def test_closed_fans_around_pixel_centre_vertices_cover_every_pixel_once(persp):
    """At a vertex exactly on a pixel centre each spoke's fp32 edge value is rounding noise of either sign; with the
    fp32 signs alone 8 of 253 random fans left the centre pixel uncovered (a hole in a closed surface) and 134 covered
    it twice.  Exact signs with the symbolic tie rule cover every pixel of every fan exactly once."""
    rng = np.random.default_rng(123 + persp)
    for _ in range(75):
        pos, tri, (px, py) = D.pixel_centre_fan(rng, 64, 64, persp)
        cnt = D.coverage_count(pos, tri, (64, 64))[0]
        assert int(cnt.max()) == 1, (px, py)
        assert bool((cnt[py - 1:py + 2, px - 1:px + 2] == 1).all()), (px, py)      # inside the ring (inradius > 2 px)


def test_pixel_centre_grid_is_watertight():
    """A grid whose vertices all lie on pixel centres (a UV-space bake): every pixel strictly inside it, vertex pixels
    included, is covered exactly once."""
    H = W = 64
    pos, tri = D.pixel_centre_grid(H, W, 3, 5, 4, 17, 18)
    cnt = D.coverage_count(pos, tri, (H, W))[0]
    assert int(cnt.max()) == 1
    assert bool((cnt[5:58, 6:56] == 1).all())
    ids = D.rasterize_ids(pos, tri, (H, W))[0]
    assert bool(((ids > 0) == (cnt > 0)).all())


def test_exact_sign_helpers():
    c = D.pixel_centre(20, 64)
    assert D.det3_sign_exact((0.0, 0.0, 1.0), (1.0, 0.0, 1.0), (0.0, 1.0, 1.0)) == 1
    assert D.det3_sign_exact((0.0, 1.0, 1.0), (1.0, 0.0, 1.0), (0.0, 0.0, 1.0)) == -1
    assert D.det3_sign_exact((c, c, 1.0), (2 * c, 2 * c, 2.0), (0.3, 0.1, 1.0)) == 0       # same point projectively
    # an edge through the point: exact zero, decided by (a, b): exactly one of the two orientations covers it
    pj, pk = [c, -0.5, 0.0, 1.0], [c, 0.5, 0.0, 1.0]
    assert D.edge_inside_exact(pj, pk, c, 0.0, 1.0) != D.edge_inside_exact(pk, pj, c, 0.0, 1.0)


def test_window_mode_matches_the_full_frame():
    v, f, _ = D.icosphere(2)
    pos = D.clip_positions(v, O.orbit_camera(20, 30, 1.75), D.gl_perspective(49.1, 1.0))
    full = D.rasterize_ids(pos, f, (48, 48))
    assert torch.equal(D.rasterize_ids(pos, f, (48, 48), window=(10, 30, 5, 41)), full[:, 10:30, 5:41])


# ---------------- mip level: finite gradient at isotropic and zero footprints ---------------------------------------
@pytest.mark.parametrize("da", [(0.01, 0.0, 0.0, 0.01), (0.0, 0.0, 0.0, 0.0), (0.01, 0.002, 0.0, 0.01), (0.004, 0.0, 0.0, 0.0)])
def test_mip_level_gradient_is_finite(da):
    x = torch.tensor(da, dtype=torch.float64).reshape(1, 1, 1, 4).requires_grad_(True)
    D.mip_level(x, 64, 64, 7).sum().backward()
    assert bool(torch.isfinite(x.grad).all())


def test_mip_level_subgradient_at_the_isotropic_point():
    """At an isotropic footprint (A = B, C = 0) the root term sqrt(0.25 (A-B)^2 + C^2) is a cone point; its gradient is
    taken as 0 there, so the level's gradient is the mean of the two one-sided derivatives along every direction, and
    the derivative itself along directions that keep the footprint isotropic (scaling and rotating uv_da)."""
    x0 = torch.tensor([0.05, 0.0, 0.0, 0.05], dtype=torch.float64)
    f = lambda x: float(D.mip_level(x.reshape(1, 1, 1, 4), 64, 64, 7).sum())
    x = x0.clone().reshape(1, 1, 1, 4).requires_grad_(True)
    D.mip_level(x, 64, 64, 7).sum().backward()
    g = x.grad.reshape(4)
    assert bool(torch.isfinite(g).all()) and float(g.abs().max()) > 0
    h = 1e-7
    for d in (x0, torch.tensor([0.0, 0.05, -0.05, 0.0], dtype=torch.float64)):            # scale; rotate
        right = (f(x0 + h * d) - f(x0)) / h
        assert abs(right - float(g @ d)) <= 1e-6 * max(1.0, abs(right))
    rng = np.random.default_rng(0)
    for _ in range(5):
        d = torch.from_numpy(rng.standard_normal(4))
        right = (f(x0 + h * d) - f(x0)) / h; left = (f(x0) - f(x0 - h * d)) / h
        assert left - 1e-6 <= float(g @ d) <= right + 1e-6
        assert abs(0.5 * (left + right) - float(g @ d)) <= 1e-5 * max(1.0, abs(right))
