"""Mesh-path kernels (dr_raster.cu, dr_ops.cu and the mip-mapped texture in gs_b200/meshops.py) against a float64
evaluation of the same operation, at the edges where they make discrete decisions: vertices and edges on pixel centres,
degenerate and behind-the-eye triangles, the small/queued triangle split, the depth range and depth ties (R1); the
rasterizer's values and position gradient on ordinary and grazing triangles (R2); interpolate's batch, attribute-count
and derivative variants (I); bilinear texture at texel centres and borders, wrap seams, huge uv, clamp borders,
degenerate texture shapes, channel counts and the mip path (T); antialias at silhouette crossings exactly on pixel
centres, image borders, open, non-manifold and behind-the-eye topology (A); and windows of a config-4 frame (C4).
Every scene has a CPU test of its premise.

References.  Triangle ids (and antialias's discrete decisions) are the ones the fp32 contract fixes: ids are compared bit
for bit with `oracle/dr_oracle.py`, and the float64 values are the oracle's operations
run in float64 on those ids, at the fp32 pixel centres.  Gradients are float64 autograd through the same operations.

Bars (derivation), u = 2^-24, gamma_n = n u / (1 - n u); each comparison has a per-element bar K_ELEM (= 2) times an
fp32 error bound, and a fixed norm-relative cap.
- Edge values e_i = (a X + b Y) + c: five roundings deep, E_i = gamma_5 M_i with M_i the sum of |terms|; S = e0 + e1 + e2:
  E_S = sum E_i + gamma_2 sum |e_i|.  u = e0 / S: (E_0 + |u| E_S) / |S| + u |u| (the 1/|S| is the condition factor that
  grows on grazing triangles; an e_i whose fp32 sign contradicts the exact coverage is replaced by 0, an error below
  E_i); z/w = (sum z_i e_i) / det: (sum |z_i| E_i + gamma_3 sum |z_i e_i| + |z/w| E_det) / |det|
  + u |z/w| with E_det = gamma_5 sum |terms|.  rast_db = (a0 S - e0 sa) sx / S^2: first-order propagation of the errors
  of a0 (gamma_2), sa (gamma_4), e0 and S through the quotient, plus gamma_4 of the result.
- Position gradient: each pixel adds e_c br_r, br_r = k (gu (A0r S - e0 SAr) + gv (A1r S - e1 SAr)), k = -1/(S^2 det):
  per term E_c |br| + |e_c| dbr + u |e_c br|, dbr propagating the coefficient, e, S and det errors; the reds into an
  element add gamma_n sum |term| for n terms in any order.
- Interpolate: out = u a0 + v a1 + (1 - u - v) a2 on the kernel's own (u, v): gamma_4 sum |terms| + 2u (1 + |u| + |v|) |a2|
  (1 - u - v cancels near the third vertex's opposite edge); derivatives gamma_3 sum |terms|; attribute gradients
  gamma_(n + 4) sum |terms| over the n pixels that add into them, plus that absolute 2u (1 + |u| + |v|) |g| per term of
  the third vertex.
- Texture: the reference is evaluated at the kernel's fp32 texel coordinate x = fl(fl(uv W) - 1/2), the discrete input
  the contract fixes (as the ids are for the rasterizer): it sets the cell and the fraction, which at |uv| = 1e4 keeps
  a few bits and at 1e7 none.  Every scene checks that float64 lands in the same cell (no exclusions).  Values:
  gamma_7 max |t| (six roundings deep, nonnegative weights summing to 1 up to rounding); uv gradients: gamma_(C + 6) sum_c |g| 2 max |t| W; texel
  gradients: gamma_(n + 3) sum |g|.  The mip path (Python glue over the same kernel) is compared at 64 u absolute for
  values; its gradients (through the pyramid, the level of detail and the tent weights) only at 1e-4 of the largest
  element and 1e-3 norm-relative, the same as `test_gpu_mesh.py`'s bar: no bound is derived for that chain.
- Antialias: the scenes place vertices on a 1/16-pixel grid with w = 1 at power-of-two resolutions, so screen
  positions, crossings fa/fb and the side tests are exact in fp32, and no crossing lands exactly on a pixel centre
  except through an exact fa = 0 or along an axis-parallel edge (checked on the CPU): every decision then matches float64.  t carries the
  rounding of the crossing, a few u times the pixel coordinates (<= W), times the colour difference: 16 u (1 + W)
  (1 + |colour|).  Position gradients: 1e-5 of the largest element, and REL_AA_POS norm-relative.
Apart from the mip-path gradients, the fixed norm-relative caps are ten or more times tighter than `test_gpu_mesh.py`'s
(2e-4 .. 1e-3).  Tests print each
scene's worst error against both bars."""
import math

import numpy as np
import pytest
import torch

from oracle import dr_oracle as D
from oracle import gs_oracle as O

U = 2.0 ** -24
K_ELEM = 2.0
REL_VAL = 1e-6            # rasterize / interpolate / texture values, norm-relative
REL_GRAD = 1e-5           # gradients, norm-relative
REL_AA_POS = 1e-4         # antialias position gradient (a chain of four quotients), norm-relative


def gam(n):
    n = np.asarray(n, dtype=np.float64) if not torch.is_tensor(n) else n.double()
    return n * U / (1 - n * U)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def dr():
    import nvdiffrast.torch as dr
    return dr


def check(name, got, ref, bar, cap, mask=None):
    got = got.detach().cpu().double(); ref = ref.detach().cpu().double()
    bar = torch.as_tensor(bar).double().expand_as(ref)
    if mask is not None:
        got, ref, bar = got[mask], ref[mask], bar[mask]
    err = (got - ref).abs()
    ratio = float((err / (K_ELEM * bar)).max()) if err.numel() else 0.0
    rel = float((got - ref).norm() / ref.norm()) if float(ref.norm()) > 0 else float(err.max() if err.numel() else 0.0)
    print(f"{name}: worst err/bar {ratio:.3g}, norm-rel {rel:.3g} (cap {cap:g})")
    assert ratio <= 1.0, (name, ratio)
    assert rel <= cap, (name, rel)
    return ratio, rel


def _rast(dr, pos, tri, res, dev):
    return dr.rasterize(dr.RasterizeCudaContext(), pos.to(dev), tri.to(dev), res)


def _per_triangle_views(pos, tri):
    """One view per triangle, holding only that triangle's vertices (the rest at (0, 0, 0, 0), which makes every other
    triangle degenerate): counts how many triangles cover each pixel in one rasterize call."""
    F = tri.shape[0]
    keep = torch.zeros(F, pos.shape[1], dtype=torch.bool)
    keep[torch.arange(F)[:, None], tri.long()] = True
    return torch.where(keep[..., None], pos.expand(F, -1, -1), torch.zeros(()))


def _gpu_count(dr, pos, tri, res, dev):
    rast, _ = _rast(dr, _per_triangle_views(pos, tri), tri, res, dev)
    return (rast[..., 3] > 0).sum(0).cpu()


def _ids_equal(dr, pos, tri, res, dev):
    rast, db = _rast(dr, pos, tri, res, dev)
    ref = D.rasterize_ids(pos, tri, res)
    assert torch.equal(rast[..., 3].cpu().long(), ref), int((rast[..., 3].cpu().long() != ref).sum())
    return rast, db, ref


# ============================================ R1: coverage =========================================================
@pytest.mark.gpu
@pytest.mark.parametrize("persp", [False, True])
def test_r1_closed_fans_cover_every_pixel_exactly_once(dr, dev, persp):
    """Closed fans whose centre vertex lies exactly on a pixel centre, where the spokes' fp32 edge values are rounding
    noise of either sign: every pixel is covered by at most one triangle (one view per triangle) and the pixels around
    the centre by exactly one; the ids match the oracle bit for bit.  The seeds include fans that fp32 signs alone
    leave with a hole at the centre."""
    rng = np.random.default_rng(123 + persp)
    for _ in range(75):
        pos, tri, (px, py) = D.pixel_centre_fan(rng, 64, 64, persp)
        _ids_equal(dr, pos, tri, (64, 64), dev)
        cnt = _gpu_count(dr, pos, tri, (64, 64), dev)
        assert int(cnt.max()) == 1 and bool((cnt[py - 1:py + 2, px - 1:px + 2] == 1).all()), (px, py)


@pytest.mark.gpu
def test_r1_pixel_centre_grid_is_watertight(dr, dev):
    H = W = 64
    pos, tri = D.pixel_centre_grid(H, W, 3, 5, 4, 17, 18)
    _ids_equal(dr, pos, tri, (H, W), dev)
    cnt = _gpu_count(dr, pos, tri, (H, W), dev)
    assert int(cnt.max()) == 1 and bool((cnt[5:58, 6:56] == 1).all())       # vertex pixels included


def _direction_pairs():
    """For each of the 8 directions: two triangles sharing an edge through 9 pixel centres (endpoints and apexes on
    pixel centres too), the shared edge listed in the direction's order."""
    out = []
    for dx, dy in ((1, 0), (1, 1), (0, 1), (-1, 1), (-1, 0), (-1, -1), (0, -1), (1, -1)):
        c = 32
        P = lambda i, j: [D.pixel_centre(i, 64), D.pixel_centre(j, 64), 0.0, 1.0]
        a, b = P(c - 4 * dx, c - 4 * dy), P(c + 4 * dx, c + 4 * dy)
        l, r = P(c - 6 * dy, c + 6 * dx), P(c + 6 * dy, c - 6 * dx)
        pos = torch.tensor([[a, b, l, r]], dtype=torch.float32)
        out.append(((dx, dy), pos, torch.tensor([[0, 1, 2], [1, 0, 3]], dtype=torch.int32)))
    return out


def test_r1_premise_direction_edges_run_through_pixel_centres():
    for (dx, dy), pos, _ in _direction_pairs():
        a, b = pos[0, 0], pos[0, 1]
        for k in range(-3, 4):                           # the shared edge passes exactly through 7 pixel centres
            c = (D.pixel_centre(32 + k * dx, 64), D.pixel_centre(32 + k * dy, 64), 1.0)
            assert D.det3_sign_exact((a[0], a[1], 1.0), (b[0], b[1], 1.0), c) == 0


@pytest.mark.gpu
def test_r1_edges_through_pixel_centres_in_eight_directions(dr, dev):
    for d, pos, tri in _direction_pairs():
        _ids_equal(dr, pos, tri, (64, 64), dev)
        cnt = _gpu_count(dr, pos, tri, (64, 64), dev)
        assert int(cnt.max()) == 1, d
        assert all(int(cnt[32 + k * d[1], 32 + k * d[0]]) == 1 for k in range(-3, 4)), d


def _degenerate_scene():
    c = D.pixel_centre
    rows = [[c(10, 64), c(10, 64), 0, 1], [c(20, 64), c(20, 64), 0, 1], [c(30, 64), c(30, 64), 0, 1],      # collinear
            [c(40, 64), c(12, 64), 0, 1], [c(50, 64), c(12, 64), 0, 1],                                      # repeated vertex
            [0.1, 0.2, 0, 1], [0.2, 0.4, 0, 2], [0.3, 0.6, 0, 3]]                                             # same point projectively
    pos = torch.tensor([rows], dtype=torch.float32)
    tri = torch.tensor([[0, 1, 2], [3, 4, 4], [3, 3, 3], [5, 6, 7], [2, 1, 0]], dtype=torch.int32)
    return pos, tri


def test_r1_premise_degenerate_triangles_have_zero_exact_area():
    pos, tri = _degenerate_scene()
    for t in tri.tolist():
        assert D.det3_sign_exact(*[(pos[0, i, 0].item(), pos[0, i, 1].item(), pos[0, i, 3].item()) for i in t]) == 0


@pytest.mark.gpu
def test_r1_zero_area_triangles_cover_nothing(dr, dev):
    pos, tri = _degenerate_scene()
    rast, _, _ = _ids_equal(dr, pos, tri, (64, 64), dev)
    assert int((rast[..., 3] > 0).sum()) == 0


@pytest.mark.gpu
def test_r1_vertices_behind_the_eye_and_on_w0(dr, dev):
    rng = np.random.default_rng(3)
    p = torch.from_numpy(rng.uniform(-1.5, 1.5, (2, 30, 4)).astype(np.float32))
    p[..., 3] = torch.from_numpy(rng.uniform(-0.5, 1.5, (2, 30)).astype(np.float32))
    p[0, :5, 3] = 0.0
    p[..., 2] = p[..., 3] * 0.5
    tri = torch.from_numpy(rng.integers(0, 30, (40, 3)).astype(np.int32))
    assert bool((p[..., 3] <= 0).any())
    rast, _, ref = _ids_equal(dr, p, tri, (48, 40), dev)
    assert int((ref > 0).sum()) > 0


def _large_area_tris():
    """Right triangles whose kernel bounding box (fp32, one pixel of slack per side) holds 255, 256 and 258 pixels, around
    LARGE_AREA = 256 (257 is prime: no box of at least 3 x 3 pixels has that area)."""
    W = H = 64
    f32 = np.float32
    out = []
    for target in (255, 256, 258):
        found = None
        for w_px in range(3, 55):
            for h_px in range(3, 55):
                x0, y0 = 4.3, 5.7
                x1, y1 = x0 + w_px - 0.6, y0 + h_px - 0.6
                ndc = lambda v, n: float(f32(v / n * 2 - 1))
                xs = [ndc(x0, W), ndc(x1, W), ndc(x0, W)]; ys = [ndc(y0, H), ndc(y0, H), ndc(y1, H)]
                sx = [f32((f32(x) / f32(1) + f32(1)) * f32(0.5 * W)) for x in xs]
                sy = [f32((f32(y) / f32(1) + f32(1)) * f32(0.5 * H)) for y in ys]
                bx = (min(W - 1, math.ceil(max(sx) - f32(0.5)) + 1) - max(0, math.floor(min(sx) - f32(0.5)) - 1) + 1)
                by = (min(H - 1, math.ceil(max(sy) - f32(0.5)) + 1) - max(0, math.floor(min(sy) - f32(0.5)) - 1) + 1)
                if bx * by == target:
                    found = (xs, ys, bx * by)
                    break
            if found:
                break
        assert found, target
        out.append(found)
    return out


def test_r1_premise_large_area_boxes():
    assert [a for _, _, a in _large_area_tris()] == [255, 256, 258]


@pytest.mark.gpu
def test_r1_small_and_queued_triangles_at_the_large_area_split(dr, dev):
    """Both paths must give the fp32-contract ids (and the split runs with B = 2).  Which path a triangle takes is not
    observable from the outputs, by design, so this cannot tell an off-by-one in LARGE_AREA from the right split."""
    rows, tri = [], []
    for k, (xs, ys, _) in enumerate(_large_area_tris()):
        for j in range(3):
            rows.append([xs[j], ys[j], 0.1 * k - 0.2, 1.0])
        tri.append([3 * k, 3 * k + 1, 3 * k + 2])
    pos = torch.tensor([rows], dtype=torch.float32)
    pos = torch.cat([pos, pos * torch.tensor([1.0, 1.0, -1.0, 1.0])])              # B = 2, reversed depth order
    tri = torch.tensor(tri, dtype=torch.int32)
    rast, _, ref = _ids_equal(dr, pos, tri, (64, 64), dev)
    assert set(ref[0].unique().tolist()) == {0, 1, 2, 3}


@pytest.mark.gpu
@pytest.mark.parametrize("z", [1.0, -1.0])
def test_r1_depth_exactly_at_the_clip_range(dr, dev, z):
    pos = torch.tensor([[[-0.9, -0.9, z, 1.0], [0.9, -0.9, z, 1.0], [-0.9, 0.9, z, 1.0],
                         [-1.8, -1.8, 2 * z, 2.0], [1.8, -1.8, 2 * z, 2.0], [1.8, 1.8, 2 * z, 2.0]]], dtype=torch.float32)
    tri = torch.tensor([[0, 1, 2], [3, 4, 5]], dtype=torch.int32)
    rast, _, ref = _ids_equal(dr, pos, tri, (32, 32), dev)
    assert int((ref > 0).sum()) > 100
    assert bool((rast[..., 2][rast[..., 3] > 0].abs() <= 1).all())


@pytest.mark.gpu
def test_r1_equal_depths_lowest_id_wins(dr, dev):
    base = torch.tensor([[-0.9, -0.9, 0.3, 1.0], [0.9, -0.9, 0.3, 1.0], [-0.9, 0.9, 0.3, 1.0]])
    pos = torch.cat([base, base])[None].expand(2, -1, -1).contiguous()
    tri = torch.tensor([[3, 4, 5], [0, 1, 2], [3, 4, 5]], dtype=torch.int32)             # bit-identical depths
    rast, _, ref = _ids_equal(dr, pos, tri, (32, 32), dev)
    assert set(ref.unique().tolist()) == {0, 1}


@pytest.mark.gpu
def test_r1_out_of_range_indices_are_skipped(dr, dev):
    v, f, _ = D.icosphere(1)
    pos = D.clip_positions(v, O.orbit_camera(10, 20, 1.75), D.gl_perspective(49.1, 1.0))
    V = v.shape[0]
    bad = torch.tensor([[V, 0, 1], [0, -1, 2], [1, 2, 2 ** 31 - 1], [-2 ** 31, 3, 4]], dtype=torch.int32)
    tri = torch.cat([f[:30], bad, f[30:]])
    rast, _ = _rast(dr, pos, tri, (48, 48), dev)
    safe = torch.cat([f[:30], torch.zeros(4, 3, dtype=torch.int32), f[30:]])          # degenerate: skipped, ids kept
    assert torch.equal(rast[..., 3].cpu().long(), D.rasterize_ids(pos, safe, (48, 48)))


# ============================================ R2: rasterize values and backward ====================================
def _raster_bars(pos, tri, ids, res, window=None):
    """Per-pixel fp32 bars of (u, v, z/w, db0..3) and the float64 pieces of the backward bound (ids: [B, window])."""
    h, w = res
    B = pos.shape[0]
    P = pos.detach().double()
    xs, ys = D._pixel_ndc(h, w, torch.float32)
    y0, y1, x0, x1 = window if window is not None else (0, h, 0, w)
    X = xs.double()[x0:x1][None, None, :].expand_as(ids); Y = ys.double()[y0:y1][None, :, None].expand_as(ids)
    t = tri.long()[(ids - 1).clamp_min(0)]
    bidx = torch.arange(B)[:, None, None].expand_as(ids)
    p = [P[bidx, t[..., k]] for k in range(3)]
    (a0, b0, c0), (a1, b1, c1), (a2, b2, c2), det = D._tri_setup(*p)
    A = [(a0, b0, c0), (a1, b1, c1), (a2, b2, c2)]
    e = [(a * X + b * Y) + c for a, b, c in A]
    S = e[0] + e[1] + e[2]
    ab = lambda v: v.abs()
    M = []
    for i in range(3):
        pj, pk = p[(i + 1) % 3], p[(i + 2) % 3]
        M.append((ab(pj[..., 1] * pk[..., 3]) + ab(pk[..., 1] * pj[..., 3])) * ab(X) +
                 (ab(pk[..., 0] * pj[..., 3]) + ab(pj[..., 0] * pk[..., 3])) * ab(Y) + ab(pj[..., 0] * pk[..., 1]) + ab(pk[..., 0] * pj[..., 1]))
    Ei = [gam(5) * m for m in M]
    ES = Ei[0] + Ei[1] + Ei[2] + gam(2) * (ab(e[0]) + ab(e[1]) + ab(e[2]))
    Mdet = sum(ab(p[k][..., 0]) * (ab(p[(k + 1) % 3][..., 1] * p[(k + 2) % 3][..., 3]) + ab(p[(k + 2) % 3][..., 1] * p[(k + 1) % 3][..., 3]))
               for k in range(3))
    Edet = gam(5) * Mdet
    uu, vv = e[0] / S, e[1] / S
    z = [pk[..., 2] for pk in p]
    zw = (z[0] * e[0] + z[1] * e[1] + z[2] * e[2]) / det
    bu = (Ei[0] + ab(uu) * ES) / ab(S) + U * ab(uu)
    bv = (Ei[1] + ab(vv) * ES) / ab(S) + U * ab(vv)
    bz = (sum(ab(z[i]) * Ei[i] for i in range(3)) + gam(3) * sum(ab(z[i] * e[i]) for i in range(3)) + ab(zw) * Edet) / ab(det) + U * ab(zw)
    mA = lambda i, r: [ab(p[(i + 1) % 3][..., 1] * p[(i + 2) % 3][..., 3]) + ab(p[(i + 2) % 3][..., 1] * p[(i + 1) % 3][..., 3]),
                       ab(p[(i + 2) % 3][..., 0] * p[(i + 1) % 3][..., 3]) + ab(p[(i + 1) % 3][..., 0] * p[(i + 2) % 3][..., 3]),
                       ab(p[(i + 1) % 3][..., 0] * p[(i + 2) % 3][..., 1]) + ab(p[(i + 2) % 3][..., 0] * p[(i + 1) % 3][..., 1])][r]
    SAm = [sum(mA(i, r) for i in range(3)) for r in range(3)]
    SA = [A[0][r] + A[1][r] + A[2][r] for r in range(3)]
    sxy = (2.0 / w, 2.0 / h)
    bdb = []
    for i in (0, 1):
        for r in (0, 1):
            num = A[i][r] * S - e[i] * SA[r]
            d_num = gam(2) * mA(i, r) * ab(S) + ab(A[i][r]) * ES + Ei[i] * ab(SA[r]) + ab(e[i]) * gam(4) * SAm[r] + gam(2) * (ab(A[i][r] * S) + ab(e[i] * SA[r]))
            bdb.append((d_num / S ** 2 + 2 * ab(num) / ab(S) ** 3 * ES) * sxy[r] + gam(4) * ab(num / S ** 2 * sxy[r]))
    return dict(p=p, A=A, e=e, S=S, det=det, Ei=Ei, ES=ES, Edet=Edet, mA=mA, SA=SA, SAm=SAm, t=t,
                bars=[bu, bv, bz, bdb[0], bdb[1], bdb[2], bdb[3]])


def _raster_dpos_bar(info, g, ids, V):
    """Per-element bound of the kernel's position gradient (see the module docstring)."""
    B = ids.shape[0]
    hit = ids > 0
    p, A, e, S, det, Ei, ES, Edet, mA, SA, SAm = (info[k] for k in ("p", "A", "e", "S", "det", "Ei", "ES", "Edet", "mA", "SA", "SAm"))
    gu, gv = g[..., 0].double(), g[..., 1].double()
    k = 1.0 / (S * S * det).abs()
    bar = torch.zeros(B, V, 4, dtype=torch.float64); tabs = torch.zeros(B, V, 4, dtype=torch.float64)
    cnt = torch.zeros(B, V, 4, dtype=torch.float64)
    bidx = torch.arange(B)[:, None, None].expand_as(ids)
    for r, comp in ((0, 0), (1, 1), (2, 3)):
        br = k * (gu * (A[0][r] * S - e[0] * SA[r]) + gv * (A[1][r] * S - e[1] * SA[r]))
        chain = k * (gu.abs() * (A[0][r].abs() * S.abs() + e[0].abs() * SA[r].abs()) + gv.abs() * (A[1][r].abs() * S.abs() + e[1].abs() * SA[r].abs()))
        dbr = k * (gu.abs() * (gam(2) * mA(0, r) * S.abs() + A[0][r].abs() * ES + Ei[0] * SA[r].abs() + e[0].abs() * gam(4) * SAm[r]) +
                   gv.abs() * (gam(2) * mA(1, r) * S.abs() + A[1][r].abs() * ES + Ei[1] * SA[r].abs() + e[1].abs() * gam(4) * SAm[r])) + \
            (2 * ES / S.abs() + Edet / det.abs() + gam(8)) * chain
        for c in range(3):
            term = (e[c] * br).abs()
            terr = Ei[c] * br.abs() + e[c].abs() * dbr + U * term
            vi = info["t"][..., c]
            sel = hit & ((gu != 0) | (gv != 0))
            bar.index_put_((bidx[sel], vi[sel], torch.full_like(vi[sel], comp)), terr[sel], accumulate=True)
            tabs.index_put_((bidx[sel], vi[sel], torch.full_like(vi[sel], comp)), term[sel], accumulate=True)
            cnt.index_put_((bidx[sel], vi[sel], torch.full_like(vi[sel], comp)), torch.ones_like(term[sel]), accumulate=True)
    return bar + gam(cnt) * tabs + 1e-300


def _r2_scene():
    v, f, _ = D.icosphere(2)
    views = [(20, 30), (-10, 200)]
    proj = D.gl_perspective(49.1, 1.0)
    pos = torch.cat([D.clip_positions(v, O.orbit_camera(el, az, 1.75), proj) for el, az in views])
    # grazing slivers: 20 px long, 1e-3 .. 1e-1 px wide, along pixel-centre rows (one above, one below the row, so one
    # of each pair covers the row's centres), in front of the sphere
    rng = np.random.default_rng(5)
    extra, et = [], []
    V = v.shape[0]
    for s in range(4):
        x0, y0 = int(rng.integers(4, 24)), int(rng.integers(4, 44))
        wid = 10.0 ** rng.uniform(-3, -1) * 2 / 48
        for sgn in (1, -1):
            k = len(extra)
            extra += [[D.pixel_centre(x0, 48), D.pixel_centre(y0, 48), -0.99, 1.0], [D.pixel_centre(x0 + 20, 48), D.pixel_centre(y0, 48), -0.99, 1.0],
                      [D.pixel_centre(x0 + 10, 48), D.pixel_centre(y0, 48) + sgn * wid, -0.99, 1.0]]
            et.append([V + k, V + k + 1, V + k + 2])
    ex = torch.tensor(extra, dtype=torch.float32)[None].expand(2, -1, -1)
    return torch.cat([pos, ex], 1).contiguous(), torch.cat([f, torch.tensor(et, dtype=torch.int32)]), (48, 48)


def test_r2_premise_grazing_triangles_have_small_S():
    pos, tri, res = _r2_scene()
    ids = D.rasterize_ids(pos, tri, res)
    info = _raster_bars(pos, tri, ids, res)
    hit = ids > 0
    cond = (info["ES"] / info["S"].abs())[hit]
    grazing = (ids > tri.shape[0] - 8)
    assert int(grazing.sum()) > 0 and float(cond.max()) > 20 * float(cond.median())


@pytest.mark.gpu
def test_r2_rasterize_values_and_position_gradient(dr, dev):
    pos, tri, res = _r2_scene()
    rast, db, ids = _ids_equal(dr, pos, tri, res, dev)
    ref, ref_db = D.rasterize(pos.double(), tri, res)
    info = _raster_bars(pos, tri, ids, res)
    hit = ids > 0
    sphere = hit & (ids <= tri.shape[0] - 8)          # the fixed caps leave out the grazing slivers (element bars only)
    print(f"R2: {int((hit & ~sphere).sum())} grazing-sliver pixels, largest condition E_S/|S| "
          f"{float((info['ES'] / info['S'].abs())[hit].max()):.3g}")
    for ch, nm in ((0, "u"), (1, "v"), (2, "z/w")):
        check(f"R2 {nm}", rast[..., ch], ref[..., ch], info["bars"][ch], math.inf, hit)
        check(f"R2 {nm} (sphere)", rast[..., ch], ref[..., ch], info["bars"][ch], REL_VAL * 10, sphere)
    for ch in range(4):
        check(f"R2 rast_db[{ch}]", db[..., ch], ref_db[..., ch], info["bars"][3 + ch], math.inf, hit)
        check(f"R2 rast_db[{ch}] (sphere)", db[..., ch], ref_db[..., ch], info["bars"][3 + ch], REL_VAL * 20, sphere)
    assert float(rast[..., :2][~hit.to(dev)].abs().max()) == 0 and float(db[~hit.to(dev)].abs().max()) == 0
    g = torch.rand(pos.shape[0], *res, 4, generator=torch.Generator().manual_seed(2)) - 0.5
    p64 = pos.double().requires_grad_(True)
    r64, _ = D.rasterize(p64, tri, res)
    (r64[..., :2] * g[..., :2].double()).sum().backward()
    pg = pos.clone().to(dev).requires_grad_(True)
    rg, _ = dr.rasterize(dr.RasterizeCudaContext(), pg, tri.to(dev), res)
    (rg * g.to(dev)).sum().backward()
    bar = _raster_dpos_bar(info, g, ids, pos.shape[1])
    check("R2 d pos", pg.grad, p64.grad, bar, math.inf)
    on_sphere = torch.zeros_like(bar, dtype=torch.bool); on_sphere[:, :pos.shape[1] - 24] = True
    check("R2 d pos (sphere vertices)", pg.grad, p64.grad, bar, REL_GRAD * 10, on_sphere)


# ============================================ I: interpolate ======================================================
@pytest.mark.gpu
@pytest.mark.parametrize("A", [1, 3, 5, 16])
@pytest.mark.parametrize("attr_b", [1, 2])
@pytest.mark.parametrize("with_da", [False, True])
def test_i_interpolate_forward_and_backward(dr, dev, A, attr_b, with_da):
    pos, tri, res = _r2_scene()
    B = pos.shape[0]
    rast, db = _rast(dr, pos, tri, res, dev)
    r64, d64 = rast.cpu().double(), db.cpu().double()
    gen = torch.Generator().manual_seed(A * 10 + attr_b)
    attr = torch.randn(attr_b, pos.shape[1], A, generator=gen)
    ag = attr.clone().to(dev).requires_grad_(True)
    a64 = attr.double().requires_grad_(True)
    out, da = dr.interpolate(ag, rast, tri.to(dev), rast_db=db if with_da else None, diff_attrs="all" if with_da else None)
    o64, da64 = D.interpolate(a64, r64, tri, rast_db=d64 if with_da else None, diff_attrs="all" if with_da else None)
    ids = r64[..., 3].long(); hit = ids > 0
    t = tri.long()[(ids - 1).clamp_min(0)]
    ab = attr.double() if attr_b == B else attr.double().expand(B, -1, -1)
    bidx = torch.arange(B)[:, None, None].expand(B, *res)
    a0, a1, a2 = (ab[bidx, t[..., k]].abs() for k in range(3))
    uu, vv = r64[..., 0:1].abs(), r64[..., 1:2].abs()
    w2 = (1 - r64[..., 0:1] - r64[..., 1:2]).abs()
    bar = gam(4) * (uu * a0 + vv * a1 + w2 * a2) + 2 * U * (1 + uu + vv) * a2 + 1e-300
    check(f"I out A={A} attr_B={attr_b}", out, o64, bar, REL_VAL)
    assert float(out[~hit.to(dev)].abs().max()) == 0
    g = torch.randn(*o64.shape, generator=gen).double()
    loss64 = (o64 * g).sum()
    lossg = (out * g.to(dev)).sum()
    gda = None
    if with_da:
        bda = torch.stack([gam(3) * (d64[..., 0:1].abs() * (a0 + a2) + d64[..., 2:3].abs() * (a1 + a2)),
                           gam(3) * (d64[..., 1:2].abs() * (a0 + a2) + d64[..., 3:4].abs() * (a1 + a2))], -1).reshape(B, *res, 2 * A) + 1e-300
        check(f"I out_da A={A} attr_B={attr_b}", da, da64, bda, REL_VAL * 10)
        assert float(da[~hit.to(dev)].abs().max()) == 0
        gda = torch.randn(*da64.shape, generator=gen).double()
        loss64 = loss64 + (da64 * gda).sum(); lossg = lossg + (da * gda.to(dev)).sum()
    loss64.backward(); lossg.backward()
    # sum |term| per attribute element: |u g| + |v g| + |w g| (+ |db . g_da| terms), scattered like the kernel does
    mag = torch.zeros(attr_b, pos.shape[1], A, dtype=torch.float64); cnt = torch.zeros_like(mag)
    gab = g.abs()
    terms = [uu * gab, vv * gab, w2 * gab]
    if with_da:
        gx, gy = gda.reshape(B, *res, A, 2).abs().unbind(-1)
        c0 = d64[..., 0:1].abs() * gx + d64[..., 1:2].abs() * gy; c1 = d64[..., 2:3].abs() * gx + d64[..., 3:4].abs() * gy
        terms = [terms[0] + c0, terms[1] + c1, terms[2] + c0 + c1]
    bsel = bidx if attr_b == B else torch.zeros_like(bidx)
    w2err = torch.zeros_like(mag)                       # 1 - u - v in fp32: an absolute 2u (1 + |u| + |v|) per term
    for k in range(3):
        mag.index_put_((bsel[hit], t[..., k][hit]), terms[k][hit], accumulate=True)
        cnt.index_put_((bsel[hit], t[..., k][hit]), torch.ones_like(terms[k][hit]), accumulate=True)
    w2err.index_put_((bsel[hit], t[..., 2][hit]), (2 * U * (1 + uu + vv) * gab)[hit], accumulate=True)
    check(f"I d attr A={A} attr_B={attr_b} da={with_da}", ag.grad, a64.grad, gam(cnt + 4) * mag + 1.01 * w2err + 1e-300, REL_GRAD)


@pytest.mark.gpu
def test_i_diff_attrs_subset_is_refused_and_all_equals_the_full_list(dr, dev):
    pos, tri, res = _r2_scene()
    rast, db = _rast(dr, pos, tri, res, dev)
    attr = torch.randn(1, pos.shape[1], 3, device=dev)
    with pytest.raises(NotImplementedError):
        dr.interpolate(attr, rast, tri.to(dev), rast_db=db, diff_attrs=[0, 2])
    _, d_all = dr.interpolate(attr, rast, tri.to(dev), rast_db=db, diff_attrs="all")
    _, d_lst = dr.interpolate(attr, rast, tri.to(dev), rast_db=db, diff_attrs=[0, 1, 2])
    assert torch.equal(d_all, d_lst)


# ============================================ T: texture ==========================================================
def _tex_ref_uv(tex, uv):
    """uv for the float64 reference that reproduces the kernel's fp32 texel coordinate x = fl(fl(uv W) - 1/2) (which
    fixes the cell and the fraction, as the ids do for the rasterizer), and the pixels where it does not (counted)."""
    Ht, Wt = tex.shape[1], tex.shape[2]
    x32 = uv[..., 0] * Wt - 0.5; y32 = uv[..., 1] * Ht - 0.5
    ur = torch.stack([(x32.double() + 0.5) / Wt, (y32.double() + 0.5) / Ht], -1)
    moved = (torch.floor(ur[..., 0] * Wt - 0.5) != torch.floor(x32.double())) | (torch.floor(ur[..., 1] * Ht - 0.5) != torch.floor(y32.double()))
    return ur, moved


def _tex_cases():
    g = torch.Generator().manual_seed(9)
    cases = []
    # texel centres and texel borders (power-of-two sizes: uv W - 1/2 is exact)
    i = torch.arange(16, dtype=torch.float32)
    uvc = torch.stack(torch.meshgrid((i + 0.5) / 16, (i + 0.5) / 8, indexing="xy"), -1)[None]
    uvb = torch.stack(torch.meshgrid(i / 16, i / 8, indexing="xy"), -1)[None]
    cases += [("centres", torch.rand(1, 8, 16, 3, generator=g), uvc, "wrap"), ("borders", torch.rand(1, 8, 16, 3, generator=g), uvb, "wrap")]
    seam = torch.tensor([0.0, 1.0, -1.0, -0.25, 2.0, -0.03125, 1.03125, 0.5], dtype=torch.float32)
    uvs = torch.stack(torch.meshgrid(seam, seam, indexing="xy"), -1)[None]
    cases += [("wrap seam", torch.rand(1, 8, 16, 4, generator=g), uvs, "wrap"), ("clamp border", torch.rand(1, 8, 16, 4, generator=g), uvs, "clamp")]
    for big in (1e4, 1e7):
        uvh = ((torch.rand(1, 12, 12, 2, generator=g) * 2 - 1) * big).float()
        cases += [(f"|uv| {big:g} wrap", torch.rand(1, 16, 16, 3, generator=g), uvh, "wrap"),
                  (f"|uv| {big:g} clamp", torch.rand(1, 16, 16, 3, generator=g), uvh, "clamp")]
    uvr = torch.rand(2, 10, 12, 2, generator=g) * 3 - 1
    for (th, tw) in ((1, 1), (1, 7), (7, 1)):
        cases.append((f"tex {th}x{tw}", torch.rand(1, th, tw, 3, generator=g), uvr, "wrap"))
    for C in (1, 3, 4, 5):
        cases.append((f"C={C}", torch.rand(1, 8, 12, C, generator=g), uvr, "wrap"))
    cases.append(("tex_B=2", torch.rand(2, 8, 12, 3, generator=g), uvr, "clamp"))
    return cases


def test_t_premise_centres_and_borders_are_exact_in_fp32():
    cases = _tex_cases()
    for name, tex, uv, _ in cases[:2]:
        x = uv[..., 0] * tex.shape[2] - 0.5
        frac = (x - torch.floor(x)).unique().tolist()
        assert frac == ([0.0] if name == "centres" else [0.5])              # centres: the cell switches exactly here
    big = [c for c in cases if c[0].startswith("|uv| 1e+07")][0]
    assert float(big[2].abs().max()) > 2 ** 23 / 16                          # x = uv W beyond 2^23: no fraction bits left
    for _, tex, uv, _ in cases:
        assert int(_tex_ref_uv(tex, uv)[1].sum()) == 0


@pytest.mark.gpu
def test_t_texture_forward_and_backward(dr, dev):
    for name, tex, uv, mode in _tex_cases():
        ur, moved = _tex_ref_uv(tex, uv)
        assert int(moved.sum()) == 0, name
        tg = tex.clone().to(dev).requires_grad_(True); ug = uv.clone().to(dev).requires_grad_(True)
        t64 = tex.double().requires_grad_(True); u64 = ur.clone().requires_grad_(True)
        out = dr.texture(tg, ug, filter_mode="linear", boundary_mode=mode)
        ref = D.texture(t64, u64, "linear", mode)
        tmax = float(tex.abs().max())
        check(f"T out {name}", out, ref, gam(7) * tmax, REL_VAL)
        g = torch.rand(*ref.shape, generator=torch.Generator().manual_seed(1)).double() - 0.5
        (out * g.to(dev)).sum().backward(); (ref * g).sum().backward()
        n = uv.shape[0] * uv.shape[1] * uv.shape[2] * 4
        check(f"T d tex {name}", tg.grad, t64.grad, gam(n + 3) * float(g.abs().sum()), REL_GRAD)
        C = tex.shape[3]
        ubar = (g.abs().sum(-1) * 2 * tmax * gam(C + 6))[..., None] * torch.tensor([tex.shape[2], tex.shape[1]]).double() + 1e-300
        check(f"T d uv {name}", ug.grad, u64.grad, ubar, REL_GRAD)


@pytest.mark.gpu
def test_t_border_gradient_takes_the_upper_cell(dr, dev):
    """At x = uv W - 1/2 exactly on an integer the cell [x, x + 1] is used (fx = 0): d/du = W (t[x+1] - t[x])."""
    tex = torch.tensor([[0.0, 1.0, 3.0, 7.0]]).reshape(1, 1, 4, 1)
    uv = torch.tensor([[[[1.5 / 4, 0.5]]]])
    ug = uv.clone().to(dev).requires_grad_(True)
    dr.texture(tex.to(dev), ug, filter_mode="linear").sum().backward()
    assert float(ug.grad[0, 0, 0, 0]) == 4 * (3.0 - 1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["isotropic", "zero", "integer_lod", "max_mip_level", "odd_size"])
def test_t_mip_path(dr, dev, case):
    g = torch.Generator().manual_seed(4)
    Ht, Wt = (24, 40) if case == "odd_size" else (32, 32)
    tex = torch.rand(1, Ht, Wt, 3, generator=g)
    uv = torch.rand(1, 12, 14, 2, generator=g)
    if case == "isotropic":
        da = torch.zeros(1, 12, 14, 4); da[..., 0] = 3.0 / Wt; da[..., 3] = 3.0 / Ht
    elif case == "zero":
        da = torch.zeros(1, 12, 14, 4)
    elif case == "integer_lod":
        da = torch.zeros(1, 12, 14, 4); da[..., 0] = 4.0 / Wt; da[..., 3] = 1.0 / Ht
    else:
        da = (torch.rand(1, 12, 14, 4, generator=g) - 0.5) * 0.4
    mml = 2 if case == "max_mip_level" else None
    tg = tex.clone().to(dev).requires_grad_(True); ug = uv.clone().to(dev).requires_grad_(True); dg = da.clone().to(dev).requires_grad_(True)
    t64 = tex.double().requires_grad_(True); u64 = uv.double().requires_grad_(True); d64 = da.double().requires_grad_(True)
    out = dr.texture(tg, ug, uv_da=dg, max_mip_level=mml)
    ref = D.texture(t64, u64, "linear-mipmap-linear", uv_da=d64, max_mip_level=mml)
    check(f"T mip {case}", out, ref, 64 * U, REL_VAL * 10)
    w = torch.rand(*ref.shape, generator=g).double()
    (out * w.to(dev)).sum().backward(); (ref * w).sum().backward()
    for nm, a, b in (("tex", tg.grad, t64.grad), ("uv", ug.grad, u64.grad), ("uv_da", dg.grad, d64.grad)):
        assert bool(torch.isfinite(a).all()), (case, nm)
        scale = float(b.abs().max()) + 1e-30
        check(f"T mip {case} d {nm}", a, b, 1e-4 * scale + 1e-12, REL_GRAD * 100)


def test_t_mip_premises():
    pyr = D.mip_pyramid(torch.zeros(1, 24, 40, 1))
    assert [tuple(t.shape[1:3]) for t in pyr] == [(24, 40), (12, 20), (6, 10), (3, 5)]        # stops at an odd side
    assert len(D.mip_pyramid(torch.zeros(1, 32, 32, 1), 2)) == 3
    da = torch.zeros(1, 1, 1, 4); da[..., 0] = 4.0 / 32; da[..., 3] = 1.0 / 32
    assert float(D.mip_level(da, 32, 32, 6)) == 2.0                                         # LOD exactly on an integer


# ============================================ A: antialias ========================================================
G16 = 1.0 / 16


def _aa_pos(pts_px, H, W, w=None):
    """Vertices given in pixel units on a 1/16-pixel grid (exact in fp32), clip space with w = 1 unless given."""
    rows = []
    for k, (x, y, z) in enumerate(pts_px):
        ww = 1.0 if w is None else w[k]
        rows.append([(x * 2.0 / W - 1.0) * ww, (y * 2.0 / H - 1.0) * ww, z * ww, ww])
    return torch.tensor([rows], dtype=torch.float32)


def _aa_scenes():
    H = W = 32
    sc = {}
    # silhouette crossing at t = 0, 0.5 and 1 from the covered pixel, both directions (an open quad's right edge at
    # x = 10.5 + t, rows on pixel centres -> fa = 0 exactly at the edge's lower vertex)
    for t in (0.0, 0.5, 1.0):
        for flip in (False, True):
            xe = 10.5 + t
            pts = [(2.5, 3.5, 0.1), (xe, 3.5, 0.1), (xe, 27.5, 0.1), (2.5, 27.5, 0.1)]
            if flip:
                pts = [(W - x, y, z) for x, y, z in pts]
            sc[f"t={t} {'<-' if flip else '->'}"] = (_aa_pos(pts, H, W), torch.tensor([[0, 1, 2], [0, 2, 3]], dtype=torch.int32))
    # image-border pixels: a triangle running off the frame
    sc["border"] = (_aa_pos([(-4.0, -3.0, 0.2), (40.0, 5.25, 0.2), (7.125, 40.0, 0.2)], H, W), torch.tensor([[0, 1, 2]], dtype=torch.int32))
    # open fan (boundary edges) and a non-manifold edge shared by three triangles
    sc["open fan"] = (_aa_pos([(16.0, 16.0, 0.0), (26.0625, 17.5, 0.0), (17.3125, 27.0, 0.0), (5.5, 20.25, 0.0)], H, W),
                      torch.tensor([[0, 1, 2], [0, 2, 3]], dtype=torch.int32))
    sc["non-manifold"] = (_aa_pos([(6.0, 6.0, 0.0), (24.0625, 9.0, 0.0), (14.0, 27.125, 0.3), (20.5, 24.0, -0.2), (9.25, 22.0, 0.1)], H, W),
                          torch.tensor([[0, 1, 2], [1, 0, 3], [0, 1, 4]], dtype=torch.int32))
    # a vertex behind the eye (its triangle is not antialiased), next to an ordinary one
    pb = _aa_pos([(4.0, 4.0, 0.0), (20.5, 6.0, 0.0), (10.0, 20.0, 0.0), (30.0, 28.0, 0.0)], H, W)
    pb[0, 3] = torch.tensor([0.3, 0.9, 0.0, -0.5])
    sc["behind eye"] = (pb, torch.tensor([[0, 1, 2], [1, 3, 2]], dtype=torch.int32))
    # a farther surface against background and against a nearer one
    sc["far vs near"] = (_aa_pos([(2.0, 2.0, 0.6), (30.0625, 2.0, 0.6), (2.0, 30.0625, 0.6), (8.5, 8.5, -0.4), (22.0625, 9.0, -0.4), (9.0, 24.1875, -0.4)], H, W),
                         torch.tensor([[0, 1, 2], [3, 4, 5]], dtype=torch.int32))
    return sc, (H, W)


def test_a_premise_scene_coordinates_are_exact_and_partner_rule():
    sc, (H, W) = _aa_scenes()
    for name, (pos, tri) in sc.items():
        P = pos[0].double()
        ok = P[:, 3] > 0
        s = (P[ok, :2] / P[ok, 3:4] + 1.0) * torch.tensor([W / 2, H / 2], dtype=torch.float64)
        assert bool(((s * 16) == torch.round(s * 16)).all()), name          # screen positions on the 1/16 grid
    # a crossing exactly on a pixel centre (t = 0 or 1) must come from an exact fa = 0 (or fb = 0) or an edge
    # perpendicular to the pixel pair (cross = pa whatever sp rounds to): elsewhere sp = -fa /
    # (fb - fa) rounds, and fp32 (with or without a fused multiply-add) and float64 may land on either side of t = 1
    from fractions import Fraction as Fr
    for name, (pos, tri) in sc.items():
        P = pos[0].double()
        opp_all = D.edge_opposites(tri)
        scr = lambda k: ((Fr(float(P[k, 0])) / Fr(float(P[k, 3])) + 1) * (W // 2), (Fr(float(P[k, 1])) / Fr(float(P[k, 3])) + 1) * (H // 2))
        side = lambda a, b, c: (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])
        for f_, t in enumerate(tri.tolist()):
            if not bool((P[t, 3] > 0).all()):
                continue
            S = [scr(k) for k in t]
            for e in range(3):
                a, b = S[(e + 1) % 3], S[(e + 2) % 3]
                o = int(opp_all[f_, e])
                if o >= 0 and (float(P[o, 3]) <= 0 or side(a, b, S[e]) * side(a, b, scr(o)) <= 0):
                    continue                                                   # not a silhouette edge
                for fix in (0, 1):
                    for j in range(H if fix == 1 else W):
                        c = Fr(2 * j + 1, 2)
                        fa, fb = a[fix] - c, b[fix] - c
                        if fa == fb or fa == 0 or fb == 0 or a[1 - fix] == b[1 - fix] or not ((fa < 0) != (fb < 0)):
                            continue
                        cross = a[1 - fix] + (-fa / (fb - fa)) * (b[1 - fix] - a[1 - fix])
                        assert (cross - Fr(1, 2)).denominator != 1, (name, t, e, fix, j)
    opp = D.edge_opposites(sc["non-manifold"][1])
    # edge (0,1) is shared by triangles 0, 1, 2: sorted by (edge key, triangle, edge), 0 pairs with 1 and 1, 2 with
    # their predecessor
    assert opp[0, 2] == 3 and opp[1, 2] == 2 and opp[2, 2] == 3
    assert int((D.edge_opposites(sc["open fan"][1]) < 0).sum()) == 4


@pytest.mark.gpu
def test_a_antialias_forward_and_backward(dr, dev):
    from gs_b200 import meshops
    sc, (H, W) = _aa_scenes()
    for name, (pos, tri) in sc.items():
        assert torch.equal(meshops.get_topology(tri.to(dev), pos.shape[1]).cpu().long(), D.edge_opposites(tri))
        rast, _, ids = _ids_equal(dr, pos, tri, (H, W), dev)
        g = torch.Generator().manual_seed(3)
        color = torch.rand(1, H, W, 3, generator=g)
        cg = color.clone().to(dev).requires_grad_(True); pg = pos.clone().to(dev).requires_grad_(True)
        c64 = color.double().requires_grad_(True); p64 = pos.double().requires_grad_(True)
        out = dr.antialias(cg, rast, pg, tri.to(dev))
        ref = D.antialias(c64, rast.cpu().double(), p64, tri)
        changed = (ref - c64).detach().abs().sum(-1) > 0
        print(f"A {name}: {int(changed.sum())} pixels blended")
        check(f"A out {name}", out, ref, 16 * U * (1 + W) * (1 + color.double()), REL_VAL * 10)
        w = torch.rand(*ref.shape, generator=g).double() - 0.5
        (out * w.to(dev)).sum().backward(); (ref * w).sum().backward()
        check(f"A d color {name}", cg.grad, c64.grad, 16 * U * (1 + W) * (1 + w.abs()), REL_GRAD)
        scale = float(p64.grad.abs().max())
        if scale > 0:
            check(f"A d pos {name}", pg.grad, p64.grad, 1e-5 * scale, REL_AA_POS)
        else:
            assert float(pg.grad.abs().max()) == 0.0, name
    sc_t = {k: v for k, v in sc.items() if k.startswith("t=")}
    assert len(sc_t) == 6


# ============================================ C4: config-4 scale ==================================================
@pytest.mark.gpu
def test_c4_config4_windows_ids_bit_exact_and_values(dr, dev):
    """The 327,680-triangle sphere, 8 views at 1920 x 1080: ids bit-exact against the oracle on windows at the centre,
    on the silhouette and on empty background of two views; values there within the R2 bars (the fixed cap applies at the
    centre, where no triangle is seen edge-on)."""
    H, W = 1080, 1920
    views = [(0, 45.0 * k) for k in range(8)]
    v, f, _ = D.icosphere(7)
    proj = D.gl_perspective(49.1, W / H)
    pos = torch.cat([D.clip_positions(v, O.orbit_camera(el, az, 1.75), proj) for el, az in views])
    rast, db = _rast(dr, pos, f, (H, W), dev)
    ids = rast[..., 3].long()
    hit = ids > 0
    xs = torch.nonzero(hit[0].any(0)).flatten(); lo, hi = int(xs.min()), int(xs.max())
    wins = [(520, 560, 940, 980), (520, 560, lo - 8, lo + 24), (520, 560, hi - 24, hi + 8), (0, 24, 0, 24)]
    for b in (0, 3):
        for win in wins:
            # at the silhouette the triangles are seen edge-on (small S): element bars only, as for R2's slivers
            cap = REL_VAL * 10 if win == wins[0] else math.inf
            ref = D.rasterize_ids(pos[b:b + 1], f, (H, W), window=win)
            got = ids[b:b + 1, win[0]:win[1], win[2]:win[3]].cpu()
            assert torch.equal(got, ref), (b, win, int((got != ref).sum()))
            if int((ref > 0).sum()) == 0:
                continue
            info = _raster_bars(pos[b:b + 1], f, ref, (H, W), win)
            r64 = _r64_at(pos[b:b + 1], f, ref, (H, W), win)
            m = ref > 0
            for ch in range(3):
                check(f"C4 view {b} window {win} ch {ch}", rast[b:b + 1, win[0]:win[1], win[2]:win[3], ch].cpu(), r64[..., ch],
                      info["bars"][ch], cap, m)


def _r64_at(pos, tri, ids, res, window):
    """Float64 rasterize values (u, v, z/w) on given ids over a window (the oracle's value formulas)."""
    h, w = res
    P = pos.double()
    xs, ys = D._pixel_ndc(h, w, torch.float32)
    y0, y1, x0, x1 = window
    X = xs.double()[x0:x1][None, None, :]; Y = ys.double()[y0:y1][None, :, None]
    t = tri.long()[(ids - 1).clamp_min(0)]
    p = [P[0, t[..., k]] for k in range(3)]
    (a0, b0, c0), (a1, b1, c1), (a2, b2, c2), det = D._tri_setup(*p)
    e0 = (a0 * X + b0 * Y) + c0; e1 = (a1 * X + b1 * Y) + c1; e2 = (a2 * X + b2 * Y) + c2
    S = e0 + e1 + e2
    zw = (p[0][..., 2] * e0 + p[1][..., 2] * e1 + p[2][..., 2] * e2) / det
    return torch.stack([e0 / S, e1 / S, zw], -1)
