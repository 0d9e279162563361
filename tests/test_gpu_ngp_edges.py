"""Instant-NGP kernels against a float64 evaluation of the same operation, at config-3 scale and at the edges where the
kernels go wrong: ray-ordered samples in the run-reducing hash-grid scatter (S1), points on cell faces, at the box
boundary and outside it (S2), marcher rays that are axis-parallel, start inside the box or on a face, graze an edge,
or use occupancy resolutions up to the shared-memory limit (S3), packed rays from empty to 1500 samples with empty,
saturated and subnormal-transmittance stretches (S4), the fused MLP up to 2e7 rows (S5), and one 1920 x 1080 frame of
the config-3 render (S6).  Every scene has a CPU test of its premise.

References.  Grid: the corner indices and fp32 fractions of `oracle/ngp_oracle.py`'s pinned-order
`grid_corner_indices` (bit-exact with the kernels'), with the trilinear weights, the products and every sum in float64;
per table entry also the contribution count n and sum |term|.  Weights: the sequential recurrence in float64 on the fp32
inputs (alpha = -expm1(-sigma dt)), and nerfacc's own fp32 formula 1 - exp(-x) with a correctly rounded exp, which
separates "worse than nerfacc would be" from "worse than exact".  Accumulate and MLP: float64 torch (on the GPU for the
big GEMMs).  Integer outputs (sample lists, counts) are compared bit for bit with the fp32 oracle.

Bars (derivation), u = 2^-24, gamma_n = n u / (1 - n u).  Each comparison has a per-element bar K_ELEM (= 2) times an
fp32 forward error bound, and a fixed norm-relative bar.
- Grid scatter: a term w g has <= 6 roundings (1 - frac, two weight products, the product with g), the run kernel's
  shuffle tree adds <= 5 levels, and the reds into an entry are a sum of <= n terms in any order: |err| <=
  gamma_(n + 11) sum |term|.  Forward feature: 8 sequential fmas of such weights: gamma_13 sum |w e|.  TV: one
  rounding of weight * (integer sum) and n reds: gamma_(n + 2) sum |term|.
- Weights (per ray, first order): x = sigma (te - ts) has two roundings; -expm1f is within 1 ulp, so
  e_a = 2u x e^-x + 2u a.  c = 1 - a: e_c = e_a + u c.  T_(i+1) = T_i c_i: E_(i+1) = E_i (c + e_c) + T_i e_c +
  u T_(i+1) + 2^-149 (the last term covers a subnormal rounding).  w = T a: E_w = E a + T e_a + E e_a + u w + 2^-149.
  Backward: dalpha = gw T + ga - G T, G_i = gt + gw a + G c, each with <= 4 roundings on its |terms| plus the input
  errors E, e_a, e_c carried through the same recurrences (`weights_bounds`).  nerfacc's formula: |a_ref - a| <= u/2
  e^-x + u/2 a + u x e^-x; the kernel's alpha must stay within twice that.
- Accumulate: out = sum of n products, gamma_(n + 1) sum |w v|; dw = sum of C products, gamma_C sum |g v|; dv one
  rounding.
- MLP: y and dL/dx are dot products of Din + H and H + Dout terms with fp32 intermediates: gamma_(Din + H + Dout)
  times the |.|-chain.  The weight gradients are sums over the rows: each tile of 128 rows is summed, the tile sums of a
  CTA are added in turn, the CTAs' totals meet in reds: gamma_(128 + tiles per CTA + CTAs + Dout + Din) times the
  |.|-product.  Rows whose fp64 hidden pre-activation lies within 4 gamma_Din sum |W1 x| of 0 (where fp32's ReLU mask
  may differ) get zero upstream gradient; their count is reported.
- Config-3 frame: the chain through exp, sigmoid and the ReLU masks has no useful worst-case bound, so S6 uses fixed
  bars only: the image to C6_IMG absolute, the gradients to C6_REL norm-relative and to C6_ELEM of the largest
  element; rays with a sample whose fp64 hidden pre-activation lies within 64 u sum |W1 f| of 0 get no upstream gradient.
The fixed norm-relative bars are ten or more times tighter than `test_gpu_ngp.py`'s.  Tests print each scene's worst
error against both bars."""
import ctypes as C
import math
from functools import lru_cache

import numpy as np
import pytest
import torch

from oracle import gs_oracle as O
from oracle import ngp_oracle as G

U = 2.0 ** -24
TINY = 2.0 ** -149
K_ELEM = 2.0
GRID_REL = 1e-5            # hash-grid gradients and features, norm-relative (the suite's ray-ordered bar is 1e-3)
W_REL = 1e-6               # weights / transmittance / alpha / accumulate, norm-relative
DSIG_REL = 1e-5            # d sigma, norm-relative
MLP_REL = 5e-6             # MLP weight gradients, norm-relative (dL/dx and y: MLP_REL / 5)
C6_IMG = 2e-5
C6_REL = 1e-4
C6_ELEM = 1e-3
PLS3 = float(np.exp2(np.log2(512 / 16) / 15))       # config 3: GridEncoder(num_levels=16, desired_resolution=512)
AABB = torch.tensor([-1.0, -1, -1, 1, 1, 1])
# (num_levels, per_level_scale, base_resolution): config 3; all levels per sample; fewer levels than the coarse cap;
# the reference's grids
GRID_CASES = {"c3": (16, PLS3, 16), "base160": (4, 2.0, 160), "L2": (2, 2.0, 16), "L12": (12, 2.0, 16)}


def gam(n):
    n = np.asarray(n, dtype=np.float64)
    return n * U / (1.0 - n * U)


def report(name, err, bar, ref=None):
    """worst error / element bar, and the norm-relative error; returns (ratio, rel)"""
    err = np.abs(np.asarray(err, dtype=np.float64)).ravel()
    bar = np.asarray(bar, dtype=np.float64).ravel()
    ratio = float((err / np.maximum(bar, 1e-300)).max()) if err.size else 0.0
    rel = float(np.linalg.norm(err) / max(np.linalg.norm(ref), 1e-300)) if ref is not None else float("nan")
    print(f"{name}: max err {float(err.max()) if err.size else 0.0:.3g}, worst err/bar {ratio:.3g}, norm-rel {rel:.3g}")
    return ratio, rel


def coarse_l0(L, pls, base):
    """levels the backward sends through the run-reducing kernel: resolution <= 128, at most 8 (ngp_ops.cu)"""
    l0 = 0
    while l0 < L and G._level_geometry(l0, pls, base)[1] <= 128 and l0 < 8:
        l0 += 1
    return l0


# ---------------------------------------------------------------------------------------------------------------------
# float64 hash-grid reference
# ---------------------------------------------------------------------------------------------------------------------
def grid_ref64(x, L, pls, base, g=None, emb=None):
    """x [N,3] fp32 in [-1,1] (any device).  Returns dict: d_emb / n / abs (per entry, from g [N,2L]) and feat / feat_abs
    (from emb [T,2]); float64 throughout after the oracle's integer indices and fp32 fractions."""
    off = G.grid_offsets(num_levels=L, per_level_scale=pls, base_resolution=base)
    x01 = (x.float() + 1.0) / 2.0
    T = int(off[-1])
    res = {}
    if g is not None:
        res["d_emb"] = torch.zeros(T, 2, dtype=torch.float64, device=x.device)
        res["abs"] = torch.zeros(T, 2, dtype=torch.float64, device=x.device)
        res["n"] = torch.zeros(T, dtype=torch.int64, device=x.device)
    if emb is not None:
        res["feat"] = torch.zeros(x.shape[0], 2 * L, dtype=torch.float64, device=x.device)
        res["feat_abs"] = torch.zeros_like(res["feat"])
    for l in range(L):
        idx, _, frac = G.grid_corner_indices(x01, l, off, pls, base)
        f = frac.double()
        w = torch.stack([math.prod((f[:, d] if (c >> d) & 1 else 1.0 - f[:, d]) for d in range(3)) for c in range(8)], 1)
        gi = idx + int(off[l])
        if g is not None:
            term = w[:, :, None] * g[:, None, 2 * l:2 * l + 2].double()
            res["d_emb"].index_add_(0, gi.reshape(-1), term.reshape(-1, 2))
            res["abs"].index_add_(0, gi.reshape(-1), term.abs().reshape(-1, 2))
            nz = (g[:, 2 * l:2 * l + 2] != 0).any(1)
            res["n"].index_add_(0, gi[nz].reshape(-1), torch.ones_like(gi[nz].reshape(-1)))
        if emb is not None:
            e = emb.double()[gi]                                      # [N,8,2]
            res["feat"][:, 2 * l:2 * l + 2] = (e * w[:, :, None]).sum(1)
            res["feat_abs"][:, 2 * l:2 * l + 2] = (e.abs() * w[:, :, None]).sum(1)
    return res


def check_grid_bwd(name, d_emb, ref):
    d = d_emb.double().to(ref["d_emb"].device)
    err = (d - ref["d_emb"]).abs()
    bar = K_ELEM * torch.from_numpy(gam(ref["n"].cpu().numpy() + 11.0)).to(d.device)[:, None] * ref["abs"]
    untouched = ref["n"] == 0
    assert bool((d[untouched] == 0).all()), f"{name}: gradient in an entry no sample reaches"
    ratio, rel = report(name, err.cpu().numpy(), bar.cpu().numpy(), ref["d_emb"].cpu().numpy())
    assert ratio <= 1.0 and rel <= GRID_REL, (name, ratio, rel)


def _grid_bwd_abi(x, g, L, pls, base, misalign=False):
    """ngp_b200_grid_encode_bwd through the C ABI; misalign: d_emb 8 bytes past a 16-byte boundary (the .v4 reds off)"""
    from gs_b200 import _lib
    from kiui.gridencoder import GridEncoder
    enc = GridEncoder(num_levels=L, per_level_scale=pls, base_resolution=base)
    T = int(enc._offsets_np[-1])
    buf = torch.zeros(2 * T + 4, device=x.device)
    base_ptr = buf.data_ptr()
    assert base_ptr % 16 == 0
    start = 2 if misalign else 0
    d_emb = buf[start:start + 2 * T].view(T, 2)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(_lib.lib.ngp_b200_grid_encode_bwd(C.c_void_p(x.data_ptr()), x.shape[0], enc._off_ptr, L, 1.0, float(pls), int(base),
                                                 C.c_void_p(g.data_ptr()), C.c_void_p(d_emb.data_ptr()), stream))
    torch.cuda.synchronize()
    return d_emb.clone()


# ---------------------------------------------------------------------------------------------------------------------
# S1: ray-ordered samples from the marcher on a config-3-like camera
# ---------------------------------------------------------------------------------------------------------------------
def _binary_ball(R, radius):
    g = (torch.arange(R).float() + 0.5) / R * 2 - 1
    x, y, z = torch.meshgrid(g, g, g, indexing="ij")
    return (x * x + y * y + z * z) < radius * radius


@lru_cache(maxsize=None)
def c3_rays():
    return G.get_rays(O.orbit_camera(0, 30, 1.75), 1080, 1920, 49.1)


@lru_cache(maxsize=None)
def s1_samples():
    """samples of a 24 x 20 block of the 1920 x 1080 config-3 rays (centre and silhouette rows of the sphere r = 0.5 on
    a 64^3 grid, step 5e-3, stratified), then a 12 x 20 block of a camera on the cube diagonal (cells crossed corner to
    corner: runs of up to 46 samples at resolution 16), trimmed to N not a multiple of 32; gout uniform in [-1, 1)"""
    xs = []
    for k, (cam, rows) in enumerate(((c3_rays(), torch.cat([torch.arange(520, 532), torch.arange(700, 712)])),
                                     (G.get_rays(O.orbit_camera(35.26, -45, 1.75), 1080, 1920, 49.1), torch.arange(530, 542)))):
        ro, rd = cam
        sel = (rows[:, None] * 1920 + torch.arange(950, 970)[None, :]).reshape(-1)
        toff = torch.rand(sel.numel(), generator=torch.Generator().manual_seed(31 + k)) * 5e-3
        ri, t0, t1 = G.march(ro[sel], rd[sel], _binary_ball(64, 0.5), AABB, 0.01, 100.0, 5e-3, toff)
        xs.append(ro[sel][ri] + rd[sel][ri] * (t0 + t1)[:, None] / 2.0)
    x = torch.cat(xs)
    n = x.shape[0] - (1 if x.shape[0] % 32 == 0 else 0)
    x = x[:n].contiguous()
    g = torch.rand(n, 32, generator=torch.Generator().manual_seed(32)) * 2 - 1
    return x, g


def warp_runs(keys):
    """keys [N] int64 in sample order -> (lengths of the runs of equal keys inside each 32-sample warp, lengths of the
    runs over the whole sequence, number of runs that continue across a lane-31 / lane-0 boundary)"""
    k = keys.numpy()
    n = k.size
    brk = np.ones(n, dtype=bool)
    brk[1:] = k[1:] != k[:-1]
    glob = np.diff(np.flatnonzero(np.r_[brk, True]))
    wb = brk.copy()
    wb[::32] = True
    warp = np.diff(np.flatnonzero(np.r_[wb, True]))
    cross = int((~brk[32::32]).sum())
    return warp, glob, cross


def s1_premise_stats():
    x, _ = s1_samples()
    L, pls, base = GRID_CASES["c3"]
    off = G.grid_offsets(num_levels=L, per_level_scale=pls, base_resolution=base)
    x01 = (x + 1.0) / 2.0
    stats = {}
    for l in range(coarse_l0(L, pls, base)):
        scale, _ = G._level_geometry(l, pls, base)
        pg = torch.floor(x01 * float(scale) + 0.5).to(torch.int64)
        key = pg[:, 0] | (pg[:, 1] << 10) | (pg[:, 2] << 20)
        kxy = pg[:, 0] | (pg[:, 1] << 10)
        w, gl, cr = warp_runs(key)
        # cells that differ in z only, next to each other inside one warp
        same_w = (torch.arange(x.shape[0] - 1) % 32) != 31
        zonly = int(((kxy[1:] == kxy[:-1]) & (key[1:] != key[:-1]) & same_w).sum())
        stats[l] = (w, gl, cr, zonly)
    return x.shape[0], off, stats


def test_s1_premise():
    N, off, stats = s1_premise_stats()
    assert N % 32 and N % 256 and N > 50000
    # config 3's level geometry: the scale of level 9 is 16 * 2^3 - 1 = 127 exactly in torch-ngp's fp32 formula, so its
    # resolution is 128 (not 129), and the coarse cap of 8 levels (not the resolution) ends the run kernel's levels
    L, pls, base = GRID_CASES["c3"]
    assert G._level_geometry(9, pls, base) == (np.float32(127.0), 128)
    assert [G._level_geometry(l, pls, base)[1] for l in (3, 6, 12, 15)] == [32, 64, 256, 512]
    assert coarse_l0(*GRID_CASES["c3"]) == 8 and G._level_geometry(8, pls, base)[1] <= 128
    assert coarse_l0(*GRID_CASES["base160"]) == 0 and coarse_l0(*GRID_CASES["L2"]) == 2 and coarse_l0(*GRID_CASES["L12"]) == 4
    # level 7 is the first hashed level and is a run-kernel level; 3 and 6 are dense
    for l, hashed in ((3, False), (6, False), (7, True), (8, True)):
        res = G._level_geometry(l, pls, base)[1]
        assert ((res + 1) ** 3 > int(off[l + 1] - off[l])) == hashed, l
    all_w = np.concatenate([s[0] for s in stats.values()])
    all_g = np.concatenate([s[1] for s in stats.values()])
    for length in (1, 2, 31, 32):
        assert (all_w == length).any(), length
    assert (all_g > 32).any()
    assert sum(s[2] for s in stats.values()) > 0                     # runs continuing across a lane-31 / lane-0 boundary
    assert sum(s[3] for s in stats.values()) > 0                     # neighbours in one warp that differ in z only
    print({l: (int(s[0].max()), int(s[1].max()), s[2], s[3]) for l, s in stats.items()})


# ---------------------------------------------------------------------------------------------------------------------
# S2: grid geometry edges
# ---------------------------------------------------------------------------------------------------------------------
def _pos32(x, scale):
    x01 = np.float32(np.float32(np.float32(x) + np.float32(1.0)) / np.float32(2.0))
    return np.float32(np.float32(x01 * np.float32(scale)) + np.float32(0.5))


def face_coordinate(scale, m):
    """an fp32 x in [-1, 1] whose position at this level's scale is exactly the integer m (a cell face), or None"""
    x0 = np.float32(2.0 * (m - 0.5) / float(scale) - 1.0)
    for k in range(0, 200):
        for s in (1, -1):
            x = x0
            for _ in range(k):
                x = np.nextafter(x, np.float32(s * 2.0), dtype=np.float32)
            if -1.0 <= x <= 1.0 and _pos32(x, scale) == np.float32(m):
                return x
    return None


@lru_cache(maxsize=None)
def s2_points(L, pls, base):
    """points with one coordinate on a cell face of every level (several faces per level and axis), box corners and
    faces, one ulp inside +-1, and random points; all in [-1, 1]"""
    rng = np.random.default_rng(21)
    pts = []
    for l in range(L):
        scale, res = G._level_geometry(l, pls, base)
        for m in sorted(set([1, 2, res // 2, res // 2 + 1, res - 1] + rng.integers(1, res, 4).tolist())):
            c = face_coordinate(scale, m)
            if c is None:
                continue
            for a in range(3):
                p = rng.uniform(-1, 1, 3).astype(np.float32)
                p[a] = c
                pts.append(p)
    one_in = np.nextafter(np.float32(1.0), np.float32(0.0), dtype=np.float32)
    for v in ([-1, -1, -1], [1, 1, 1], [1, -1, 1], [-1, 1, -1], [1, 0.3, -0.2], [-1, 0.3, 0.7], [one_in, one_in, one_in],
              [-one_in, -one_in, -one_in], [one_in, -one_in, 0.1], [0, 0, 0]):
        pts.append(np.array(v, dtype=np.float32))
    pts += list(rng.uniform(-1, 1, (2000, 3)).astype(np.float32))
    return torch.from_numpy(np.stack(pts)).contiguous()


def s2_face_counts(x, L, pls, base):
    x01 = (x + 1.0) / 2.0
    out = []
    for l in range(L):
        scale, _ = G._level_geometry(l, pls, base)
        pos = x01 * float(scale) + 0.5
        out.append([int((pos[:, a] == torch.floor(pos[:, a])).sum()) for a in range(3)])
    return out


@lru_cache(maxsize=None)
def tv_points(L, pls, base):
    """TV edges inside the box: corners (pg = 0 on every level at x = -1), one ulp inside +1, and random points"""
    rng = np.random.default_rng(22)
    one_in = np.nextafter(np.float32(1.0), np.float32(0.0), dtype=np.float32)
    pts = [np.array(v, dtype=np.float32) for v in ([-1, -1, -1], [1, 1, 1], [one_in, -1, 0.2], [-1, one_in, one_in])]
    pts += list(rng.uniform(-1, 1, (3000, 3)).astype(np.float32))
    return torch.from_numpy(np.stack(pts)).contiguous()


# pg = res needs x01 >= (res + 0.5) / scale > 1: a point outside the box.  On a multi-level grid the same point lies
# beyond res on the finer levels too, where the oracle clamps a neighbour's other coordinates to [0, res] and the kernel
# does not (torch-ngp skips points outside the box altogether); so pg = res is checked on single-level grids, with the
# other two coordinates inside the box
TV_RES_BASES = (16, 100)            # a dense and a hashed single-level grid


@lru_cache(maxsize=None)
def tv_res_points(base):
    rng = np.random.default_rng(25)
    scale, res = G._level_geometry(0, 2.0, base)
    x = np.float32(2.0 * (res + 0.25) / float(scale) - 1.0)
    pts = []
    for a in range(3):
        for _ in range(20):
            p = rng.uniform(-1, 1, 3).astype(np.float32)
            p[a] = x
            pts.append(p)
    pts += list(rng.uniform(-1, 1, (1000, 3)).astype(np.float32))
    return torch.from_numpy(np.stack(pts)).contiguous()


def test_s2_premise():
    for L, pls, base in (GRID_CASES["c3"], (16, 2.0, 16)):
        x = s2_points(L, pls, base)
        assert float(x.abs().max()) <= 1.0
        counts = s2_face_counts(x, L, pls, base)
        assert all(min(c) >= 1 for c in counts), counts                     # faces on every level and axis
        off = G.grid_offsets(num_levels=L, per_level_scale=pls, base_resolution=base)
        x01 = (x + 1.0) / 2.0
        kinds = set()
        for l in range(L):
            scale, res = G._level_geometry(l, pls, base)
            hashed = (res + 1) ** 3 > int(off[l + 1] - off[l])
            px = torch.floor(x01[:, 0] * float(scale) + 0.5).to(torch.int64)
            kinds |= {(hashed, int(p) & 1) for p in px.unique()}
        assert kinds == {(False, 0), (False, 1), (True, 0), (True, 1)}       # dense and hashed levels, even and odd x
        xt = tv_points(L, pls, base)
        x01 = (xt + 1.0) / 2.0
        for l in range(L):
            scale, res = G._level_geometry(l, pls, base)
            pg = torch.floor(x01 * float(scale) + 0.5).to(torch.int64)
            assert bool((pg == 0).any()) and int(pg.max()) <= res - 1, l
    for b in TV_RES_BASES:
        scale, res = G._level_geometry(0, 2.0, b)
        pg = torch.floor((tv_res_points(b) + 1.0) / 2.0 * float(scale) + 0.5).to(torch.int64)
        assert int(pg.max()) == res and int((pg == res).any(1).sum()) == 60 and int((pg > res).sum()) == 0
        assert ((res + 1) ** 3 > 2 ** 19) == (b == 100)


# ---------------------------------------------------------------------------------------------------------------------
# S3: marcher edges
# ---------------------------------------------------------------------------------------------------------------------
def edge_rays():
    """(origins, directions, names): axis-parallel rays with +0 / -0 components, origins inside the box and on face
    planes (some in the plane: (plane - o) * (1/+-0) is NaN there), rays through and tangent to an edge"""
    s = 1.0 / math.sqrt(2.0)
    rays = [("x+0+0", (-2, 0.1, 0.2), (1, 0.0, 0.0)), ("x-0+0", (-2, 0.1, 0.2), (1, -0.0, 0.0)),
            ("-x-0-0", (2, -0.3, 0.4), (-1, -0.0, -0.0)), ("in_z", (0.1, -0.2, 0.3), (0.0, 0.0, 1)),
            ("in_y-0", (0.1, -0.2, 0.3), (-0.0, 1, -0.0)), ("in_diag", (0.05, 0.05, 0.05), (0.48, -0.6, 0.64)),
            ("lo_face_in", (-1, 0.2, 0.3), (1, 0.0, 0.0)), ("hi_face_in", (1, 0.2, 0.3), (-1, 0.0, -0.0)),
            ("lo_face_out", (-1, 0.2, 0.3), (-1, 0.0, 0.0)), ("lo_face_oblique", (-1, 0.2, 0.3), (0.6, 0.0, 0.8)),
            ("in_lo_plane+0", (-1, 0.2, 0.3), (0.0, 1, 0.0)), ("in_lo_plane-0", (-1, 0.2, 0.3), (-0.0, 0.6, 0.8)),
            ("in_hi_plane", (1, 0.2, 0.3), (0.0, 0.0, -1)), ("through_edge", (-2, -2, 0.1), (s, s, 0.0)),
            ("tangent_edge", (-2, 0, 0.1), (s, -s, 0.0)), ("along_edge", (-1, -1, -2), (0.0, 0.0, 1)),
            ("corner_diag", (-2, -2, -2), (1 / math.sqrt(3),) * 3)]
    o = torch.tensor([r[1] for r in rays], dtype=torch.float32)
    d = torch.tensor([r[2] for r in rays], dtype=torch.float32)
    return o, d, [r[0] for r in rays]


# rays lying in a face plane, parallel to it: the slab test yields (plane - o) * (1/+-0) = 0 * inf = NaN on that axis.
# The kernel's fminf / fmaxf drop the NaN (the other bound, +-inf, wins); torch.minimum / .max propagate it and every
# comparison with NaN is false.  Both give no samples; the oracle's rule is the one pinned: a ray of measure zero on the
# box surface does not enter the box.
IN_PLANE = ("in_lo_plane+0", "in_lo_plane-0", "in_hi_plane", "along_edge")
MARCH_CASES = [(1, 0.01, 100.0, False), (7, 0.01, 100.0, True), (48, 2.5, 100.0, False), (100, 0.01, 2.2, True),
               (117, 0.01, 100.0, True)]


@lru_cache(maxsize=None)
def march_inputs(R, strat):
    o, d, names = edge_rays()
    ro, rd = G.get_rays(O.orbit_camera(15, 40, 1.75), 24, 32, 49.1)
    ro = torch.cat([o, ro]); rd = torch.cat([d, rd])
    g = torch.Generator().manual_seed(R)
    binary = torch.ones(R, R, R, dtype=torch.bool) if R == 1 else torch.rand(R, R, R, generator=g) < 0.5
    toff = (torch.rand(ro.shape[0], generator=g) * 5e-3) if strat else None
    return ro.contiguous(), rd.contiguous(), binary, toff, names


def test_s3_premise():
    o, d, names = edge_rays()
    inv = 1.0 / d
    assert bool(torch.isinf(inv).any()) and bool((torch.signbit(d) & (d == 0)).any())
    ri, ts, te = G.march(o, d, torch.ones(8, 8, 8, dtype=torch.bool), AABB, 0.01, 100.0, 5e-3)
    cnt = torch.bincount(ri, minlength=len(names))
    t0 = (AABB[:3][None] - o) * inv
    nan_rows = torch.isnan(t0).any(1) | torch.isnan((AABB[3:][None] - o) * inv).any(1)
    assert {names[i] for i in torch.nonzero(nan_rows)[:, 0].tolist()} >= set(IN_PLANE)
    for n in IN_PLANE:
        assert int(cnt[names.index(n)]) == 0, n
    for n in ("in_z", "lo_face_in", "hi_face_in", "through_edge", "x-0+0"):
        assert int(cnt[names.index(n)]) > 100, n
    assert int(cnt[names.index("tangent_edge")]) == 0 and int(cnt[names.index("lo_face_out")]) == 0
    # shared memory: R = 117 fits 200 KiB, 118 does not
    assert (117 ** 3 + 31) // 32 * 4 <= 200 * 1024 < (118 ** 3 + 31) // 32 * 4
    # the midpoint rule: with dt = 0.25 from t = 0, the far plane 0.625 is the midpoint of interval 2 exactly; "<" keeps
    # intervals 0 and 1 only
    ri, _, _ = G.march(torch.zeros(1, 3), torch.tensor([[1.0, 0.0, 0.0]]), torch.ones(4, 4, 4, dtype=torch.bool), AABB, 0.0, 0.625, 0.25)
    assert ri.numel() == 2
    # near plane beyond the exit: camera rays leave the box before t = 2.5 or after it
    ro, rd, _, _, _ = march_inputs(48, False)
    tmin, tmax = G.ray_aabb(ro, rd, AABB)
    ok = tmax > tmin
    assert bool((tmax[ok] < 2.5).any()) and bool((tmax[ok] > 2.5).any())


# ---------------------------------------------------------------------------------------------------------------------
# S4: packed rendering
# ---------------------------------------------------------------------------------------------------------------------
S4_RAYS = [(0, "rand"), (1, "rand"), (2, "rand"), (0, "rand"), (255, "zero_runs"), (256, "small"), (257, "sat"), (0, "rand"),
           (1000, "subnormal"), (1500, "rand"), (300, "small"), (64, "sat"), (0, "rand")]


@lru_cache(maxsize=None)
def s4_inputs():
    g = torch.Generator().manual_seed(41)
    ris, tss, tes, sigs = [], [], [], []
    for r, (n, kind) in enumerate(S4_RAYS):
        if n == 0:
            continue
        dt = 5e-3 * (1 + 0.2 * torch.rand(n, generator=g))
        ts = 0.5 + torch.cumsum(dt, 0) - dt
        te = ts + dt
        dtf = (te - ts)
        if kind == "rand":
            x = torch.rand(n, generator=g) * 0.25
        elif kind == "zero_runs":
            x = torch.rand(n, generator=g) * 0.05
            x[10:60] = 0; x[100:101] = 0; x[200:255] = 0
        elif kind == "small":
            x = torch.exp(torch.empty(n).uniform_(math.log(1e-8), math.log(1e-3), generator=g))
        elif kind == "sat":
            x = torch.rand(n, generator=g) * 0.1
            x[n // 3] = 95.0; x[n // 3 + 5] = 200.0
        else:
            x = 0.0875 + torch.rand(n, generator=g) * 0.0125
        ris.append(torch.full((n,), r, dtype=torch.int64)); tss.append(ts); tes.append(te)
        sigs.append((x / dtf).float())
    n_rays = len(S4_RAYS)
    ri = torch.cat(ris); ts = torch.cat(tss).float(); te = torch.cat(tes).float(); sig = torch.cat(sigs)
    S = ri.numel()
    vals = {C_: torch.rand(S, C_, generator=g) for C_ in (1, 2, 3, 4)}
    up = {"gw": torch.rand(S, generator=g) * 2 - 1, "gt": (torch.rand(S, generator=g) * 2 - 1) * 0.1,
          "ga": torch.rand(S, generator=g) * 2 - 1}
    return ri, ts, te, sig, n_rays, vals, up


def weights_ref64(ts, te, sig, ri, n_rays, gw=None, gt=None, ga=None):
    """float64 recurrence on the fp32 inputs, plus the first-order fp32 error bounds of the kernels (module docstring)
    and nerfacc's fp32 formula with a correctly rounded exp.  Returns a dict of float64 numpy arrays."""
    ts64, te64, s64 = ts.double().numpy(), te.double().numpy(), sig.double().numpy()
    dt = te64 - ts64
    x = s64 * dt
    a = -np.expm1(-x)
    c = np.exp(-x)
    ea = 2 * U * x * c + 2 * U * a
    ec = ea + U * c
    x32 = (sig * (te - ts)).numpy().astype(np.float32)
    a_nerfacc = (np.float32(1.0) - np.exp(-x32.astype(np.float64)).astype(np.float32)).astype(np.float64)
    b_nerfacc = U / 2 * c + U / 2 * a + U * x * c
    S = x.size
    T = np.zeros(S); E = np.zeros(S); w = np.zeros(S); Ew = np.zeros(S)
    start, cnt = (v.numpy() for v in G.packed_ranges(ri, n_rays))
    z = np.zeros(S)
    gw = z if gw is None else gw.double().numpy(); gt = z if gt is None else gt.double().numpy()
    ga = z if ga is None else ga.double().numpy()
    dsig = np.zeros(S); Ed = np.zeros(S)
    for s, n in zip(start.tolist(), cnt.tolist()):
        Ti, Ei = 1.0, 0.0
        for i in range(s, s + n):
            T[i], E[i] = Ti, Ei
            w[i] = Ti * a[i]
            Ew[i] = Ei * a[i] + Ti * ea[i] + Ei * ea[i] + U * w[i] + TINY
            Tn = Ti * c[i]
            Ei = Ei * (c[i] + ec[i]) + Ti * ec[i] + U * Tn + TINY
            Ti = Tn
        Gv, EG, MG = 0.0, 0.0, 0.0
        for i in range(s + n - 1, s - 1, -1):
            dal = gw[i] * T[i] + ga[i] - Gv * T[i]
            D = abs(gw[i]) * T[i] + abs(ga[i]) + abs(Gv) * T[i]
            Edal = (abs(gw[i]) + abs(Gv)) * E[i] + EG * (T[i] + E[i]) + 4 * U * D
            dsig[i] = dal * c[i] * dt[i]
            Ed[i] = dt[i] * (Edal * c[i] + (abs(dal) + Edal) * ec[i] + 4 * U * (abs(dal) + Edal) * c[i]) + TINY
            Gn = gt[i] + gw[i] * a[i] + Gv * c[i]
            MG = abs(gt[i]) + abs(gw[i]) * a[i] + abs(Gv) * c[i]
            EG = abs(gw[i]) * ea[i] + EG * (c[i] + ec[i]) + abs(Gv) * ec[i] + 4 * U * MG
            Gv = Gn
    return {"x": x, "a": a, "ea": ea, "T": T, "ET": E, "w": w, "Ew": Ew, "a_nerfacc": a_nerfacc, "b_nerfacc": b_nerfacc,
            "dsig": dsig, "Edsig": Ed}


def test_s4_premise():
    ri, ts, te, sig, n_rays, _, _ = s4_inputs()
    cnt = torch.bincount(ri, minlength=n_rays)
    assert int(cnt[0]) == 0 and int(cnt[-1]) == 0 and bool((cnt[1:-1] == 0).any())
    for n in (1, 2, 255, 256, 257):
        assert bool((cnt == n).any()), n
    assert int(cnt.max()) >= 1000
    ref = weights_ref64(ts, te, sig, ri, n_rays)
    x = ref["x"]
    assert (x >= 90).sum() >= 2 and (sig == 0).sum() >= 100
    assert ((x >= 1e-8) & (x <= 1e-3)).sum() >= 500
    T = ref["T"]
    assert ((T > 0) & (T < 2.0 ** -126)).sum() >= 10                 # fp64 transmittance in fp32's subnormal range
    assert ((T > 2.0 ** -126)).sum() > 0
    # the fp32 kernels see the same: the recurrence in fp32 reaches subnormals too
    a32 = (1.0 - torch.exp(-(sig * (te - ts)).double())).float()
    sub = ri == 8
    T32 = torch.cumprod(torch.cat([torch.ones(1), 1 - a32[sub][:-1]]), 0)
    assert bool(((T32 > 0) & (T32 < 2.0 ** -126)).any())


# ---------------------------------------------------------------------------------------------------------------------
# S5: fused MLP
# ---------------------------------------------------------------------------------------------------------------------
MLP_DIMS = [(di, do) for di in (24, 32) for do in (1, 2, 3, 4)]
MLP_N = (1, 127, 128, 129, 396 * 128 + 1, 20_000_000)


def mlp_neff(N, din, dout):
    tiles = (N + 127) // 128
    grid = min(tiles, 132 * 3)
    return 128 + (tiles + grid - 1) // grid + grid + dout + din


def test_s5_premise():
    # 396 CTAs: 396 * 128 + 1 rows give CTA 0 a second tile of one row; 2e7 rows give each CTA ~395 tiles
    assert (396 * 128 + 1 + 127) // 128 == 397
    assert mlp_neff(20_000_000, 32, 4) < 1000 and mlp_neff(1, 24, 1) == 128 + 1 + 1 + 1 + 24
    from gs_b200 import _lib  # noqa: F401  (the support table comes from the library)
    for di, do in MLP_DIMS:
        assert _lib.lib.ngp_b200_mlp2_supported(di, 32, do)
    assert not _lib.lib.ngp_b200_mlp2_supported(16, 32, 1) and not _lib.lib.ngp_b200_mlp2_supported(32, 32, 5)


# ---------------------------------------------------------------------------------------------------------------------
# GPU tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["default", "v4off"])
def test_s1_ray_ordered_grid_backward(dev, route):
    """default: d_emb 16-byte aligned, the .v4 reds; v4off: d_emb misaligned, which selects the scalar-red kernels"""
    x, g = s1_samples()
    xg, gg = x.to(dev), g.to(dev)
    for name, (L, pls, base) in GRID_CASES.items():
        gl = gg[:, :2 * L].contiguous()
        ref = grid_ref64(xg, L, pls, base, g=gl)
        check_grid_bwd(f"S1 {route} {name}", _grid_bwd_abi(xg, gl, L, pls, base, misalign=route == "v4off"), ref)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["c3", "pls2"])
def test_s2_grid_geometry_edges(dev, case):
    from kiui.gridencoder import GridEncoder
    L, pls, base = GRID_CASES["c3"] if case == "c3" else (16, 2.0, 16)
    x = s2_points(L, pls, base)
    torch.manual_seed(23)
    enc = GridEncoder(num_levels=L, per_level_scale=pls, base_resolution=base).to(dev)
    enc.embeddings.data.uniform_(-1, 1)
    emb = enc.embeddings.detach().clone()
    gout = torch.rand(x.shape[0], 2 * L, generator=torch.Generator().manual_seed(24)) * 2 - 1
    ref = grid_ref64(x.to(dev), L, pls, base, g=gout.to(dev), emb=emb)
    out = enc(x.to(dev))
    err = (out.detach().double() - ref["feat"]).abs()
    ratio, rel = report(f"S2 {case} features", err.cpu().numpy(), (K_ELEM * gam(13) * ref["feat_abs"]).cpu().numpy(),
                        ref["feat"].cpu().numpy())
    assert ratio <= 1.0 and rel <= GRID_REL
    (out * gout.to(dev)).sum().backward()
    check_grid_bwd(f"S2 {case} backward", enc.embeddings.grad, ref)
    # d_emb 8 bytes past a 16-byte boundary: the .v4 reds turn themselves off, the result stays within the bars
    check_grid_bwd(f"S2 {case} backward, d_emb misaligned", _grid_bwd_abi(x.to(dev), gout.to(dev), L, pls, base, True), ref)
    check_tv(f"S2 {case} TV", enc, tv_points(L, pls, base), L, pls, base)


@pytest.mark.gpu
@pytest.mark.parametrize("base", TV_RES_BASES)
def test_s2_tv_gradient_at_pg_res(dev, base):
    from kiui.gridencoder import GridEncoder
    torch.manual_seed(26)
    enc = GridEncoder(num_levels=1, base_resolution=base).to(dev)
    enc.embeddings.data.uniform_(-1, 1)
    check_tv(f"S2 TV pg = res, base {base}", enc, tv_res_points(base), 1, 2.0, base)


def check_tv(name, enc, xt, L, pls, base, w=1e-3):
    emb = enc.embeddings.detach().clone()
    enc.embeddings.grad = torch.zeros_like(enc.embeddings)
    enc.grad_total_variation(w, inputs=xt.to(emb.device))
    off = G.grid_offsets(num_levels=L, per_level_scale=pls, base_resolution=base)
    ref_tv = G.grad_total_variation(xt, emb.cpu().double(), off, w, num_levels=L, per_level_scale=pls, base_resolution=base)
    # per entry: n contributions (the points whose base corner it is), each |weight * (sum of <= 6 signs)| <= 6 w
    n_e = torch.zeros(emb.shape[0], dtype=torch.float64)
    for l in range(L):
        idx, _, _ = G.grid_corner_indices((xt + 1.0) / 2.0, l, off, pls, base)
        n_e.index_add_(0, idx[:, 0] + int(off[l]), torch.ones(xt.shape[0], dtype=torch.float64))
    err = (enc.embeddings.grad.cpu().double() - ref_tv).abs()
    bar = (K_ELEM * torch.from_numpy(gam(n_e.numpy() + 2)) * 6 * w * n_e + TINY)[:, None].expand(-1, 2)
    ratio, rel = report(name, err.numpy(), bar.numpy(), ref_tv.numpy())
    assert ratio <= 1.0 and rel <= GRID_REL


@pytest.mark.gpu
@pytest.mark.parametrize("R,near,far,strat", MARCH_CASES)
def test_s3_marcher_edges_bit_exact(dev, R, near, far, strat):
    from gs_b200 import ngp
    ro, rd, binary, toff, names = march_inputs(R, strat)
    ri_r, ts_r, te_r = G.march(ro, rd, binary, AABB, near, far, 5e-3, toff)
    ri, ts, te = ngp.march_rays(ro.to(dev), rd.to(dev), binary.to(dev), AABB.to(dev), near, far, 5e-3,
                                None if toff is None else toff.to(dev))
    assert torch.equal(ri.cpu(), ri_r) and torch.equal(ts.cpu(), ts_r) and torch.equal(te.cpu(), te_r)
    cnt = torch.bincount(ri.cpu(), minlength=ro.shape[0])
    for n in IN_PLANE:
        assert int(cnt[names.index(n)]) == 0, n
    print(f"S3 R={R}: {ri.numel()} samples, bit-exact")


@pytest.mark.gpu
def test_s3_marcher_midpoint_on_far_plane(dev):
    from gs_b200 import ngp
    ri, ts, te = ngp.march_rays(torch.zeros(1, 3, device=dev), torch.tensor([[1.0, 0.0, 0.0]], device=dev),
                                torch.ones(4, 4, 4, dtype=torch.bool, device=dev), AABB.to(dev), 0.0, 0.625, 0.25)
    assert ri.numel() == 2 and ts.cpu().tolist() == [0.0, 0.25] and te.cpu().tolist() == [0.25, 0.5]


@pytest.mark.gpu
@pytest.mark.parametrize("R", [118, 128])
def test_s3_marcher_refuses_grids_beyond_shared_memory(dev, R):
    from gs_b200 import ngp
    ro, rd = G.get_rays(O.orbit_camera(15, 40, 1.75), 4, 4, 49.1)
    with pytest.raises(RuntimeError, match="shared memory"):
        ngp.march_rays(ro.to(dev), rd.to(dev), torch.ones(R, R, R, dtype=torch.bool, device=dev), AABB.to(dev), 0.01, 100.0, 5e-3)


@pytest.mark.gpu
def test_s3_full_frame_sample_list(dev):
    """1920 x 1080 config-3 rays, sphere r = 0.5 on 64^3, stratified: the whole list against the oracle's fp32 ops run
    on the device (the same elementwise IEEE operations), and 4096 sampled rays, the longest among them, against the
    oracle on the CPU"""
    from gs_b200 import ngp
    ro, rd = c3_rays()
    n = ro.shape[0]
    binary = _binary_ball(64, 0.5)
    toff = torch.rand(n, generator=torch.Generator().manual_seed(33)) * 5e-3
    ri, ts, te = ngp.march_rays(ro.to(dev), rd.to(dev), binary.to(dev), AABB.to(dev), 0.01, 100.0, 5e-3, toff.to(dev))
    cnt = torch.bincount(ri, minlength=n)
    off = torch.cumsum(cnt, 0) - cnt
    rog, rdg, bg, tg, ag = ro.to(dev), rd.to(dev), binary.to(dev), toff.to(dev), AABB.to(dev)
    step = 1 << 15
    for a in range(0, n, step):
        b = min(n, a + step)
        r_ri, r_ts, r_te = G.march(rog[a:b], rdg[a:b], bg, ag, 0.01, 100.0, 5e-3, tg[a:b])
        assert torch.equal(torch.bincount(r_ri, minlength=b - a), cnt[a:b]), a
        s0, s1 = int(off[a]), int(off[b - 1] + cnt[b - 1])
        assert torch.equal(r_ri + a, ri[s0:s1]) and torch.equal(r_ts, ts[s0:s1]) and torch.equal(r_te, te[s0:s1]), a
    longest = int(torch.argmax(cnt))
    pick = torch.randperm(n, generator=torch.Generator().manual_seed(34))[:4095]
    pick = torch.unique(torch.cat([pick, torch.tensor([longest])]))
    c_ri, c_ts, c_te = G.march(ro[pick], rd[pick], binary, AABB, 0.01, 100.0, 5e-3, toff[pick])
    cc = cnt.cpu()
    sel = torch.cat([torch.arange(int(off[r]), int(off[r]) + int(cc[r])) for r in pick.tolist()])
    assert torch.equal(pick[c_ri], ri.cpu()[sel]) and torch.equal(c_ts, ts.cpu()[sel]) and torch.equal(c_te, te.cpu()[sel])
    print(f"S3 1080p: {ri.numel()} samples, longest ray {int(cc[longest])}, bit-exact")


def _weights_fwd(ts, te, sig, ri, n_rays, dev):
    import nerfacc
    return nerfacc.render_weight_from_density(ts.to(dev), te.to(dev), sig.to(dev), ray_indices=ri.to(dev), n_rays=n_rays)


@pytest.mark.gpu
def test_s4_weights_forward(dev):
    ri, ts, te, sig, n_rays, _, _ = s4_inputs()
    w, T, a = (v.cpu().double().numpy() for v in _weights_fwd(ts, te, sig, ri, n_rays, dev))
    ref = weights_ref64(ts, te, sig, ri, n_rays)
    for name, got, key, ekey in (("alpha", a, "a", "ea"), ("T", T, "T", "ET"), ("w", w, "w", "Ew")):
        ratio, rel = report(f"S4 {name}", np.abs(got - ref[key]), K_ELEM * ref[ekey], ref[key])
        assert ratio <= 1.0 and rel <= W_REL, (name, ratio, rel)
    # against nerfacc's fp32 formula with a correctly rounded exp
    e_ref = np.abs(ref["a_nerfacc"] - ref["a"])
    ratio, _ = report("S4 alpha vs nerfacc's formula bound", np.abs(a - ref["a"]), 2 * ref["b_nerfacc"] + TINY)
    small = (ref["x"] >= 1e-8) & (ref["x"] <= 1e-3)
    print(f"S4 alpha at sigma*dt in [1e-8, 1e-3]: kernel max rel {float((np.abs(a - ref['a']) / ref['a'])[small].max()):.3g}, "
          f"nerfacc formula max rel {float((e_ref / ref['a'])[small].max()):.3g}")
    assert ratio <= 1.0
    sat = ref["x"] >= 90
    assert (a[sat] == 1.0).all()
    after = np.zeros_like(sat)
    for r in np.unique(ri.numpy()[sat]):
        idx = np.flatnonzero((ri.numpy() == r))
        first = idx[np.flatnonzero(sat[idx])[0]]
        after[first + 1:idx[-1] + 1] = True
    assert (T[after] == 0).all() and (w[after] == 0).all()


PATTERNS = [(a, b, c) for a in (0, 1) for b in (0, 1) for c in (0, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", PATTERNS, ids=["".join(n for n, f in zip(("w", "t", "a"), p) if f) or "none" for p in PATTERNS])
def test_s4_weights_backward_every_none_pattern(dev, pattern):
    from gs_b200 import _lib, ngp
    ri, ts, te, sig, n_rays, _, up = s4_inputs()
    ups = [up[k] if f else None for k, f in zip(("gw", "gt", "ga"), pattern)]
    ref = weights_ref64(ts, te, sig, ri, n_rays, *ups)
    tsg, teg, sg, rig = ts.to(dev), te.to(dev), sig.to(dev), ri.to(dev)
    rng = ngp._ranges(rig, n_rays)
    w, T, a = ngp._Weights.apply(tsg, teg, sg, rng, n_rays)
    d = torch.full_like(sg, float("nan"))
    P = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    ug = [None if u is None else u.to(dev).contiguous() for u in ups]
    _lib.check(_lib.lib.ngp_b200_weights_bwd(P(tsg), P(teg), P(sg), P(rng), n_rays, P(T), P(a), P(ug[0]), P(ug[1]), P(ug[2]), P(d),
                                             C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    got = d.cpu().double().numpy()
    if not any(pattern):
        assert (got == 0).all()
        return
    ratio, rel = report(f"S4 dsigma {pattern}", np.abs(got - ref["dsig"]), K_ELEM * ref["Edsig"], ref["dsig"])
    assert ratio <= 1.0 and rel <= DSIG_REL


@pytest.mark.gpu
@pytest.mark.parametrize("Cv", [None, 1, 2, 3, 4])
def test_s4_accumulate(dev, Cv):
    import nerfacc
    ri, ts, te, sig, n_rays, vals, _ = s4_inputs()
    w = _weights_fwd(ts, te, sig, ri, n_rays, dev)[0].detach().cpu()
    v = None if Cv is None else vals[Cv]
    wg = w.to(dev).requires_grad_(True)
    vg = None if v is None else v.to(dev).requires_grad_(True)
    out = nerfacc.accumulate_along_rays(wg, values=vg, ray_indices=ri.to(dev), n_rays=n_rays)
    Cc = 1 if v is None else Cv
    src = w.double()[:, None] * (torch.ones(w.numel(), 1, dtype=torch.float64) if v is None else v.double())
    ref = torch.zeros(n_rays, Cc, dtype=torch.float64).index_add(0, ri, src)
    asum = torch.zeros(n_rays, Cc, dtype=torch.float64).index_add(0, ri, src.abs())
    cnt = torch.bincount(ri, minlength=n_rays).double()[:, None]
    ratio, rel = report(f"S4 accumulate C={Cv}", (out.detach().cpu().double() - ref).abs().numpy(),
                        (K_ELEM * torch.from_numpy(gam((cnt + 1).numpy())) * asum).numpy(), ref.numpy())
    assert ratio <= 1.0 and rel <= W_REL
    gout = torch.rand(n_rays, Cc, generator=torch.Generator().manual_seed(45)) * 2 - 1
    out.backward(gout.to(dev))
    g_i = gout.double()[ri]
    vv = torch.ones(w.numel(), 1, dtype=torch.float64) if v is None else v.double()
    dw = (g_i * vv).sum(1)
    ratio, rel = report(f"S4 accumulate dw C={Cv}", (wg.grad.cpu().double() - dw).abs().numpy(),
                        (K_ELEM * gam(Cc) * (g_i * vv).abs().sum(1)).numpy() + TINY, dw.numpy())
    assert ratio <= 1.0 and rel <= W_REL
    if v is not None:
        dv = w.double()[:, None] * g_i
        ratio, rel = report(f"S4 accumulate dv C={Cv}", (vg.grad.cpu().double() - dv).abs().numpy(),
                            (K_ELEM * U * dv.abs()).numpy() + TINY, dv.numpy())
        assert ratio <= 1.0 and rel <= W_REL


@pytest.mark.gpu
def test_s4_accumulate_refuses_five_channels(dev):
    import nerfacc
    ri, ts, te, sig, n_rays, _, _ = s4_inputs()
    w = torch.rand(ri.numel(), device=dev)
    with pytest.raises(RuntimeError, match="channels"):
        nerfacc.accumulate_along_rays(w, values=torch.rand(ri.numel(), 5, device=dev), ray_indices=ri.to(dev), n_rays=n_rays)


def _mlp_ref_pass(x, W1, W2, gy, chunk=1 << 21):
    """float64 reference in row chunks: y, dL/dx (errors and bars computed against the given fp32 outputs lazily) and the
    weight gradients with their |.|-sums"""
    out = {"gW1": 0, "gW2": 0, "aW1": 0, "aW2": 0, "aW2h": 0}
    W1d, W2d = W1.double(), W2.double()
    for a in range(0, x.shape[0], chunk):
        xd = x[a:a + chunk].double(); gd = gy[a:a + chunk].double()
        h = xd @ W1d.T
        act = h.clamp_min(0)
        gh = (gd @ W2d) * (h > 0)
        gha = (gd.abs() @ W2d.abs()) * (h > 0)
        out["gW1"] = out["gW1"] + gh.T @ xd
        out["aW1"] = out["aW1"] + gha.T @ xd.abs()
        out["gW2"] = out["gW2"] + gd.T @ act
        out["aW2"] = out["aW2"] + gd.abs().T @ act
        out["aW2h"] = out["aW2h"] + gd.abs().T @ (xd.abs() @ W1d.abs().T)
        yield a, xd, gd, h, act, gh, gha, out


@pytest.mark.gpu
@pytest.mark.parametrize("din,dout", MLP_DIMS)
def test_s5_fused_mlp_at_scale(dev, din, dout):
    from kiui.nn import MLP
    torch.manual_seed(50 + din + dout)
    m = MLP(din, dout, 32, 2, bias=False).to(dev)
    W1, W2 = m.net[0].weight.detach(), m.net[1].weight.detach()
    gen = torch.Generator(device=dev)
    for N in MLP_N:
        gen.manual_seed(N + din)
        x = torch.randn(N, din, device=dev, generator=gen)
        gy = torch.randn(N, dout, device=dev, generator=gen)
        excl = torch.zeros(N, dtype=torch.bool, device=dev)
        for a in range(0, N, 1 << 21):
            xd = x[a:a + (1 << 21)].double()
            h = xd @ W1.double().T
            tau = 4 * float(gam(din)) * (xd.abs() @ W1.double().abs().T)
            excl[a:a + (1 << 21)] = (h.abs() <= tau).any(1)
        gy[excl] = 0
        xr = x.clone().requires_grad_(True)
        y = m(xr)
        gx, gW1, gW2 = torch.autograd.grad(y, [xr, m.net[0].weight, m.net[1].weight], gy)
        # torch's fp32 GEMMs on the same rows (the baseline)
        xt = x.clone().requires_grad_(True)
        yt = torch.relu(xt @ m.net[0].weight.T) @ m.net[1].weight.T
        tgx, tgW1, tgW2 = torch.autograd.grad(yt, [xt, m.net[0].weight, m.net[1].weight], gy)
        del xt, yt
        neff = mlp_neff(N, din, dout)
        worst = {"y": 0.0, "gx": 0.0}
        num = {"y": 0.0, "gx": 0.0, "ty": 0.0, "tgx": 0.0}
        den = {"y": 0.0, "gx": 0.0}
        for a, xd, gd, h, act, gh, gha, ref in _mlp_ref_pass(x, W1, W2, gy):
            b = a + xd.shape[0]
            yref = act @ W2.double().T
            ybar = K_ELEM * float(gam(din + 32 + 2)) * ((xd.abs() @ W1.double().abs().T) @ W2.double().abs().T)
            ey = (y[a:b].double() - yref).abs()
            worst["y"] = max(worst["y"], float((ey / ybar.clamp_min(1e-300)).max()))
            num["y"] += float((ey ** 2).sum()); den["y"] += float((yref ** 2).sum())
            num["ty"] += float(((yt_ := torch.relu(x[a:b] @ W1.T) @ W2.T).double() - yref).pow(2).sum())
            gxref = gh @ W1.double()
            gxbar = K_ELEM * float(gam(32 + dout + 2)) * (gha @ W1.double().abs()) + TINY
            egx = (gx[a:b].double() - gxref).abs()
            worst["gx"] = max(worst["gx"], float((egx / gxbar).max()))
            num["gx"] += float((egx ** 2).sum()); den["gx"] += float((gxref ** 2).sum())
            num["tgx"] += float((tgx[a:b].double() - gxref).pow(2).sum())
            del yt_
        rels = {k: math.sqrt(num[k] / max(den[k], 1e-300)) for k in ("y", "gx")}
        trel = {k: math.sqrt(num["t" + k] / max(den[k], 1e-300)) for k in ("y", "gx")}
        bar1 = K_ELEM * float(gam(neff)) * ref["aW1"] + TINY
        bar2 = K_ELEM * (float(gam(neff)) * ref["aW2"] + float(gam(din + 2)) * ref["aW2h"]) + TINY
        r1 = float(((gW1.double() - ref["gW1"]).abs() / bar1).max()); r2 = float(((gW2.double() - ref["gW2"]).abs() / bar2).max())
        rel1 = float((gW1.double() - ref["gW1"]).norm() / ref["gW1"].norm()); rel2 = float((gW2.double() - ref["gW2"]).norm() / ref["gW2"].norm())
        t1 = float((tgW1.double() - ref["gW1"]).norm() / ref["gW1"].norm()); t2 = float((tgW2.double() - ref["gW2"]).norm() / ref["gW2"].norm())
        print(f"S5 {din}-32-{dout} N={N}: excluded rows {int(excl.sum())}; err/bar y {worst['y']:.3g} gx {worst['gx']:.3g} "
              f"gW1 {r1:.3g} gW2 {r2:.3g}; norm-rel y {rels['y']:.3g} (torch {trel['y']:.3g}) gx {rels['gx']:.3g} "
              f"(torch {trel['gx']:.3g}) gW1 {rel1:.3g} (torch {t1:.3g}) gW2 {rel2:.3g} (torch {t2:.3g})")
        assert max(worst.values()) <= 1.0 and r1 <= 1.0 and r2 <= 1.0, (N, worst, r1, r2)
        assert rels["y"] <= MLP_REL / 5 and rels["gx"] <= MLP_REL / 5 and rel1 <= MLP_REL and rel2 <= MLP_REL, (N, rels, rel1, rel2)
        del x, gy, xr, y, gx, tgx, excl
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# S6: one config-3 frame
# ---------------------------------------------------------------------------------------------------------------------
def _enc64(x, emb64, L, pls, base):
    """differentiable float64 encode (oracle indices and fractions, weights in float64)"""
    off = G.grid_offsets(num_levels=L, per_level_scale=pls, base_resolution=base)
    x01 = (x.float() + 1.0) / 2.0
    outs = []
    for l in range(L):
        idx, _, frac = G.grid_corner_indices(x01, l, off, pls, base)
        f = frac.double()
        w = torch.stack([math.prod((f[:, d] if (c >> d) & 1 else 1.0 - f[:, d]) for d in range(3)) for c in range(8)], 1)
        outs.append((emb64[idx + int(off[l])] * w[:, :, None]).sum(1))
    return torch.cat(outs, 1)


@pytest.mark.gpu
def test_s6_config3_frame(dev):
    import nerfacc
    from kiui.gridencoder import GridEncoder
    from kiui.nn import MLP, trunc_exp
    H, W, L = 1080, 1920, 16
    torch.manual_seed(60)
    enc_d = GridEncoder(num_levels=L, desired_resolution=512).to(dev); enc_c = GridEncoder(num_levels=L, desired_resolution=512).to(dev)
    enc_d.embeddings.data.uniform_(-0.1, 0.1); enc_c.embeddings.data.uniform_(-0.1, 0.1)
    mlp_d, mlp_c = MLP(2 * L, 1, 32, 2, bias=False).to(dev), MLP(2 * L, 3, 32, 2, bias=False).to(dev)
    pls = float(enc_d.per_level_scale)
    assert pls == PLS3
    est = nerfacc.OccGridEstimator(roi_aabb=AABB.to(dev), resolution=64, levels=1).to(dev)
    est.binaries = _binary_ball(64, 0.5).to(dev)[None]; est.occs = est.binaries.flatten().float()
    ro, rd = (t.to(dev) for t in c3_rays())

    def sigma_fn(t0, t1, ri):
        return trunc_exp(mlp_d(enc_d(ro[ri] + rd[ri] * (t0 + t1)[:, None] / 2.0))).squeeze(-1)
    from gs_b200 import ngp
    ngp.set_rng(torch.Generator().manual_seed(61))
    try:
        with torch.no_grad():
            ri, t0, t1 = est.sampling(ro, rd, sigma_fn=sigma_fn, near_plane=0.01, far_plane=100, render_step_size=5e-3,
                                      stratified=True, cone_angle=0)
    finally:
        ngp.set_rng(None)
    n = H * W
    cnt = torch.bincount(ri, minlength=n)
    pick = torch.randperm(n, generator=torch.Generator().manual_seed(62))[:4095].to(dev)
    pick = torch.unique(torch.cat([pick, torch.argmax(cnt)[None]]))
    insub = torch.zeros(n, dtype=torch.bool, device=dev); insub[pick] = True
    smask = insub[ri]
    p = ro[ri] + rd[ri] * (t0 + t1)[:, None] / 2.0
    # fp64 chain on the subset's samples
    ps, ris = p[smask].contiguous(), ri[smask]
    e64 = {k: e.embeddings.detach().double().requires_grad_(True) for k, e in (("d", enc_d), ("c", enc_c))}
    W64 = {k: [l.weight.detach().double().requires_grad_(True) for l in m.net] for k, m in (("d", mlp_d), ("c", mlp_c))}
    fd = _enc64(ps, e64["d"], L, pls, 16); fc = _enc64(ps, e64["c"], L, pls, 16)
    hd = fd @ W64["d"][0].T; hc = fc @ W64["c"][0].T
    # rays with a sample on a ReLU edge (module docstring) get no upstream gradient
    edge = ((hd.abs() <= 64 * U * (fd.abs() @ W64["d"][0].abs().T)).any(1) |
            (hc.abs() <= 64 * U * (fc.abs() @ W64["c"][0].abs().T)).any(1)).detach()
    bad = torch.zeros(n, dtype=torch.bool, device=dev); bad[ris[edge]] = True
    target = torch.zeros(n, 3, device=dev)
    keep = insub & ~bad
    target[keep] = torch.rand(int(keep.sum()), 3, generator=torch.Generator().manual_seed(63)).to(dev)
    # GPU: the whole frame
    sig = trunc_exp(mlp_d(enc_d(p))).squeeze(-1); rgb = torch.sigmoid(mlp_c(enc_c(p)))
    w, _, _ = nerfacc.render_weight_from_density(t0, t1, sig, ray_indices=ri, n_rays=n)
    col = nerfacc.accumulate_along_rays(w, values=rgb, ray_indices=ri, n_rays=n)
    alp = nerfacc.accumulate_along_rays(w, values=None, ray_indices=ri, n_rays=n)
    img = col + (1 - alp)
    (img * target).sum().backward()
    # fp64: the subset alone
    sig64 = G.trunc_exp(torch.relu(hd) @ W64["d"][1].T).squeeze(-1)
    rgb64 = torch.sigmoid(torch.relu(hc) @ W64["c"][1].T)
    pos = torch.searchsorted(pick, ris)                                 # row of each subset sample
    start = torch.zeros(pick.numel(), dtype=torch.int64, device=dev)
    cs = cnt[pick]
    start[1:] = torch.cumsum(cs, 0)[:-1]
    col_i = torch.arange(ris.numel(), device=dev) - start[pos]
    M = int(cs.max())
    x64 = sig64 * (t1[smask] - t0[smask]).double()
    A = torch.zeros(pick.numel(), M, dtype=torch.float64, device=dev).index_put((pos, col_i), -torch.expm1(-x64))
    Tp = torch.cumprod(torch.cat([torch.ones(pick.numel(), 1, dtype=torch.float64, device=dev), 1 - A[:, :-1]], 1), 1)
    W_ = (Tp * A)[pos, col_i]
    col64 = torch.zeros(pick.numel(), 3, dtype=torch.float64, device=dev).index_add(0, pos, W_[:, None] * rgb64)
    alp64 = torch.zeros(pick.numel(), dtype=torch.float64, device=dev).index_add(0, pos, W_)
    img64 = col64 + (1 - alp64)[:, None]
    (img64 * target[pick].double()).sum().backward()
    e_img = (img.detach()[pick].double() - img64.detach()).abs()
    e_alp = (alp.detach()[pick, 0].double() - alp64.detach()).abs()
    r_img, rel_img = report("S6 image", e_img.cpu().numpy(), np.full(e_img.shape, C6_IMG), img64.detach().cpu().numpy())
    r_alp, rel_alp = report("S6 alpha", e_alp.cpu().numpy(), np.full(e_alp.shape, C6_IMG), alp64.detach().cpu().numpy())
    print(f"S6: {ri.numel()} samples, {pick.numel()} rays compared, {int((insub & bad).sum())} excluded (ReLU edge), "
          f"longest ray {int(cnt.max())}")
    assert r_img <= 1.0 and r_alp <= 1.0 and rel_img <= C6_IMG and rel_alp <= C6_IMG
    pairs = [("emb_d", enc_d.embeddings.grad, e64["d"].grad), ("emb_c", enc_c.embeddings.grad, e64["c"].grad)]
    pairs += [(f"mlp_{k}{i}", m.net[i].weight.grad, W64[k][i].grad) for k, m in (("d", mlp_d), ("c", mlp_c)) for i in (0, 1)]
    for name, got, ref in pairs:
        err = (got.double() - ref).abs()
        ratio, rel = report(f"S6 grad {name}", err.cpu().numpy(), np.full(err.shape, C6_ELEM * float(ref.abs().max())),
                            ref.cpu().numpy())
        assert ratio <= 1.0 and rel <= C6_REL, (name, ratio, rel)
