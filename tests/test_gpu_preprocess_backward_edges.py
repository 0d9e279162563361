"""Per-Gaussian preprocess backward (csrc/gs_backward.cu) against a float64 evaluation of the same chain, at the edges
where it goes wrong: the near plane (S1), the 1.3 tanfov frustum clamp (S2), the SH clamp at every degree and
coefficient count (S3), covariances from extreme scales, scale modifiers, unnormalised quaternions and near-singular
precomputed matrices (S4), and the multi-view kernel's view chunks, Gaussian ranges and partial visibility (S5).
Every scene has a CPU test of its premise; the oracle's restatement is pinned on the CPU by float64 finite
differences and at hand-built quirk points.

The kernels are fed through `gs_b200_debug_preprocess_backward[_multi]` with per-splat sums chosen here, so every
gradient element is attributable to one Gaussian and one set of inputs.  The one-view kernel runs once per view with
accumulation (the Python optimisation loop's order), the multi-view kernel through the step's own chunk and range code
(balanced chunks of at most 16 views, the last chunk split over Gaussian ranges as with a gradient sink), and the
oracle sums the views over the chunk boundaries the library reports (`gs_b200_step_view_chunks`).  Reference and bars: `oracle/gs_bwd_oracle.py`
(float64 values, fp32 decisions, a running fp32 error bound per element; an element passes within BAR_K = 2 times
its bound, and must be exactly 0 where the oracle is exactly 0).  Radii come from the fp32 forward oracle, whose
integer outputs are the kernels' bit for bit; S3 also runs the rasterizer end to end and checks that the sign of
every rendered colour channel decides its SH gradient.  Two runs of every launch must agree bit for bit."""
import ctypes as C
import math
from functools import lru_cache

import numpy as np
import pytest
import torch

from oracle import gs_bwd_oracle as B
from oracle import gs_oracle as O

f32 = np.float32
FOVY = 49.1


# ---------------------------------------------------------------------------------------------------------------------
# scene helpers
# ---------------------------------------------------------------------------------------------------------------------
def settings(W, H, deg, radius=1.75, elev=0.0, azim=0.0, mod=1.0, target=None):
    return O.minicam_settings(O.orbit_camera(elev, azim, radius, target=target), W, H, FOVY, sh_degree=deg,
                              scale_modifier=mod)


def view_of(st):
    W, H = st.image_width, st.image_height
    tfx, tfy = f32(st.tanfovx), f32(st.tanfovy)
    return {"m": st.viewmatrix.numpy().astype(f32).reshape(16), "p": st.projmatrix.numpy().astype(f32).reshape(16),
            "cam": st.campos.numpy().astype(f32), "tanfovx": tfx, "tanfovy": tfy,
            "fx": f32(f32(W) / (f32(2) * tfx)), "fy": f32(f32(H) / (f32(2) * tfy)), "W": W, "H": H}


def fwd_pre(cl, st):
    """the fp32 forward oracle (its integer outputs are the kernels' bit for bit)"""
    t = lambda k: None if cl.get(k) is None else torch.as_tensor(cl[k])          # noqa: E731
    shs = t("shs")
    if shs is None and cl.get("colors_precomp") is None:
        shs = torch.zeros(len(cl["means3D"]), 1, 3)
    return O.preprocess(t("means3D"), t("scales"), t("rotations"), t("opacities"), shs, t("colors_precomp"),
                        t("cov3D_precomp"), None, st)


def fwd_radii(cl, st):
    return fwd_pre(cl, st)["radii"].numpy().astype(np.int32)


def rand_sg(rng, n, scale=1.0):
    """per-splat sums (sum w dx, sum w dy, dL/ddepth, 0, sum w dx^2, sum w dx dy, sum w dy^2, dL/do, dL/drgb, 0), fp32
    values"""
    sg = np.zeros((n, 12))
    sg[:, 0:3] = rng.uniform(-1, 1, (n, 3))
    sg[:, 4:8] = rng.uniform(-1, 1, (n, 4))
    sg[:, 4] = np.abs(sg[:, 4]) * 3; sg[:, 6] = np.abs(sg[:, 6]) * 3
    sg[:, 8:11] = rng.uniform(-1, 1, (n, 3))
    return (sg * scale).astype(f32).astype(np.float64)


def oracle(cl, sts, sg, radii, chunk=1, bounds=None):
    deg = sts[0].sh_degree
    shs = cl.get("shs")
    M = shs.shape[1] if shs is not None else 0
    vs = []
    for st in sts:
        vw = view_of(st)
        vw.update(B.decisions(vw, deg, cl["means3D"], shs))
        vs.append(vw)
    with np.errstate(all="ignore"):
        return B.preprocess_backward(vs, deg, M, cl["means3D"], sg, radii, shs=shs, colors_precomp=cl.get("colors_precomp"),
                                     scales=cl.get("scales"), rots=cl.get("rotations"),
                                     cov3D_precomp=cl.get("cov3D_precomp"), mod=sts[0].scale_modifier, chunk=chunk,
                                     bounds=bounds)


# ---------------------------------------------------------------------------------------------------------------------
# kernel runners
# ---------------------------------------------------------------------------------------------------------------------
def _dev(a, dtype=torch.float32):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a)).to(dtype).cuda().contiguous()


def run_one(cl, sts, sg, radii):
    """the one-view kernel once per view, accumulating into zeroed gradients; returns name -> flat numpy"""
    from gs_b200 import _lib
    from gs_b200 import rasterizer as R
    N = len(cl["means3D"])
    shs = cl.get("shs")
    M = shs.shape[1] if shs is not None else 0
    inp = {k: _dev(cl.get(k)) for k in ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations",
                                        "cov3D_precomp")}
    if inp["opacities"] is None:
        inp["opacities"] = torch.full((N, 1), 0.5, device="cuda")
    sizes = {"means3D": 3 * N, "means2D": 3 * N, "shs": 3 * N * M, "colors": 3 * N, "opacities": N, "scales": 3 * N,
             "rotations": 4 * N, "cov3D": 6 * N}
    want = {"means3D": True, "means2D": True, "shs": shs is not None, "colors": cl.get("colors_precomp") is not None,
            "opacities": True, "scales": cl.get("scales") is not None, "rotations": cl.get("scales") is not None,
            "cov3D": cl.get("cov3D_precomp") is not None}
    out = {k: torch.zeros(sizes[k], device="cuda") if want[k] else None for k in sizes}
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())               # noqa: E731
    for v, st in enumerate(sts):
        keep = []
        rs = R.GaussianRasterizationSettings(st.image_height, st.image_width, st.tanfovx, st.tanfovy, st.bg.cuda(),
                                             st.scale_modifier, st.viewmatrix.cuda(), st.projmatrix.cuda(),
                                             st.sh_degree, st.campos.cuda(), False, False)
        view = R._make_view(rs, keep)
        rad = _dev(radii[v], torch.int32)
        sgd = _dev(sg[v], torch.float64)
        _lib.check(_lib.lib.gs_b200_debug_preprocess_backward(
            C.byref(view), N, M, p(inp["means3D"]), p(inp["shs"]), p(inp["colors_precomp"]), p(inp["opacities"]),
            p(inp["scales"]), p(inp["rotations"]), p(inp["cov3D_precomp"]), p(rad), p(sgd),
            p(out["means3D"]), p(out["means2D"]), p(out["shs"]), p(out["colors"]), p(out["opacities"]),
            p(out["scales"]), p(out["rotations"]), p(out["cov3D"]), 1, R._stream()))
    torch.cuda.synchronize()
    return {k: t.cpu().numpy() for k, t in out.items() if t is not None}


def step_chunks(V):
    """the multi-view step's view chunk boundaries [v0 of each chunk..., V], as the library computes them"""
    from gs_b200 import _lib
    b = (C.c_int32 * (V + 1))()
    n = _lib.lib.gs_b200_step_view_chunks(V, b)
    assert n > 0, _lib.last_error()
    return list(b[:n + 1])


def run_multi(cl, sts, sg, radii, nparts=1):
    """the multi-view kernel as the step drives it; returns name -> flat numpy"""
    from gs_b200 import _lib
    from gs_b200 import rasterizer as R
    N, M = len(cl["means3D"]), cl["shs"].shape[1]
    st0 = sts[0]
    views = np.zeros((len(sts), 40), f32)
    for v, st in enumerate(sts):
        views[v, :16] = st.viewmatrix.numpy().reshape(16); views[v, 16:32] = st.projmatrix.numpy().reshape(16)
        views[v, 32:35] = st.campos.numpy(); views[v, 35:38] = st.bg.numpy()
        views[v, 38], views[v, 39] = st.tanfovx, st.tanfovy
    d = {k: _dev(cl[k]) for k in ("means3D", "shs", "scales", "rotations")}
    vd, rad, sgd = _dev(views), _dev(np.stack(radii), torch.int32), _dev(np.stack(sg), torch.float64)
    g = torch.full((N * (3 + 3 * M + 1 + 3 + 4 + 3),), float("nan"), device="cuda")
    _lib.check(_lib.lib.gs_b200_debug_preprocess_backward_multi(
        len(sts), st0.image_height, st0.image_width, st0.sh_degree, st0.scale_modifier, C.c_void_p(vd.data_ptr()), N, M,
        *(C.c_void_p(d[k].data_ptr()) for k in ("means3D", "shs", "scales", "rotations")), C.c_void_p(rad.data_ptr()),
        C.c_void_p(sgd.data_ptr()), C.c_void_p(g.data_ptr()), nparts, R._stream()))
    torch.cuda.synchronize()
    g = g.cpu().numpy()
    o, out = 0, {}
    for k, n in (("means3D", 3 * N), ("shs", 3 * N * M), ("opacities", N), ("scales", 3 * N), ("rotations", 4 * N),
                 ("means2D", 3 * N)):
        out[k] = g[o:o + n]; o += n
    out["means2D"] = out["means2D"].reshape(N, 3)[:, :2].reshape(-1)       # the step leaves the third column alone
    return out


def compare(tag, got, ref):
    worst = {}
    for k, v in got.items():
        r = ref[k]
        if k == "means2D" and v.size != r.v.size:
            r = B.E(r.v.reshape(-1, 3)[:, :2].reshape(-1), r.e.reshape(-1, 3)[:, :2].reshape(-1))
        worst[k], _ = B.check(f"{tag} {k}", v, r)
    print(tag, "worst error / bar:", {k: f"{w:.3g}" for k, w in worst.items()})
    return max(worst.values())


def both_kernels(tag, cl, sts, sg, radii, nparts=1, multi=True):
    """one-view and (SH + scales clouds) multi-view kernel, each against the oracle in its order and run twice"""
    a, b = run_one(cl, sts, sg, radii), run_one(cl, sts, sg, radii)
    for k in a:
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), f"{tag}: one-view {k} differs between runs"
    w = compare(f"{tag} one-view", a, oracle(cl, sts, sg, radii, chunk=1))
    if multi:
        a, b = run_multi(cl, sts, sg, radii, nparts), run_multi(cl, sts, sg, radii, nparts)
        for k in a:
            assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), f"{tag}: multi-view {k} differs between runs"
        ref = oracle(cl, sts, sg, radii, bounds=step_chunks(len(sts)))
        w = max(w, compare(f"{tag} multi-view", a, ref))
    return w


def _walk(f, x0, target, steps=64):
    """fp32 x near x0 with f(x) == target, nearest first; None when no x within `steps` ulps does"""
    x0 = f32(x0)
    up, dn = x0, x0
    for _ in range(steps):
        for x in (up, dn):
            if f(x) == target:
                return x
        up, dn = np.nextafter(up, f32(np.inf)), np.nextafter(dn, f32(-np.inf))
    return None


# ---------------------------------------------------------------------------------------------------------------------
# S1: near plane.  Camera 0.25 from the origin on +z (axis-aligned view matrix: t is exact in any contraction), so
# t.z = 0.25 - z reaches every fp32 value near 0.2.
# ---------------------------------------------------------------------------------------------------------------------
S1_ULPS = (0, 1, 2, 3, 5, 8)


@lru_cache(None)
def s1_scene():
    W, H, deg = 64, 192, 1
    st = settings(W, H, deg, radius=0.25)
    m = st.viewmatrix.numpy().reshape(16)
    tz_of = lambda z: B.view_t32(m, np.array([[0, 0, z]], f32))[2][0]      # noqa: E731
    targets = [f32(0.2)]
    for _ in range(max(S1_ULPS)):
        targets.append(np.nextafter(targets[-1], f32(1)))
    tzs = [targets[k] for k in S1_ULPS] + [f32(v) for v in (0.21, 0.23, 0.25, 0.27, 0.3)]
    zs = [_walk(tz_of, 0.25 - float(t), t) for t in tzs]
    rng = np.random.default_rng(1)
    rows = []
    for z, t in zip(zs, tzs):
        for sx in (0.0005, 0.004, 0.09):           # ~0.1 px, ~1 px and a whole-square footprint at t.z 0.2
            off = rng.uniform(-0.6, 0.6, 2) * float(t) * np.array([st.tanfovx, st.tanfovy])
            rows.append((off[0], off[1], z, sx))
    rows = np.array(rows, np.float64)
    n = len(rows)
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    cl = {"means3D": rows[:, :3].astype(f32), "scales": (rows[:, 3:4] * rng.uniform(0.5, 1.5, (n, 3))).astype(f32),
          "rotations": q.astype(f32), "opacities": np.full((n, 1), 0.7, f32),
          "shs": rng.uniform(-0.5, 0.5, (n, 4, 3)).astype(f32)}
    return cl, st, np.array([tz_of(z) for z in rows[:, 2].astype(f32)]), tzs


def test_s1_premise():
    cl, st, tz, tzs = s1_scene()
    assert all(t is not None for t in tzs)
    radii = fwd_radii(cl, st)
    assert np.all(tz[:3] == f32(0.2)) and np.all(radii[:3] == 0), "t.z = 0.2f must be culled"
    one_up = np.nextafter(f32(0.2), f32(1))
    assert np.all(tz[3:6] == one_up) and np.all(radii[3:] > 0), "everything above 0.2f is visible"
    pre = fwd_pre(cl, st)
    rows = (pre["rect_max"] - pre["rect_min"])[:, 1].numpy()
    assert rows.max() > 8, "a footprint over more than 8 tile rows (tight_spans' whole-square path)"


@pytest.mark.gpu
def test_s1_near_plane():
    cl, st, tz, _ = s1_scene()
    radii = fwd_radii(cl, st)
    rng = np.random.default_rng(2)
    sg = [rand_sg(rng, len(radii))]
    got = run_one(cl, [st], sg, [radii])
    for k, v in got.items():
        per = v.reshape(len(radii), -1)
        assert np.all(per[radii == 0] == 0), f"S1: culled Gaussian has a nonzero {k} gradient"
    both_kernels("S1", cl, [st], sg, [radii])


# ---------------------------------------------------------------------------------------------------------------------
# S2: frustum clamp.  t.x / t.z (and t.y / t.z) at +-limit exactly as fp32 computes it, one ulp inside and outside, and
# far outside; off-screen centres whose footprints reach the image.
# ---------------------------------------------------------------------------------------------------------------------
def outside(k):
    """S2 case k: -1 one ulp inside, 0 at the limit, 1 one ulp outside, +-9 far outside"""
    return k == 1 or abs(k) == 9


@lru_cache(None)
def s2_scene():
    W, H, deg = 64, 48, 0
    st = settings(W, H, deg)
    vw = view_of(st)
    m = vw["m"]
    lims = (f32(1.3) * vw["tanfovx"], f32(1.3) * vw["tanfovy"])
    rng = np.random.default_rng(3)
    rows, kinds = [], []
    for axis in (0, 1):
        lim = lims[axis]
        for sign in (1, -1):
            for k in (-1, 0, 1):
                target = f32(sign * lim)
                for _ in range(abs(k)):
                    target = np.nextafter(target, f32(sign * k * np.inf))       # k = 1: outwards
                for z in (0.5, 0.75, -0.25):
                    tz = B.view_t32(m, np.array([[0, 0, z]], f32))[2][0]

                    def ratio(c, z=z, axis=axis):
                        p = np.zeros((1, 3), f32); p[0, 2] = z; p[0, axis] = c
                        t = B.view_t32(m, p)
                        return (t[axis] / t[2])[0]
                    c0 = float(target) * float(tz) * (1 if axis == 0 else -1)
                    c = _walk(ratio, c0, target, 256)
                    if c is None:
                        continue
                    p = [0.0, 0.0, z]; p[axis] = c
                    p[1 - axis] = rng.uniform(-0.1, 0.1)
                    rows.append(p); kinds.append((axis, k))
                    break
        for sign in (1, -1):        # far outside: centres off-screen, footprints reaching in
            for fac in (1.6, 2.2):
                z = 0.5
                tz = 1.25
                p = [0.0, 0.0, z]; p[axis] = sign * fac * float(lim) * tz * (1 if axis == 0 else -1)
                rows.append(p); kinds.append((axis, 9 * sign))
    rows = np.array(rows, f32)
    n = len(rows)
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    scl = np.where(np.array([abs(k[1]) == 9 for k in kinds])[:, None], 0.6, 0.1) * rng.uniform(0.6, 1.4, (n, 3))
    cl = {"means3D": rows, "scales": scl.astype(f32), "rotations": q.astype(f32), "opacities": np.full((n, 1), 0.7, f32),
          "shs": rng.uniform(-0.5, 0.5, (n, 1, 3)).astype(f32)}
    return cl, st, kinds


def test_s2_premise():
    cl, st, kinds = s2_scene()
    vw = view_of(st)
    inx, iny = B.clamp_masks32(vw["m"], cl["means3D"], vw["tanfovx"], vw["tanfovy"])
    have = set()
    for i, (axis, k) in enumerate(kinds):
        inside = (inx if axis == 0 else iny)[i]
        assert inside != outside(k), (i, axis, k)
        have.add((axis, k))
    assert {(a, k) for a in (0, 1) for k in (-1, 0, 1, 9, -9)} <= have, "every limit case on both axes"
    radii = fwd_radii(cl, st)
    far = np.array([abs(k) == 9 for _, k in kinds])
    assert radii[far].min() > 0, "off-screen centres whose footprints reach the image are visible"
    assert np.all(radii > 0)


@pytest.mark.gpu
def test_s2_frustum_clamp():
    cl, st, kinds = s2_scene()
    radii = fwd_radii(cl, st)
    n = len(radii)
    # conic sums only: then dL/dmean = W^T (dtx, dty, dtz) with W = diag(1, -1, -1), so the clamped component's direct
    # gradient is visible on its own
    rng = np.random.default_rng(4)
    sg = np.zeros((n, 12)); sg[:, 4:7] = rng.uniform(0.2, 1.0, (n, 3)).astype(f32)
    got = run_one(cl, [st], [sg], [radii])["means3D"].reshape(n, 3)
    for i, (axis, k) in enumerate(kinds):
        clamped = outside(k)
        assert (got[i, axis] == 0) == clamped, f"S2 row {i}: axis {axis} case {k}: d/dt{'xy'[axis]} = {got[i, axis]}"
        assert got[i, 2] != 0, f"S2 row {i}: t.z lost its gradient"
    both_kernels("S2 conic", cl, [st], [sg], [radii])
    both_kernels("S2", cl, [st], [rand_sg(rng, n)], [radii])


# ---------------------------------------------------------------------------------------------------------------------
# S3: SH clamp.  One scene per (degree, M); each Gaussian's three channels take three of the target colours (before
# the max with 0), solved through the last SH coefficient so the forward's fp32 colour is exactly the target.
# ---------------------------------------------------------------------------------------------------------------------
S3_CASES = [(d, M) for d in range(4) for M in range((d + 1) ** 2, 17)]
# the colour is r + 0.5 (exact): it moves in steps of 2^-24 below 0 (|r| in [0.5, 1)) and 2^-25 above
UN, UP = f32(2.0 ** -24), f32(2.0 ** -25)
S3_TARGETS = (f32(-round(1e-3 / UN)) * UN, -3 * UN, -UN, f32(0.0), UP, 3 * UP, f32(round(1e-3 / UP)) * UP)
S3_GRID = 5                          # 5 x 5 cells of 16 px, one Gaussian per cell, 21 used


@lru_cache(None)
def s3_scene(deg, M):
    W = H = 16 * S3_GRID
    st = settings(W, H, deg)
    vw = view_of(st)
    rng = np.random.default_rng(100 * deg + M)
    n = 21
    cells = rng.permutation(S3_GRID * S3_GRID)[:n]
    px = 16 * (cells % S3_GRID) + 7.5 + rng.uniform(-2, 2, n)        # off the axis: no direction component is 0
    py = 16 * (cells // S3_GRID) + 7.5 + rng.uniform(-2, 2, n)
    dep = rng.uniform(1.4, 2.2, n)
    k = math.tan(math.radians(FOVY) / 2) * dep / (H / 2)
    means = np.stack([(px - (W - 1) / 2) * k, -(py - (H - 1) / 2) * k, 1.75 - dep], 1).astype(f32)
    nb = (deg + 1) ** 2
    shs = np.zeros((n, M, 3), f32)
    shs[:, :nb] = rng.uniform(-0.3, 0.3, (n, nb, 3))
    shs[:, nb:] = rng.uniform(-5, 5, (n, M - nb, 3))            # rows the active degree must ignore
    shs[:, 0] = -0.5 / B.SH_C0                                  # colour near 0 before the last coefficient
    dirs = means - vw["cam"][None]
    targets = np.array([[S3_TARGETS[(i + 2 * ch) % 7] for ch in range(3)] for i in range(n)], f32)
    with np.errstate(all="ignore"):
        dn = dirs.astype(np.float64) / np.linalg.norm(dirs.astype(np.float64), axis=1, keepdims=True)
        bas = np.stack([b.v for b in B._sh_basis(deg, B.E(dn[:, 0]), B.E(dn[:, 1]), B.E(dn[:, 2]))[0]], 1)
    for i in range(n):
        for ch in range(3):
            # solved through the last active coefficient (the final fma), else the one with the largest basis value
            # that reaches the target: every fp32 value within 4096 ulps of the float64 solution, in one call
            for last in [nb - 1] + [int(k) for k in np.argsort(-np.abs(bas[i]))[:3]]:
                s0 = float(shs[i, last, ch])
                base = float(B.sh_colour32(deg, shs[i:i + 1], dirs[i:i + 1])[0, ch])
                guess = f32(s0 + (float(targets[i, ch]) - base) / bas[i, last])
                cand = (np.int64(guess.view(np.int32)) + np.arange(-4096, 4097)).astype(np.int32).view(f32)
                rows = np.repeat(shs[i:i + 1], len(cand), 0)
                rows[:, last, ch] = cand
                col = B.sh_colour32(deg, rows, np.repeat(dirs[i:i + 1], len(cand), 0))[:, ch]
                hit = np.flatnonzero(col == targets[i, ch])
                if hit.size:
                    shs[i, last, ch] = cand[hit[np.argmin(np.abs(hit - 4096))]]
                    break
    cl = {"means3D": means, "shs": shs, "opacities": np.full((n, 1), 0.9, f32),
          "scales": np.repeat((1.5 * k)[:, None], 3, 1).astype(f32),
          "rotations": np.tile(np.array([1, 0, 0, 0], f32), (n, 1))}
    return cl, st


def s3_colours(deg, M):
    cl, st = s3_scene(deg, M)
    vw = view_of(st)
    return B.sh_colour32(deg, cl["shs"], cl["means3D"] - vw["cam"][None])


def test_s3_premise():
    for deg, M in S3_CASES:
        col = s3_colours(deg, M)
        cats = {"-1e-3": col == S3_TARGETS[0], "-k ulp": (col < 0) & (col >= -4 * UN), "0": col == 0,
                "+k ulp": (col > 0) & (col <= 4 * UP), "+1e-3": col == S3_TARGETS[-1]}
        for name, hit in cats.items():
            assert hit.any(axis=0).all(), f"S3 deg {deg} M {M}: no channel-wide '{name}' colour"
        cl, st = s3_scene(deg, M)
        assert np.all(fwd_radii(cl, st) > 0)
    assert len(S3_CASES) == sum(16 - (d + 1) ** 2 + 1 for d in range(4))


@pytest.mark.gpu
@pytest.mark.parametrize("deg,M", S3_CASES)
def test_s3_sh_clamp(deg, M):
    from gs_b200 import rasterizer as R
    cl, st = s3_scene(deg, M)
    n = len(cl["means3D"])
    col = s3_colours(deg, M)
    # end to end: bg 0, one splat per cell, so the centre pixel's sign is the forward colour's sign
    rs = R.GaussianRasterizationSettings(st.image_height, st.image_width, st.tanfovx, st.tanfovy,
                                         torch.zeros(3, device="cuda"), 1.0, st.viewmatrix.cuda(), st.projmatrix.cuda(),
                                         deg, st.campos.cuda(), False, False)
    inp = {k: torch.as_tensor(cl[k]).cuda().requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales",
                                                                          "rotations")}
    m2 = torch.zeros(n, 3, device="cuda", requires_grad=True)
    img, radii, _, _ = R.GaussianRasterizer(rs)(means3D=inp["means3D"], means2D=m2, shs=inp["shs"], colors_precomp=None,
                                                opacities=inp["opacities"], scales=inp["scales"],
                                                rotations=inp["rotations"], cov3D_precomp=None)
    img.sum().backward()
    radii = radii.cpu().numpy()
    assert np.array_equal(radii, fwd_radii(cl, st))
    pre = O.preprocess(*(torch.as_tensor(cl[k]) for k in ("means3D", "scales", "rotations", "opacities", "shs")), None,
                       None, None, st)
    pix = np.floor(pre["xy"].detach().numpy() + 0.5).astype(int)
    shown = img.detach().cpu().numpy()[:, pix[:, 1], pix[:, 0]].T           # [n, 3]
    dsh = inp["shs"].grad.cpu().numpy()
    nb = (deg + 1) ** 2
    assert np.all(dsh[:, nb:] == 0), "SH rows above the active degree must get exactly 0"
    assert np.array_equal(shown > 0, col > 0), "rendered colour sign differs from the forward's fp32 colour"
    live = dsh[:, 0] != 0
    bad = np.argwhere(live != (col >= 0))
    assert bad.size == 0, f"deg {deg} M {M}: SH clamp mask disagrees with the forward colour at (Gaussian, channel) " \
        f"{bad[:4].tolist()}: colour {[float(col[i, c]) for i, c in bad[:4]]}, dSH[0] {[float(dsh[i, 0, c]) for i, c in bad[:4]]}"
    # both kernels against the oracle, two views so the multi-view kernel accumulates SH rows over views, and an
    # accumulating second chunk (17 views) for the SH rows across chunks
    rng = np.random.default_rng(deg * 31 + M)
    sg = [rand_sg(rng, n) for _ in range(17)]
    both_kernels(f"S3 deg {deg} M {M}", cl, [st] * 17, sg, [fwd_radii(cl, st)] * 17)


# ---------------------------------------------------------------------------------------------------------------------
# S4: covariance.  Scale anisotropy 1e-6 .. 1e2 (cov2D at the 0.3 floor), scale modifiers 0.5 / 1 / 3, quaternion
# norms 1e-2 / 1 / 30; precomputed covariances whose 2D determinant is ~1e-4 (the 1e-7 quirk active) or exactly 0
# (culled); colours precomputed.
# ---------------------------------------------------------------------------------------------------------------------
def s4_sr_scene(mod):
    W, H, deg = 64, 48, 2
    st = settings(W, H, deg, mod=mod)
    rng = np.random.default_rng(int(mod * 10))
    rows = []
    for ratio in (1e-6, 1e-4, 1e-2, 1.0, 1e2):
        for qn in (1e-2, 1.0, 30.0):
            rows.append((ratio, qn))
    n = len(rows)
    means = np.stack([rng.uniform(-0.3, 0.3, n), rng.uniform(-0.2, 0.2, n), rng.uniform(-0.3, 0.3, n)], 1)
    base = rng.uniform(0.01, 0.03, n)
    ratio = np.array([r for r, _ in rows]); qn = np.array([q for _, q in rows])
    scales = np.stack([base, base * ratio, base * np.sqrt(ratio)], 1)
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    q *= qn[:, None] / np.sqrt(qn[:, None])         # |q|^2 = qn: R scales with |q|^2, so the footprints stay sane
    cl = {"means3D": means.astype(f32), "scales": (scales / np.maximum(qn, 1)[:, None]).astype(f32),
          "rotations": q.astype(f32), "opacities": np.full((n, 1), 0.6, f32),
          "shs": rng.uniform(-0.5, 0.5, (n, 9, 3)).astype(f32)}
    return cl, st


def cov2d32(cl, st):
    return fwd_pre(cl, st)["cov2d"].detach().numpy()


@lru_cache(None)
def s4_precomp_scene():
    """on-axis Gaussians (T diagonal) with cov3D = [[0, b, 0], [b, 0, 0], [0, 0, 0]] + tiny PSD parts: cov2D =
    [[0.3, x], [x, 0.3]], det = 0.09 - x^2; x solved for det ~1e-4 (quirk active), ~1e-2 and, by walking ulps, det
    exactly 0 in fp32 (culled).  Colours precomputed."""
    W = H = 64
    st = settings(W, H, 0)
    vw = view_of(st)
    dep = 1.25
    T = float(vw["fx"]) / dep
    rows, kind = [], []
    for tgt in (1e-4, 2e-4, 1e-2, 0.05, "zero"):
        x = math.sqrt(0.09 - (0 if tgt == "zero" else tgt))
        b = f32(-x / (T * T))                                      # T11 = -fy / tz: cb = T00 (b T11) = -b T^2
        cp = np.zeros((1, 6), f32); cp[0, 1] = b
        cl1 = {"means3D": np.array([[0, 0, 1.75 - dep]], f32), "cov3D_precomp": cp,
               "opacities": np.full((1, 1), 0.5, f32), "colors_precomp": np.full((1, 3), 0.5, f32)}
        if tgt == "zero":
            def det(bb):
                c2 = cl1.copy(); c2["cov3D_precomp"] = np.array([[0, bb, 0, 0, 0, 0]], f32)
                a, bq, c = cov2d32(c2, st)[0]
                return f32(a) * f32(c) - f32(bq) * f32(bq)
            b = _walk(det, b, f32(0.0), 4096)
            cp[0, 1] = b
        rows.append(cp[0]); kind.append(tgt)
    n = len(rows)
    rng = np.random.default_rng(5)
    cl = {"means3D": np.tile(np.array([[0, 0, 1.75 - dep]], f32), (n, 1)), "cov3D_precomp": np.array(rows, f32),
          "opacities": np.full((n, 1), 0.5, f32), "colors_precomp": rng.uniform(0, 1, (n, 3)).astype(f32)}
    # a few generic precomputed covariances, off-axis
    m = rng.normal(size=(6, 3, 3)) * 0.02
    covs = np.einsum("nij,nkj->nik", m, m)
    gen = np.stack([covs[:, 0, 0], covs[:, 0, 1], covs[:, 0, 2], covs[:, 1, 1], covs[:, 1, 2], covs[:, 2, 2]], 1)
    cl["means3D"] = np.concatenate([cl["means3D"], rng.uniform(-0.3, 0.3, (6, 3)).astype(f32)])
    cl["cov3D_precomp"] = np.concatenate([cl["cov3D_precomp"], gen.astype(f32)])
    cl["opacities"] = np.full((n + 6, 1), 0.5, f32)
    cl["colors_precomp"] = rng.uniform(0, 1, (n + 6, 3)).astype(f32)
    return cl, st, kind


def test_s4_premise():
    for mod in (0.5, 1.0, 3.0):
        cl, st = s4_sr_scene(mod)
        radii = fwd_radii(cl, st)
        assert np.all(radii > 0)
        c2 = cov2d32(cl, st)
        assert np.any(np.abs(c2[:, 0] - 0.3) < 1e-3) or np.any(np.abs(c2[:, 2] - 0.3) < 1e-3), "a cov2D at the 0.3 floor"
        qn = np.linalg.norm(cl["rotations"].astype(np.float64), axis=1)
        assert qn.min() < 0.2 and qn.max() > 5, "unnormalised quaternions, both ways"
    cl, st, kind = s4_precomp_scene()
    radii = fwd_radii(cl, st)
    c2 = cov2d32(cl, st).astype(np.float64)
    det = c2[:, 0] * c2[:, 2] - c2[:, 1] ** 2
    for i, k in enumerate(kind):
        if k == "zero":
            assert radii[i] == 0, "fp32 det exactly 0 is culled"
        else:
            assert radii[i] > 0 and abs(det[i] - k) < 0.2 * k, (k, det[i])
    d2 = det[:2] ** 2
    assert np.all(1e-7 / d2 > 2), "the 1e-7 in 1/(det^2 + 1e-7) dominates for det ~1e-4"


@pytest.mark.gpu
@pytest.mark.parametrize("mod", (0.5, 1.0, 3.0))
def test_s4_scales_rotations(mod):
    cl, st = s4_sr_scene(mod)
    radii = fwd_radii(cl, st)
    rng = np.random.default_rng(6)
    both_kernels(f"S4 mod {mod}", cl, [st], [rand_sg(rng, len(radii))], [radii])


@pytest.mark.gpu
def test_s4_precomputed_covariance_and_colours():
    cl, st, kind = s4_precomp_scene()
    radii = fwd_radii(cl, st)
    rng = np.random.default_rng(7)
    sg = rand_sg(rng, len(radii), scale=1e-3)
    got = run_one(cl, [st], [sg], [radii])
    for k, v in got.items():
        assert np.all(v.reshape(len(radii), -1)[radii == 0] == 0), f"culled Gaussian has a nonzero {k} gradient"
    both_kernels("S4 precomp", cl, [st], [sg], [radii], multi=False)


# ---------------------------------------------------------------------------------------------------------------------
# S5: multi-view structure.  Orbit views around a cloud that no view sees whole; one view looks away from it.
# ---------------------------------------------------------------------------------------------------------------------
S5_CASES = [  # (V, N, M, nparts)
    (1, 1, 16, 1), (2, 127, 9, 1), (16, 128, 16, 1), (16, 129, 16, 2), (17, 129, 16, 2), (17, 129, 9, 3),
    (33, 1000, 16, 4),
    (33, 100003, 9, 3)]


@lru_cache(None)
def s5_scene(V, N, M):
    rng = np.random.default_rng(V * 1000 + N + M)
    W, H, deg = 48, 32, (3 if M == 16 else 2)
    sts = []
    for v in range(V):
        if v == 1:
            sts.append(settings(W, H, deg, target=np.array([40.0, 0, 0], f32)))       # sees nothing
        else:
            sts.append(settings(W, H, deg, elev=rng.uniform(-30, 30), azim=360.0 * v / V + rng.uniform(0, 10)))
    means = rng.uniform(-1.0, 1.0, (N, 3))
    means[rng.random(N) < 0.03, 1] += 40.0         # straight above the orbit: no view sees these
    q = rng.normal(size=(N, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    cl = {"means3D": means.astype(f32), "scales": rng.uniform(0.005, 0.05, (N, 3)).astype(f32),
          "rotations": q.astype(f32), "opacities": np.full((N, 1), 0.5, f32),
          "shs": rng.uniform(-0.4, 0.4, (N, M, 3)).astype(f32)}
    radii = [fwd_radii(cl, st) for st in sts]
    sg = [rand_sg(rng, N) for _ in sts]
    return cl, sts, radii, sg


def s5_premise(V, N, radii):
    vis = np.stack(radii) > 0
    if V > 1:
        assert not vis[1].any(), "view 1 sees nothing"
    if N > 100:
        nv = vis.sum(0)
        assert (nv == 0).any() and ((nv > 0) & (nv < V)).any(), "Gaussians seen by none and by a subset of views"


def test_s5_premise():
    for V, N, M, nparts in S5_CASES:
        s5_premise(V, N, s5_scene(V, N, M)[2])
    assert {V for V, *_ in S5_CASES} == {1, 2, 16, 17, 33} and {N for _, N, *_ in S5_CASES} >= {1, 127, 128, 129, 100003}
    # Gaussian ranges in a single writing chunk (V <= 16) and in an accumulating last chunk (V > 16)
    assert any(p > 1 and V <= 16 for V, _, _, p in S5_CASES) and any(p > 1 and V > 16 for V, _, _, p in S5_CASES)


def test_step_view_chunks():
    """the step's chunks: as few as 16 views allow, balanced (17 views run as 9 + 8, 33 as 11 + 11 + 11)"""
    for V in range(1, 65):
        b = step_chunks(V)
        n = -(-V // 16)
        size = -(-V // n)
        assert b == [min(V, k * size) for k in range(n)] + [V], (V, b)
        assert max(np.diff(b)) <= 16 and min(np.diff(b)) >= 1
    assert step_chunks(17) == [0, 9, 17] and step_chunks(33) == [0, 11, 22, 33]


@pytest.mark.gpu
@pytest.mark.parametrize("V,N,M,nparts", S5_CASES)
def test_s5_multi_view(V, N, M, nparts):
    cl, sts, radii, sg = s5_scene(V, N, M)
    s5_premise(V, N, radii)
    both_kernels(f"S5 V {V} N {N} M {M} parts {nparts}", cl, sts, sg, radii, nparts)


# ---------------------------------------------------------------------------------------------------------------------
# the oracle's restatement on the CPU
# ---------------------------------------------------------------------------------------------------------------------
def _forward64(x, view, deg, mod, coef, hold):
    """the functional whose gradient the backward computes, in float64: coef fixes the per-splat sums' linearisation;
    `hold` = clamped (cx, cy) values held fixed where the fp32 clamp is active (the reference's t.z rule)"""
    m = np.asarray(view["m"], np.float64); p = np.asarray(view["p"], np.float64)
    mean, sc, q, sh = x[:3], x[3:6] * mod, x[6:10], x[10:].reshape(-1, 3)
    tx, ty, tz = (m[i] * mean[0] + m[4 + i] * mean[1] + m[8 + i] * mean[2] + m[12 + i] for i in range(3))
    hx, hy, hw = (p[i] * mean[0] + p[4 + i] * mean[1] + p[8 + i] * mean[2] + p[12 + i] for i in (0, 1, 3))
    pw = 1 / (hw + float(f32(1e-7)))
    px, py = ((hx * pw + 1) * view["W"] - 1) * 0.5, ((hy * pw + 1) * view["H"] - 1) * 0.5
    r, a, b, c = q
    R = np.array([[1 - 2 * (b * b + c * c), 2 * (a * b - r * c), 2 * (a * c + r * b)],
                  [2 * (a * b + r * c), 1 - 2 * (a * a + c * c), 2 * (b * c - r * a)],
                  [2 * (a * c - r * b), 2 * (b * c + r * a), 1 - 2 * (a * a + b * b)]])
    Mm = R * sc[None, :]
    S = Mm @ Mm.T
    fx, fy = float(view["fx"]), float(view["fy"])
    cx = hold[0] if hold[0] is not None else tx
    cy = hold[1] if hold[1] is not None else ty
    J = np.array([[fx / tz, 0, -fx * cx / tz ** 2], [0, fy / tz, -fy * cy / tz ** 2]])
    Wm = np.array([[m[0], m[4], m[8]], [m[1], m[5], m[9]], [m[2], m[6], m[10]]])
    T = J @ Wm
    c2 = T @ S @ T.T + 0.3 * np.eye(2)
    det = c2[0, 0] * c2[1, 1] - c2[0, 1] ** 2
    A, Bc, Cc = c2[1, 1] / det, -c2[0, 1] / det, c2[0, 0] / det
    d = mean - np.asarray(view["cam"], np.float64)
    d = d / np.linalg.norm(d)
    bas = B._sh_basis(deg, B.E(d[0:1]), B.E(d[1:2]), B.E(d[2:3]))[0]
    rgb = sum(bk.v[0] * sh[k] for k, bk in enumerate(bas)) + 0.5
    return (coef["px"] * px + coef["py"] * py + coef["dep"] * tz + coef["A"] * A + coef["B"] * Bc + coef["C"] * Cc
            + np.dot(coef["rgb"], np.maximum(rgb, 0)))


def _fd_case(seed, deg, mod, on_limit=False):
    rng = np.random.default_rng(seed)
    W, H = 64, 48
    st = settings(W, H, deg, mod=mod)
    vw = view_of(st)
    nb = (deg + 1) ** 2
    mean = np.array([rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), rng.uniform(-0.3, 0.3)])
    if on_limit:
        mean[0] = 2.0 * float(f32(1.3) * vw["tanfovx"]) * (1.75 - mean[2])    # clamped in x
    q = rng.normal(size=4) * 1.3
    x = np.concatenate([mean, rng.uniform(0.05, 0.15, 3), q, rng.uniform(-0.4, 0.4, 3 * nb)]).astype(f32).astype(np.float64)
    sg = rand_sg(rng, 1)
    cl = {"means3D": x[None, :3].astype(f32), "scales": x[None, 3:6].astype(f32), "rotations": x[None, 6:10].astype(f32),
          "shs": x[10:].reshape(1, nb, 3).astype(f32), "opacities": np.full((1, 1), 0.5, f32)}
    ref = oracle(cl, [st], [sg], [np.array([1], np.int32)], chunk=1)
    # the linearisation the backward uses: d/dpx = -(A sum w dx + B sum w dy) at the base point
    pre = O.preprocess(*(torch.as_tensor(cl[k]).double() for k in ("means3D", "scales", "rotations", "opacities", "shs")),
                       None, None, None, st)
    A0, B0, C0 = pre["conic"].detach().numpy()[0]
    s = sg[0]
    coef = {"px": -(A0 * s[0] + B0 * s[1]), "py": -(B0 * s[0] + C0 * s[1]), "dep": s[2], "A": -0.5 * s[4],
            "B": -s[5], "C": -0.5 * s[6], "rgb": s[8:11]}
    inx, iny = B.clamp_masks32(vw["m"], cl["means3D"], vw["tanfovx"], vw["tanfovy"])
    tx, ty, tz = B.view_t32(vw["m"], cl["means3D"])
    limx, limy = float(f32(1.3) * vw["tanfovx"]), float(f32(1.3) * vw["tanfovy"])
    hold = (None if inx[0] else float(np.clip(tx[0] / tz[0], -limx, limx)) * float(tz[0]),
            None if iny[0] else float(np.clip(ty[0] / tz[0], -limy, limy)) * float(tz[0]))
    f = lambda y: _forward64(y, vw, deg, mod, coef, hold)              # noqa: E731
    fd = np.zeros_like(x)
    for i in range(len(x)):
        h = 1e-6 * max(1.0, abs(x[i]))
        e = np.zeros_like(x); e[i] = h
        fd[i] = (f(x + e) - f(x - e)) / (2 * h)
    got = np.concatenate([ref["means3D"].v, ref["scales"].v, ref["rotations"].v, ref["shs"].v[:3 * nb]])
    return got, fd, inx[0]


@pytest.mark.parametrize("seed,deg,mod", [(1, 0, 1.0), (2, 1, 0.5), (3, 2, 3.0), (4, 3, 1.0), (5, 3, 0.5)])
def test_oracle_matches_finite_differences(seed, deg, mod):
    got, fd, _ = _fd_case(seed, deg, mod)
    scale = np.abs(fd).max()
    assert np.abs(got - fd).max() <= 1e-6 * scale, np.abs(got - fd).max() / scale


def test_oracle_frustum_clamp_rule_matches_finite_differences():
    """clamped in x: t.x gets no gradient through J, t.z differentiates J with lim t.z held fixed"""
    got, fd, inx = _fd_case(9, 1, 1.0, on_limit=True)
    assert not inx
    assert np.abs(got - fd).max() <= 1e-6 * np.abs(fd).max()


def test_oracle_quirk_values():
    """on the optical axis T is diagonal: dL/dcov3D = (T00^2 ga, T00 T11 gb, 0, T11^2 gc, 0, 0) with
    (ga, gb, gc) = (-cc^2 gA + cb cc gB - cb^2 gC, 2 cb cc gA - (det + 2 cb^2) gB + 2 ca cb gC,
    -cb^2 gA + ca cb gB - ca^2 gC) / (det^2 + 1e-7f); at det ~1e-4 that is 1/11 of the exact derivative"""
    cl, st, kind = s4_precomp_scene()
    vw = view_of(st)
    i = kind.index(1e-4)
    sg = np.zeros((1, 12)); sg[0, 4:7] = (0.25, -0.5, 0.75)
    one = {k: v[i:i + 1] for k, v in cl.items()}
    ref = oracle(one, [st], [sg], [np.array([1], np.int32)], chunk=1)
    T00 = float(vw["fx"]) / 1.25
    T11 = -float(vw["fy"]) / 1.25
    b = float(one["cov3D_precomp"][0, 1])
    ca = cc = float(f32(0.3)); cb = T00 * b * T11
    det = ca * cc - cb * cb
    gA, gB, gC = -0.125, 0.5, -0.375
    d2i = 1.0 / (det * det + float(f32(1e-7)))
    ga = d2i * (-cc * cc * gA + cb * cc * gB - cb * cb * gC)
    gb = d2i * (2 * cb * cc * gA - (det + 2 * cb * cb) * gB + 2 * ca * cb * gC)
    gc = d2i * (-cb * cb * gA + ca * cb * gB - ca * ca * gC)
    want = np.array([T00 * T00 * ga, T00 * T11 * gb, 0.0, T11 * T11 * gc, 0.0, 0.0])
    np.testing.assert_allclose(ref["cov3D"].v, want, rtol=1e-9, atol=0)
    exact = want * (det * det + float(f32(1e-7))) / (det * det)
    assert np.all(np.abs(ref["cov3D"].v[[0, 1, 3]]) < 0.2 * np.abs(exact[[0, 1, 3]]))


def test_oracle_sh_colour32_matches_forward_oracle():
    """sh_colour32's value is the forward oracle's colour to fp32 rounding, and exact bits on dyadic inputs"""
    rng = np.random.default_rng(8)
    for deg in range(4):
        n, M = 500, (deg + 1) ** 2
        d = rng.normal(size=(n, 3)).astype(f32)
        sh = rng.uniform(-1, 1, (n, M, 3)).astype(f32)
        col = B.sh_colour32(deg, sh, d)
        ref, _ = O.color_from_sh(deg, torch.as_tensor(d).double(), torch.zeros(3, dtype=torch.float64),
                                 torch.as_tensor(sh).double())
        raw = ref.numpy()
        ok = raw > 0.01
        np.testing.assert_allclose(col[ok], raw[ok], rtol=2e-6, atol=2e-7)
    d = np.array([[0, 0, 1]], f32)
    sh = np.zeros((1, 1, 3), f32); sh[0, 0] = (-0.5 / B.SH_C0, 0, 1)
    col = B.sh_colour32(0, sh, d)[0]
    assert col[1] == f32(0.5) and col[2] == f32(0.5) + f32(B.SH_C0)
