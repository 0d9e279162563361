"""CPU half of the forward-preprocess edge suite (tests/test_gpu_preprocess_forward_edges.py): the premise of every GPU
scene -- that it reaches the edge it is named for -- and the fp32 oracle's record floats held to a float64 evaluation
of the same chain.

The float64 evaluation (`record64`) restates the kernel's chain operation by operation on the fp32 inputs, with the
kernel's fp32 literals (0.2f, 1e-7f, 0.3f, 1.3f tanfov, the SH constants, L2E) as exact inputs and its discrete
decisions (frustum clamp side, visibility) taken from fp32, using `gs_bwd_oracle.E`: every value carries a first-order
bound e on |fp32 evaluation - exact value|.  Each operation adds u |result| (u = 2^-24, round to nearest) to the
propagated bounds of its operands: a +- b: ea + eb; a b: |a| eb + |b| ea + ea eb; a / b: (ea + |a / b| eb) /
(|b| - eb); sqrt(a): ea / (2 sqrt(a)).  Unrolled, e is k u times the sum of |terms| of the chain (k the depth of the
term), so an FMA, which drops roundings, only tightens it.  A record float r passes when |r - v| <= BAR_K e with
BAR_K = 2, room for the second-order terms the first-order bound drops; a value and bound that are both 0 must be 0.
Results in fp32's underflow range carry an absolute error of up to 2^-150 per operation instead, amplified by the
rest of the chain; there (|v| < 2^-100, e.g. b' of a Gaussian whose scale is 1e-20) the bar is 2^-100 absolute.  The
clamped colour passes when the unclamped fp32 colour passes and the clamp wrote 0 exactly where it is <= 0.  Only visible records with finite values are held to the bar; the GPU tests pin the others bit for
bit."""
import math

import numpy as np
import pytest

from oracle import gs_bwd_oracle as B
import test_gpu_preprocess_forward_edges as F

f32 = np.float32
K = B._c
TINY = 2.0 ** -100          # below this the operands underflow (absolute error 2^-150 per operation, not u |result|)


# ---------------------------------------------------------------------------------------------------------------------
# premises
# ---------------------------------------------------------------------------------------------------------------------
def _tz32(st, means):
    return B.view_t32(st.viewmatrix.numpy().astype(f32).reshape(16), means)[2]


def _hw32(st, means):
    p = st.projmatrix.numpy().astype(f32).reshape(16)
    x, y, z = (np.asarray(means, f32)[:, i] for i in range(3))
    return p[3] * x + p[7] * y + p[11] * z + p[15]


def test_f1_premise():
    cl, (st, st_hw) = F.f1_scene()
    tz = _tz32(st, cl["means3D"])
    radii = F.fwd_pre(cl, st)["radii"].numpy()
    for k in F.F1_ULPS:
        t = F.ulps_from(f32(0.2), k)
        hit = tz == t
        assert hit.any(), f"no t.z at 0.2f {k:+d} ulps"
        if k <= 0:
            assert np.all(radii[hit] == 0), "t.z <= 0.2f is culled"
        else:
            assert np.any(radii[hit] > 0), "t.z one ulp above 0.2f is kept"
    assert F.ulps_from(f32(0.2), -1) < f32(0.2) < F.ulps_from(f32(0.2), 1)
    # the second view: hw exactly 0, and hw + 1e-7f within 2^-28 of 0 on both sides, in front of the near plane
    hw = _hw32(st_hw, cl["means3D"])
    front = _tz32(st_hw, cl["means3D"]) > f32(0.2)
    assert np.any((hw == 0) & front)
    s = hw + f32(1e-7)
    for sign in (1, -1):
        assert np.any((sign * s > 0) & (sign * s <= 2.0 ** -28) & front), "hw + 1e-7f within 2^-28 of 0"
    with np.errstate(all="ignore"):
        ndc = np.abs(F.fwd_pre(cl, st_hw)["xy"].detach().numpy())
    assert np.any(ndc[front & (np.abs(s) < 1e-6)] > 1e6), "pw in the millions"
    # centres thousands of pixels off-screen whose squares reach the frame
    p = F.fwd_pre(cl, st)
    xy = p["xy"].detach().numpy()
    off = (np.abs(xy[:, 0] - st.image_width / 2) > 1000) | (np.abs(xy[:, 1] - st.image_height / 2) > 1000)
    assert np.sum(off & (radii > 0)) >= 4, "visible Gaussians centred > 1000 px off-screen"
    assert np.any(off & (radii == 0)), "and some whose squares miss the frame"


def test_f2_premise():
    cl, (st,), kinds = F.f2_scene()
    lims = F.f2_limits(st)
    m = st.viewmatrix.numpy().astype(f32).reshape(16)
    tx, ty, tz = B.view_t32(m, cl["means3D"])
    with np.errstate(all="ignore"):
        ratio = (tx / tz, ty / tz)
    inx, iny = B.clamp_masks32(m, cl["means3D"], st.tanfovx, st.tanfovy)
    have = set()
    for i, kd in enumerate(kinds):
        if kd[0] in (0, 1):
            axis, sign, k = kd
            assert ratio[axis][i] == F.ulps_from(f32(sign * lims[axis]), sign * k), (i, kd)
            assert (inx, iny)[axis][i] == (k <= 0), (i, kd)
            have.add(kd)
        elif kd[0] == "corner":
            assert ratio[0][i] == kd[1] * lims[0] and ratio[1][i] == kd[2] * lims[1], (i, kd)
            assert inx[i] and iny[i]
            have.add(kd[:1])
        else:
            assert not inx[i] and not iny[i], "both axes clamp"
            have.add(kd[:1])
    assert {(a, s, k) for a in (0, 1) for s in (1, -1) for k in F.F2_KS} | {("corner",), ("out",)} <= have
    radii = F.fwd_pre(cl, st)["radii"].numpy()
    corner = np.array([kd[0] in ("corner", "out") for kd in kinds])
    assert np.all(radii[corner] > 0) and np.mean(radii > 0) > 0.9, "the clamped footprints reach the frame"


def test_f3_premise():
    for mod in F.F3_MODS:
        cl, (st, _) = F.f3_sr_scene(mod)
        assert st.scale_modifier == mod
        p = F.fwd_pre(cl, st)
        radii = p["radii"].numpy()
        c2 = p["cov2d"].detach().numpy().astype(f32)
        tiny = np.all(cl["scales"] * f32(mod) < 1e-15, axis=1)
        assert tiny.sum() >= 5
        assert np.all(c2[tiny, 0] == f32(0.3)) and np.all(c2[tiny, 2] == f32(0.3)), \
            "scale 1e-20: the diagonal of cov2D is exactly the 0.3 dilation"
        assert np.any((c2[tiny, 1] != 0) & (np.abs(c2[tiny, 1]) < np.finfo(f32).tiny)), "and its b a denormal"
        cov = F.cov3d32(cl, mod)
        over = ~np.isfinite(cov).all(1)
        assert over.any() and np.any(over & (radii == 0)), "an overflowed covariance is culled"
        assert np.any(~np.isfinite(c2).all(1)), "cov2D overflows"
        qn = np.linalg.norm(cl["rotations"].astype(np.float64), axis=1)
        ok = np.isfinite(cov).all(1) & ~tiny
        for v in (0.0, 1e-3, 30.0):
            sel = np.isclose(qn, v, rtol=1e-5, atol=0) & ok
            assert sel.any() and np.any(radii[sel] > 0), f"a visible Gaussian with |q| = {v}"
    cl, (st,), kind = F.f3_precomp_scene()
    p = F.fwd_pre(cl, st)
    radii = p["radii"].numpy()
    c2 = p["cov2d"].detach().numpy().astype(f32)
    det = c2[:, 0] * c2[:, 2] - c2[:, 1] * c2[:, 1]
    for i, k in enumerate(kind):
        if k == "zero":
            assert det[i] == 0 and radii[i] == 0, "fp32 det exactly 0 is culled"
        elif k in (-3, -2, -1, 1, 2, 3):
            assert det[i] != 0 and abs(det[i]) < 1e-6 and radii[i] > 0, (k, det[i])
        elif k == "indefinite":
            assert radii[i] > 0 and det[i] < 0
        elif k == "negative":
            assert radii[i] == 0
        elif isinstance(k, float):
            assert radii[i] > 0 and abs(det[i] - k) < 0.2 * k
    assert sum(k in (-3, -2, -1, 1, 2, 3) for k in kind) == 6


def test_f4_premise():
    for deg, M in F.f4_cases():
        cl, (st,) = F.f4_sh_scene(deg, M)
        raw = B.sh_colour32(deg, cl["shs"], cl["means3D"] - F.cam32(st)[None])
        n = len(raw) - 4
        assert np.any(raw[:n] == 0) and np.any((raw[:n] < 0) & (raw[:n] > -1e-6)) and np.any((raw[:n] > 0) & (raw[:n] < 1e-6))
        assert not np.any(np.signbit(raw[np.isfinite(raw)]) & (raw[np.isfinite(raw)] == 0)), "no -0 colour from SH"
        nb = (deg + 1) ** 2
        if M > nb:
            assert np.isnan(cl["shs"][n, M - 1, 0]) and np.array_equal(raw[n], raw[0]), "a NaN above the degree is ignored"
        assert np.isnan(raw[n + 1, 1]) and F.fmax0(raw)[n + 1, 1] == 0, "an active NaN: colour NaN, clamped to 0"
        assert raw[n + 2, 2] == np.inf and raw[n + 3, 0] == -np.inf
        assert np.all(F.fwd_pre(cl, st)["radii"].numpy() > 0)
    # x + 0.5f is -0 only for x = -0.5f exactly, whose sum is +0: the SH colour is never -0
    x = np.nextafter(f32(-0.5), f32(0)) + np.arange(-3, 4).astype(f32) * f32(2 ** -25)
    assert not np.any(np.signbit(x + f32(0.5)) & (x + f32(0.5) == 0))
    assert not np.signbit(f32(-0.5) + f32(0.5))
    cl, (st,) = F.f4_colour_scene()
    col = cl["colors_precomp"]
    assert np.any((col == 0) & np.signbit(col)) and np.any((col == 0) & ~np.signbit(col))
    assert np.isnan(col).any() and np.isposinf(col).any() and np.isneginf(col).any()
    assert np.any((col != 0) & (np.abs(col) < np.finfo(f32).tiny)), "denormal colours"
    assert np.all(F.fwd_pre(cl, st)["radii"].numpy() > 0)


def test_f5_premise():
    assert set(F.F5_N) >= {1, 127, 128, 129, 4097} and set(F.F5_V) >= {1, 8, 9, 16, 17}
    for N in (129, 4097):
        cl, sts = F.f5_scene(N, 17)
        vis = np.stack([F.fwd_pre(cl, st)["radii"].numpy() > 0 for st in sts])
        assert not vis[1].any(), "view 1 sees nothing"
        nv = vis.sum(0)
        assert ((nv > 0) & (nv < len(sts))).any()
        assert np.any(cl["colors_precomp"] < 0), "negative precomputed colours pass unclamped"
    # 128-Gaussian CTAs: 127 and 129 leave a partial tail CTA, 128 none, 4097 a one-Gaussian tail
    assert [n % 128 for n in F.F5_N] == [1, 127, 0, 1, 1]


# ---------------------------------------------------------------------------------------------------------------------
# the fp32 oracle's record floats against float64
# ---------------------------------------------------------------------------------------------------------------------
def record64(cl, st, cov=None):
    """float64 values with fp32 error bounds (gs_bwd_oracle.E) of px, py, depth, a', b', c' and the unclamped SH colour"""
    m = [float(v) for v in st.viewmatrix.numpy().astype(f32).reshape(16)]
    p = [float(v) for v in st.projmatrix.numpy().astype(f32).reshape(16)]
    mu = np.asarray(cl["means3D"], f32).astype(np.float64)
    x, y, z = B.E(mu[:, 0]), B.E(mu[:, 1]), B.E(mu[:, 2])
    tx = x * m[0] + y * m[4] + z * m[8] + m[12]
    ty = x * m[1] + y * m[5] + z * m[9] + m[13]
    tz = x * m[2] + y * m[6] + z * m[10] + m[14]
    hx = x * p[0] + y * p[4] + z * p[8] + p[12]
    hy = x * p[1] + y * p[5] + z * p[9] + p[13]
    hw = x * p[3] + y * p[7] + z * p[11] + p[15]
    pw = 1.0 / (hw + float(f32(1e-7)))
    W, H = st.image_width, st.image_height
    px = ((hx * pw + 1.0) * float(W) - 1.0) * 0.5
    py = ((hy * pw + 1.0) * float(H) - 1.0) * 0.5
    if cov is None and cl.get("cov3D_precomp") is not None:
        cov = cl["cov3D_precomp"]
    if cov is not None:
        c = [B.E(np.asarray(cov, f32)[:, k].astype(np.float64)) for k in range(6)]
    else:
        c, _, _ = B._cov3d_fwd(np.asarray(cl["scales"], f32).astype(np.float64),
                               np.asarray(cl["rotations"], f32).astype(np.float64), float(f32(st.scale_modifier)))
    limx, limy = F.f2_limits(st)
    tfx, tfy = f32(st.tanfovx), f32(st.tanfovy)
    fx, fy = float(f32(W) / (f32(2) * tfx)), float(f32(H) / (f32(2) * tfy))
    tx32, ty32, tz32 = B.view_t32(np.array(m, f32), cl["means3D"])
    with np.errstate(all="ignore"):
        rx, ry = tx32 / tz32, ty32 / tz32
    cx = (tx / tz).where((rx >= -limx) & (rx <= limx), np.where(rx > 0, float(limx), -float(limx))) * tz
    cy = (ty / tz).where((ry >= -limy) & (ry <= limy), np.where(ry > 0, float(limy), -float(limy))) * tz
    J00, J02 = K(fx) / tz, -(cx * fx) / (tz * tz)
    J11, J12 = K(fy) / tz, -(cy * fy) / (tz * tz)
    T00, T01, T02 = J00 * m[0] + J02 * m[2], J00 * m[4] + J02 * m[6], J00 * m[8] + J02 * m[10]
    T10, T11, T12 = J11 * m[1] + J12 * m[2], J11 * m[5] + J12 * m[6], J11 * m[9] + J12 * m[10]
    v00, v01, v02 = c[0] * T00 + c[1] * T01 + c[2] * T02, c[1] * T00 + c[3] * T01 + c[4] * T02, c[2] * T00 + c[4] * T01 + c[5] * T02
    v10, v11, v12 = c[0] * T10 + c[1] * T11 + c[2] * T12, c[1] * T10 + c[3] * T11 + c[4] * T12, c[2] * T10 + c[4] * T11 + c[5] * T12
    ca = T00 * v00 + T01 * v01 + T02 * v02 + float(f32(0.3))
    cb = T00 * v10 + T01 * v11 + T02 * v12
    cc = T10 * v10 + T11 * v11 + T12 * v12 + float(f32(0.3))
    det_inv = 1.0 / (ca * cc - cb * cb)
    out = dict(px=px, py=py, depth=tz, a=(cc * det_inv) * float(F.HALF_L2E), b=(cb * det_inv) * float(F.L2E),
               c=(ca * det_inv) * float(F.HALF_L2E))
    if cl.get("shs") is not None:
        cam = [float(v) for v in F.cam32(st)]
        vx, vy, vz = x - cam[0], y - cam[1], z - cam[2]
        inv = 1.0 / B.sqrt(vx * vx + vy * vy + vz * vz)
        bas = B._sh_basis(st.sh_degree, vx * inv, vy * inv, vz * inv)[0]
        sh = np.asarray(cl["shs"], f32).astype(np.float64)
        rgb = []
        for ch in range(3):
            acc = B.zeros(len(mu))
            for k, bk in enumerate(bas):
                acc = acc + bk * sh[:, k, ch]
            rgb.append(acc + 0.5)
        out["rgb"] = rgb
    return out


def _hold(tag, got, ref):
    """|got - v| <= BAR_K e; 0 where v and e are both 0; within TINY of v where |v| < TINY.  Returns the worst
    |got - v| / e."""
    g = np.asarray(got, np.float64)
    with np.errstate(all="ignore"):
        d = np.abs(g - ref.v)
        bar = B.BAR_K * ref.e
        ok = (d <= bar) | ((ref.e == 0) & (d == 0)) | ((np.abs(ref.v) < TINY) & (d < TINY))
    bad = np.flatnonzero(~ok)
    assert bad.size == 0, f"{tag}: row {bad[0]} fp32 {g[bad[0]]!r} float64 {ref.v[bad[0]]!r} bound {ref.e[bad[0]]!r}"
    with np.errstate(all="ignore"):
        r = np.where(ref.e > 0, d / ref.e, 0)
    return float(r.max()) if r.size else 0.0


def _scenes():
    out = [("F1", *F.f1_scene()), ("F2", *F.f2_scene()[:2]), ("F3 precomp", *F.f3_precomp_scene()[:2]),
           ("F4 colours", *F.f4_colour_scene())]
    out += [(f"F3 mod {mod}", *F.f3_sr_scene(mod)) for mod in F.F3_MODS]
    out += [(f"F4 deg {d} M {M}", *F.f4_sh_scene(d, M)) for d, M in F.f4_cases()]
    out += [(f"F5 N {n}", *F.f5_scene(n, 9)) for n in (129, 4097)]
    return out


@pytest.mark.filterwarnings("ignore::RuntimeWarning")
@pytest.mark.parametrize("i", range(4 + len(F.F3_MODS) + len(F.f4_cases()) + 2))
def test_oracle_record_floats_within_float64_bound(i):
    tag, cl, sts = _scenes()[i]
    worst, nlive = 0.0, 0
    for v, st in enumerate(sts):
        rec = F.expected(cl, st).view(f32)
        ref = record64(cl, st)
        with np.errstate(all="ignore"):
            live = (rec[:, 3].view(np.int32) > 0) & np.isfinite(rec[:, :11]).all(1)
            if cl.get("shs") is not None:
                live &= np.isfinite(B.sh_colour32(st.sh_degree, cl["shs"], cl["means3D"] - F.cam32(st)[None])).all(1)
        sub = lambda e: B.E(e.v[live], e.e[live])                  # noqa: E731
        for j, key in zip((0, 1, 2, 4, 5, 6), ("px", "py", "depth", "a", "b", "c")):
            worst = max(worst, _hold(f"{tag} view {v} {key}", rec[live, j], sub(ref[key])))
        if "rgb" in ref:
            raw = B.sh_colour32(st.sh_degree, cl["shs"], cl["means3D"] - F.cam32(st)[None])[live]
            for ch in range(3):
                r = sub(ref["rgb"][ch])
                worst = max(worst, _hold(f"{tag} view {v} rgb[{ch}] before the clamp", raw[:, ch], r))
                clamped = raw[:, ch] <= 0
                assert np.all(rec[live, 8 + ch][clamped] == 0) and np.all(rec[live, 8 + ch][~clamped] == raw[~clamped, ch])
        nlive += int(live.sum())
    assert nlive > 0 or tag.startswith("F4 colours")
    print(tag, "worst |fp32 - float64| / bound:", f"{worst:.3g}")


def test_record64_quirks():
    """on the optical axis with an isotropic scale s: px = (W - 1) / 2, a' = -0.5 L2E / (fx^2 s^2 / tz^2 + 0.3), b' = 0"""
    st = F.settings(64, 48, 0)
    tz = 1.25
    s = 0.01
    cl = {"means3D": np.array([[0, 0, 1.75 - tz]], f32), "scales": np.full((1, 3), s, f32),
          "rotations": np.array([[1, 0, 0, 0]], f32), "opacities": np.ones((1, 1), f32), "shs": np.zeros((1, 1, 3), f32)}
    ref = record64(cl, st)
    fx = float(f32(64) / (f32(2) * f32(st.tanfovx)))
    A = fx * fx * float(f32(s)) ** 2 / tz ** 2 + float(f32(0.3))
    assert math.isclose(float(ref["a"].v[0]), float(F.HALF_L2E) / A, rel_tol=1e-12)
    assert abs(float(ref["b"].v[0])) <= 2 * float(ref["b"].e[0])
    assert math.isclose(float(ref["px"].v[0]), 31.5, rel_tol=1e-6)
    rec = F.expected(cl, st).view(f32)[0]
    assert rec[4] == f32(F.HALF_L2E) * f32(rec[4] / F.HALF_L2E) and rec[5] == 0
    assert rec[8] == rec[9] == rec[10] == f32(0.5)
