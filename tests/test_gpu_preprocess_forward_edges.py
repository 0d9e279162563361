"""Forward preprocess (csrc/gs_preprocess.cu): every float of the 48-byte splat record against the fp32 oracle, bit for
bit, at the edges where it goes wrong: the near plane and projections thousands of pixels off-screen (F1), the
1.3 tanfov frustum clamp on each axis and at the corners (F2), covariances from scales of 1e-20 to overflow, scale
modifiers, unnormalised and zero quaternions and precomputed matrices whose 2D determinant is 0, a few ulps from 0 or
negative (F3), the SH colour at every degree and coefficient count with colours exactly on 0 and an ulp either side,
and precomputed colours that are -0, negative, NaN or infinite (F4), and the launch shape: 1 to 4097 Gaussians,
1 to 17 views, SH rows that are not 16-byte aligned (F5).  Every scene has a CPU test of its premise in
tests/test_preprocess_forward_edges_cpu.py, which also holds the fp32 oracle's record floats to a float64 evaluation
of the same chain within a derived bound, so bit equality with the oracle here also means the records are right.

Three kernels write records, and each scene runs through every one that accepts it:
  * `preprocess_kernel`, the one-view path of `GaussianRasterizer` (`forward_with_state`'s `recs`), with SH, with
    precomputed colours and with precomputed covariances;
  * `preprocess_multi_kernel`, the step entries' batched preprocess (`gs_b200_debug_preprocess_views`, the step's own
    chunks), with SH and with precomputed colours;
  * its colour-free pass followed by `sh_colour_multi_kernel`, as the host-buffer step runs them.
The expected record of a view (`expected`): px, py and depth are the oracle's; the conic is f32(-0.5 L2E) conA,
L2E (-conB), f32(-0.5 L2E) conC with L2E the kernel's fp32 literal of log2(e) (the kernel's constant folding);
opacity is the input; rgb is `gs_bwd_oracle.sh_colour32` (the kernel's fp32 SH arithmetic) after fmaxf(., 0), or the
precomputed colour unclamped; the radius and tiles_touched words are the oracle's integers; a culled record is all
zero bits.  Values must match bit for bit, where a NaN matches any NaN (payloads are platform-dependent).  With tile
culling off every path's tiles_touched is the square's; with it on (the one-view path in mode 2, the step by default)
the float words must not move and tiles_touched is the binning's culled count.  Two runs must give the same bits."""
import ctypes as C
import dataclasses
import math
from functools import lru_cache

import numpy as np
import pytest
import torch

from oracle import gs_bwd_oracle as B
from oracle import gs_oracle as O

f32 = np.float32
FOVY = 49.1
L2E = f32(1.4426950408889634)
HALF_L2E = f32(-0.5) * L2E                 # exact: the kernel's folded -0.5f * L2E
WORDS = ("px", "py", "depth", "radius", "a'", "b'", "c'", "opacity", "r", "g", "b", "tiles")


# ---------------------------------------------------------------------------------------------------------------------
# scene helpers (shared with the CPU premise tests)
# ---------------------------------------------------------------------------------------------------------------------
def settings(W, H, deg, radius=1.75, elev=0.0, azim=0.0, mod=1.0, target=None):
    return O.minicam_settings(O.orbit_camera(elev, azim, radius, target=target), W, H, FOVY, sh_degree=deg,
                              scale_modifier=mod)


def cam32(st):
    return st.campos.numpy().astype(f32)


def walk(f, x0, target, steps=256):
    """fp32 x near x0 with f(x) == target, nearest first; None when no x within `steps` ulps does"""
    x0 = f32(x0)
    up, dn = x0, x0
    for _ in range(steps):
        for x in (up, dn):
            if f(x) == target:
                return x
        up, dn = np.nextafter(up, f32(np.inf)), np.nextafter(dn, f32(-np.inf))
    return None


def ulps_from(x, k):
    """x moved k ulps (k < 0: down)"""
    x = f32(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, f32(np.inf if k > 0 else -np.inf))
    return x


def fwd_pre(cl, st, cov=None):
    """the fp32 forward oracle; `cov` replaces scales / rotations by precomputed covariances"""
    t = lambda k: None if cl.get(k) is None else torch.as_tensor(np.ascontiguousarray(cl[k]))       # noqa: E731
    shs = t("shs")
    if shs is None and cl.get("colors_precomp") is None:
        shs = torch.zeros(len(cl["means3D"]), 1, 3)
    cov3 = t("cov3D_precomp") if cov is None else torch.as_tensor(cov)
    sc, ro = (None, None) if cov3 is not None else (t("scales"), t("rotations"))
    with np.errstate(all="ignore"):
        return O.preprocess(t("means3D"), sc, ro, t("opacities"), shs, t("colors_precomp"), cov3, None, st)


def cov3d32(cl, mod):
    """the kernel's fp32 covariance of scales / rotations (the oracle's restatement, same order)"""
    with np.errstate(all="ignore"):
        return O.cov3d_from_scale_rot(torch.as_tensor(cl["scales"]), torch.as_tensor(cl["rotations"]),
                                      mod).numpy().astype(f32)


def fmax0(x):
    """fmaxf(x, 0.f): NaN gives 0; x + 0.5f is never -0 in round-to-nearest, so the sign of a zero never arises"""
    return np.where(x > 0, x, f32(0)).astype(f32)


def sh_rgb32(cl, st):
    """the kernel's clamped SH colour for view st"""
    return fmax0(B.sh_colour32(st.sh_degree, cl["shs"], cl["means3D"].astype(f32) - cam32(st)[None]))


def expected(cl, st, colours=False, cov=None):
    """[N, 12] uint32: the record every path must write for view st (tile culling off).  colours: the precomputed-colour
    path; cov: the precomputed-covariance path with these covariances"""
    use = dict(cl)
    if colours:
        use.pop("shs", None)
    else:
        use.pop("colors_precomp", None)
    p = fwd_pre(use, st, cov)
    N = len(cl["means3D"])
    vis = p["radii"].numpy() > 0
    rec = np.zeros((N, 12), f32)
    with np.errstate(all="ignore"):
        rec[:, 0:2] = p["xy"].detach().numpy().astype(f32)
        rec[:, 2] = p["depth"].detach().numpy().astype(f32)
        rec[:, 3] = p["radii"].numpy().astype(np.int32).view(f32)
        con = p["conic"].detach().numpy().astype(f32)
        rec[:, 4] = HALF_L2E * con[:, 0]
        rec[:, 5] = L2E * -con[:, 1]
        rec[:, 6] = HALF_L2E * con[:, 2]
        rec[:, 7] = np.asarray(cl["opacities"], f32).reshape(-1)
        rec[:, 8:11] = np.asarray(cl["colors_precomp"], f32) if colours else sh_rgb32(cl, st)
        rec[:, 11] = p["tiles_touched"].numpy().astype(np.uint32).view(f32)
    rec[~vis] = 0
    return rec.view(np.uint32)


def same_bits(got, want):
    """[..., 12] uint32: equal bits, or NaN in both"""
    g, w = got.view(f32), want.view(f32)
    return (got == want) | (np.isnan(g) & np.isnan(w))


def assert_records(tag, got, want, words=range(12)):
    words = list(words)
    ok = same_bits(got[:, words], want[:, words])
    if ok.all():
        return
    bad = np.argwhere(~ok)
    lines = []
    for i, j in bad[:6]:
        k = words[j]
        lines.append(f"Gaussian {i} {WORDS[k]}: got {got[i, k].view(f32)!r} ({got[i, k]:#010x}), "
                     f"want {want[i, k].view(f32)!r} ({want[i, k]:#010x})")
    raise AssertionError(f"{tag}: {len(bad)} record words differ from the fp32 oracle\n  " + "\n  ".join(lines))


def views_of(sts):
    v = np.zeros((len(sts), 40), f32)
    for i, st in enumerate(sts):
        v[i, :16] = st.viewmatrix.numpy().reshape(16); v[i, 16:32] = st.projmatrix.numpy().reshape(16)
        v[i, 32:35] = st.campos.numpy(); v[i, 35:38] = st.bg.numpy()
        v[i, 38], v[i, 39] = st.tanfovx, st.tanfovy
    return v


# ---------------------------------------------------------------------------------------------------------------------
# F1 near plane and projection.  Camera 0.25 from the origin on +z (axis-aligned view matrix: t is exact in any
# contraction), so t.z = 0.25 - z reaches every fp32 value near 0.2.  A second view's projection matrix is shifted so
# that hw = t.z - 0.21: hw is 0 and within 2^-28 of -1e-7f (pw ~ 1e7 and ~ +-3e8) in front of the
# near plane.
# ---------------------------------------------------------------------------------------------------------------------
F1_ULPS = (-3, -2, -1, 0, 1, 2, 3)
F1_OFF = (15.0, 40.0, 100.0)                 # t.x / t.z in units of tanfovx: centres 7 to 50 frame widths off


def f1_hw_view(st):
    p = st.projmatrix.clone()
    p[3, 3] = float(f32(p[3, 3].item()) - f32(0.21))
    return dataclasses.replace(st, projmatrix=p)


@lru_cache(None)
def f1_scene():
    W, H, deg = 64, 48, 1
    st = settings(W, H, deg, radius=0.25)
    m = st.viewmatrix.numpy().astype(f32).reshape(16)
    tz_of = lambda z: B.view_t32(m, np.array([[0, 0, z]], f32))[2][0]      # noqa: E731
    st_hw = f1_hw_view(st)
    ph = st_hw.projmatrix.numpy().astype(f32).reshape(16)
    hw_of = lambda z: (ph[3] * f32(0) + ph[7] * f32(0)) + ph[11] * f32(z) + ph[15]      # noqa: E731
    rng = np.random.default_rng(11)
    rows = []
    for k in F1_ULPS:
        t = ulps_from(f32(0.2), k)
        z = walk(tz_of, 0.25 - float(t), t)
        for sx in (1e-4, 0.004, 0.05):
            for lat in ((0.0, 0.0), tuple(rng.uniform(-0.6, 0.6, 2))):
                rows.append((lat[0] * float(t) * st.tanfovx, lat[1] * float(t) * st.tanfovy, z, sx))
    zs = [walk(hw_of, 0.04 - float(hw), hw, 4096) for hw in (f32(0.0), f32(1e-7), f32(1e-6))]
    # hw is a multiple of 2^-28 here, so hw + 1e-7f is not exactly 0: the nearest hw on either side of -1e-7f
    cand = [ulps_from(f32(0.04 + 1e-7), k) for k in range(-64, 65)]
    near = cand[int(np.argmin([abs(float(hw_of(z)) + float(f32(1e-7))) for z in cand]))]
    zs += [ulps_from(near, k) for k in (-1, 0, 1)]
    for z in zs:                             # the second view's hw; t.z = hw + 0.21
        rows.append((0.0, 0.0, z, 0.01))
        rows.append((1e-3, -1e-3, z, 0.01))
    tz = 1.0
    for k in F1_OFF:                          # off-screen centres whose squares reach back into the frame
        for sgn in (1, -1):
            for sx in (3.0, 30.0, 300.0):
                rows.append((sgn * k * st.tanfovx * tz, 0.1, 0.25 - tz, sx))
                rows.append((0.05, sgn * k * st.tanfovy * tz, 0.25 - tz, sx))
    rows = np.array(rows, np.float64)
    n = len(rows)
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    cl = {"means3D": rows[:, :3].astype(f32), "scales": (rows[:, 3:4] * rng.uniform(0.5, 1.5, (n, 3))).astype(f32),
          "rotations": q.astype(f32), "opacities": rng.uniform(0.05, 1, (n, 1)).astype(f32),
          "shs": rng.uniform(-0.5, 0.5, (n, 4, 3)).astype(f32), "colors_precomp": rng.uniform(-0.2, 1.2, (n, 3)).astype(f32)}
    return cl, [st, st_hw]


# ---------------------------------------------------------------------------------------------------------------------
# F2 frustum clamp.  t.x / t.z (and t.y / t.z) at +-1.3 tanfov exactly as fp32 computes it and one ulp either side,
# on both axes; corners where both axes sit on the limit or both clamp.
# ---------------------------------------------------------------------------------------------------------------------
F2_KS = (-1, 0, 1)              # one ulp inside, on the limit, one ulp outside


def f2_limits(st):
    return f32(1.3) * f32(st.tanfovx), f32(1.3) * f32(st.tanfovy)


def _ratio_fn(m, axis, z, other=0.0):
    def ratio(c):
        p = np.zeros((1, 3), f32); p[0, 2] = z; p[0, axis] = c; p[0, 1 - axis] = other
        t = B.view_t32(m, p)
        return (t[axis] / t[2])[0]
    return ratio


def _on_ratio(m, axis, z, target, other=0.0):
    tz = B.view_t32(m, np.array([[0, 0, z]], f32))[2][0]
    c0 = float(target) * float(tz) * (1 if axis == 0 else -1)
    return walk(_ratio_fn(m, axis, z, other), c0, target, 512)


@lru_cache(None)
def f2_scene():
    W, H, deg = 64, 48, 2
    st = settings(W, H, deg)
    m = st.viewmatrix.numpy().astype(f32).reshape(16)
    lims = f2_limits(st)
    rng = np.random.default_rng(12)
    rows, kinds = [], []
    for axis in (0, 1):
        for sign in (1, -1):
            for k in F2_KS:
                target = ulps_from(f32(sign * lims[axis]), sign * k)
                for z in (0.5, 0.75, -0.25):
                    c = _on_ratio(m, axis, z, target)
                    if c is not None:
                        p = [0.0, 0.0, z]; p[axis] = c; p[1 - axis] = rng.uniform(-0.1, 0.1)
                        rows.append(p); kinds.append((axis, sign, k))
                        break
    for sx in (1, -1):                          # corners: both ratios on the limit, then both well outside
        for sy in (1, -1):
            z = 0.5
            cx = _on_ratio(m, 0, z, f32(sx * lims[0]))
            cy = _on_ratio(m, 1, z, f32(sy * lims[1]), other=cx)
            rows.append([cx, cy, z]); kinds.append(("corner", sx, sy))
            tz = 1.25
            rows.append([sx * 1.6 * float(lims[0]) * tz, -sy * 1.6 * float(lims[1]) * tz, z]); kinds.append(("out", sx, sy))
    rows = np.array(rows, f32)
    n = len(rows)
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    far = np.array([k[0] == "out" for k in kinds])
    scl = np.where(far[:, None], 0.6, 0.1) * rng.uniform(0.6, 1.4, (n, 3))
    cl = {"means3D": rows, "scales": scl.astype(f32), "rotations": q.astype(f32),
          "opacities": rng.uniform(0.05, 1, (n, 1)).astype(f32), "shs": rng.uniform(-0.5, 0.5, (n, 9, 3)).astype(f32),
          "colors_precomp": rng.uniform(-0.2, 1.2, (n, 3)).astype(f32)}
    return cl, [st], kinds


# ---------------------------------------------------------------------------------------------------------------------
# F3 covariance.  Scales from 1e-20 (cov2D is the 0.3 dilation, bit for bit) to 1e30 (s^2 overflows), per axis and
# isotropic, with unit, zero, tiny and large quaternions; scale modifiers 0.37 / 1 / 3; seen axis-aligned and
# obliquely (every term of the EWA sums non-zero).  Precomputed covariances on the optical axis with
# cov2D = [[0.3, x], [x, 0.3]] and fp32 det exactly 0, a few ulps from 0 and ~1e-4, plus an indefinite and a
# negative-definite matrix.
# ---------------------------------------------------------------------------------------------------------------------
F3_SCALES = (1e-20, 1e-12, 1e-6, 1e-3, 0.03, 1.0, 1e3, 1e8, 1e15, 1e18, 1.8e19, 3e19, 1e20, 1e30)
F3_MODS = (0.37, 1.0, 3.0)


@lru_cache(None)
def f3_sr_scene(mod):
    W, H, deg = 64, 48, 1
    st = settings(W, H, deg, mod=mod)
    rng = np.random.default_rng(13)
    quats = [np.array([1, 0, 0, 0], f32), np.zeros(4, f32)]
    for norm in (1.0, 1e-3, 30.0):
        q = rng.normal(size=4); quats.append((q / np.linalg.norm(q) * norm).astype(f32))
    rows = []
    for s in F3_SCALES:
        for q in quats:
            for shape in ((1, 1, 1), (1, 1e-3, 0.3)):
                rows.append((np.array(shape) * s / mod, q))
    n = len(rows)
    means = np.stack([rng.uniform(-0.4, 0.4, n), rng.uniform(-0.3, 0.3, n), rng.uniform(-0.3, 0.3, n)], 1)
    cl = {"means3D": means.astype(f32), "scales": np.array([r[0] for r in rows]).astype(f32),
          "rotations": np.array([r[1] for r in rows], f32), "opacities": rng.uniform(0.05, 1, (n, 1)).astype(f32),
          "shs": rng.uniform(-0.5, 0.5, (n, 4, 3)).astype(f32), "colors_precomp": rng.uniform(-0.2, 1.2, (n, 3)).astype(f32)}
    return cl, [st, settings(W, H, deg, elev=17.0, azim=31.0, mod=mod)]      # axis-aligned and oblique


F3_DETS = (1e-4, 1e-2, "zero", -3, -2, -1, 1, 2, 3)     # target det, or ulps of b from the det == 0 solution


@lru_cache(None)
def f3_precomp_scene():
    W = H = 64
    st = settings(W, H, 0)
    fx = f32(f32(W) / (f32(2) * f32(st.tanfovx)))
    dep = 1.25
    T = float(fx) / dep
    z = 1.75 - dep

    def det_of(b):
        p = fwd_pre({"means3D": np.array([[0, 0, z]], f32), "opacities": np.ones((1, 1), f32),
                     "colors_precomp": np.zeros((1, 3), f32)}, st, cov=np.array([[0, b, 0, 0, 0, 0]], f32))
        a, bq, c = p["cov2d"].detach().numpy().astype(f32)[0]
        return a * c - bq * bq

    b0 = walk(det_of, f32(-math.sqrt(0.09) / (T * T)), f32(0), 4096)
    covs, kind = [], []
    for tgt in F3_DETS:
        if isinstance(tgt, float):
            b = f32(-math.sqrt(0.09 - tgt) / (T * T))
        else:
            b = b0 if tgt == "zero" else ulps_from(b0, tgt)
        covs.append([0, b, 0, 0, 0, 0]); kind.append(tgt)
    covs += [[0.01, 0, 0, -0.01, 0, 0.01], [-0.01, 0, 0, -0.01, 0, -0.01]]
    kind += ["indefinite", "negative"]
    n = len(covs)
    rng = np.random.default_rng(14)
    m = rng.normal(size=(6, 3, 3)) * 0.02
    g = np.einsum("nij,nkj->nik", m, m)
    covs += np.stack([g[:, 0, 0], g[:, 0, 1], g[:, 0, 2], g[:, 1, 1], g[:, 1, 2], g[:, 2, 2]], 1).tolist()
    kind += ["generic"] * 6
    means = np.concatenate([np.tile(np.array([[0, 0, z]], f32), (n, 1)), rng.uniform(-0.3, 0.3, (6, 3))])
    N = len(covs)
    cl = {"means3D": means.astype(f32), "cov3D_precomp": np.array(covs, f32),
          "opacities": rng.uniform(0.05, 1, (N, 1)).astype(f32), "colors_precomp": rng.uniform(0, 1, (N, 3)).astype(f32),
          "shs": rng.uniform(-0.5, 0.5, (N, 1, 3)).astype(f32)}
    return cl, [st], kind


# ---------------------------------------------------------------------------------------------------------------------
# F4 SH and colour.  The backward suite's SH-clamp scenes (every degree, every M from (deg+1)^2 to 16, colours before
# the clamp at -1e-3, -3 / -1 ulp, exactly 0, +1 / +3 ulp and +1e-3), plus Gaussians with a NaN in an SH row above the
# degree (ignored), a NaN in an active row (colour NaN, clamped to 0) and +-inf in row 0.  Precomputed colours: -0, +0,
# +-denormal, negative, NaN and +-inf, passed through unclamped.
# ---------------------------------------------------------------------------------------------------------------------
def f4_cases():
    import test_gpu_preprocess_backward_edges as S
    return S.S3_CASES


@lru_cache(None)
def f4_sh_scene(deg, M):
    import test_gpu_preprocess_backward_edges as S
    cl, st = S.s3_scene(deg, M)
    cl = {k: v.copy() for k, v in cl.items()}
    nb = (deg + 1) ** 2
    extra = {k: np.repeat(v[:1], 4, 0) for k, v in cl.items()}
    if M > nb:
        extra["shs"][0, M - 1, 0] = np.nan
    extra["shs"][1, nb - 1, 1] = np.nan
    extra["shs"][2, 0, 2] = np.inf
    extra["shs"][3, 0, 0] = -np.inf
    cl = {k: np.concatenate([cl[k], extra[k]]) for k in cl}
    cl["colors_precomp"] = sh_rgb32(cl, st)
    return cl, [st]


F4_COLOURS = (-0.0, 0.0, -1e-45, 1e-45, -1.5e-38, -0.25, 0.75, 3.5, np.nan, np.inf, -np.inf)


@lru_cache(None)
def f4_colour_scene():
    import test_gpu_preprocess_backward_edges as S
    cl, st = S.s3_scene(0, 1)
    n = len(cl["means3D"])
    col = np.array([[F4_COLOURS[(i + 4 * c) % len(F4_COLOURS)] for c in range(3)] for i in range(n)], f32)
    return dict(cl, colors_precomp=col), [st]


# ---------------------------------------------------------------------------------------------------------------------
# F5 launch shape.  N around the 128-Gaussian CTA (the tail CTA re-reads Gaussian N-1 and must not store it), V around
# the step's 16-view chunks (17 views run as 9 + 8), SH rows at a 4-byte offset (gs_stage_rows_in's scalar path).
# ---------------------------------------------------------------------------------------------------------------------
F5_N = (1, 127, 128, 129, 4097)
F5_V = (1, 8, 9, 16, 17)


@lru_cache(None)
def f5_scene(N, V):
    rng = np.random.default_rng(N * 31 + V)
    W, H, deg, M = 48, 32, 3, 16
    sts = [settings(W, H, deg, elev=rng.uniform(-30, 30), azim=360.0 * v / V + rng.uniform(0, 10), mod=0.9)
           for v in range(V)]
    if V > 1:
        sts[1] = settings(W, H, deg, target=np.array([40.0, 0, 0], f32), mod=0.9)        # sees nothing
    means = rng.uniform(-1.0, 1.0, (N, 3))
    means[rng.random(N) < 0.03, 1] += 40.0
    q = rng.normal(size=(N, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    cl = {"means3D": means.astype(f32), "scales": rng.uniform(0.005, 0.08, (N, 3)).astype(f32),
          "rotations": q.astype(f32), "opacities": rng.uniform(0.05, 1, (N, 1)).astype(f32),
          "shs": rng.uniform(-0.5, 0.5, (N, M, 3)).astype(f32), "colors_precomp": rng.uniform(-0.2, 1.2, (N, 3)).astype(f32)}
    return cl, sts


# ---------------------------------------------------------------------------------------------------------------------
# kernel runners
# ---------------------------------------------------------------------------------------------------------------------
def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a, f32)).cuda().contiguous()


def run_one(cl, st, mode, cov=None):
    """preprocess_kernel through GaussianRasterizer's forward: [N, 12] uint32.  mode: "shs" / "colours" / "cov" (cov3D
    precomputed, SH colour); cov: the precomputed covariances"""
    from gs_b200 import rasterizer as R
    rs = R.GaussianRasterizationSettings(st.image_height, st.image_width, st.tanfovx, st.tanfovy, st.bg.cuda(),
                                         st.scale_modifier, st.viewmatrix.cuda(), st.projmatrix.cuda(), st.sh_degree,
                                         st.campos.cuda(), False, False)
    kw = {}
    if mode == "colours":
        kw["colors_precomp"] = _dev(cl["colors_precomp"])
    else:
        kw["shs"] = _dev(cl["shs"])
    if cov is not None:
        kw["cov3D_precomp"] = _dev(cov)
    else:
        kw["scales"], kw["rotations"] = _dev(cl["scales"]), _dev(cl["rotations"])
    out = R.forward_with_state(rs, _dev(cl["means3D"]), _dev(cl["opacities"]), **kw)
    torch.cuda.synchronize()
    return out["recs"].cpu().numpy().view(np.uint32).copy()


def run_multi(cl, sts, mode, misalign=False):
    """the step's batched preprocess: [V, N, 12] uint32.  mode: "shs" / "colours" / "geom" (colour-free pass, then the
    colour pass); misalign: SH rows at a 4-byte offset from a 16-byte boundary"""
    from gs_b200 import _lib
    from gs_b200 import rasterizer as R
    N, V = len(cl["means3D"]), len(sts)
    st0 = sts[0]
    ins = {k: _dev(cl[k]) for k in ("means3D", "opacities", "scales", "rotations")}
    sh, col, M = None, None, 0
    if mode != "colours":
        shs = np.ascontiguousarray(cl["shs"], f32)
        M = shs.shape[1]
        flat = torch.zeros(shs.size + 4, device="cuda")
        off = 1 if misalign else 0
        flat[off:off + shs.size] = torch.as_tensor(shs.reshape(-1)).cuda()
        sh = C.c_void_p(flat.data_ptr() + 4 * off)
        assert (flat.data_ptr() + 4 * off) % 16 == (4 if misalign else 0)
    else:
        colt = _dev(cl["colors_precomp"])
        col = C.c_void_p(colt.data_ptr())
    vd = _dev(views_of(sts))
    out = torch.full((V, N, 12), float("nan"), device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())              # noqa: E731
    _lib.check(_lib.lib.gs_b200_debug_preprocess_views(
        V, st0.image_height, st0.image_width, st0.sh_degree, st0.scale_modifier, p(vd), N, M, p(ins["means3D"]), sh,
        col, p(ins["opacities"]), p(ins["scales"]), p(ins["rotations"]), int(mode == "geom"), p(out), R._stream()))
    torch.cuda.synchronize()
    return out.cpu().numpy().view(np.uint32).copy()


def twice(tag, fn):
    a, b = fn(), fn()
    assert np.array_equal(a, b), f"{tag}: two runs differ"
    return a


def one_view_paths(cl, sts, modes):
    """{path: [V][N, 12]} of the one-view kernel"""
    out = {}
    for mode in modes:
        cov = None
        if mode == "cov":
            cov = cl["cov3D_precomp"] if "cov3D_precomp" in cl else cov3d32(cl, sts[0].scale_modifier)
        elif "cov3D_precomp" in cl:
            cov = cl["cov3D_precomp"]
        out[f"one-view {mode}"] = [twice(f"one-view {mode}", lambda st=st: run_one(cl, st, mode, cov)) for st in sts]
    return out


def multi_paths(cl, sts, modes, misalign=False):
    return {f"multi {m}" + (" misaligned" if misalign else ""):
            list(twice(f"multi {m}", lambda m=m: run_multi(cl, sts, m, misalign))) for m in modes}


def check_scene(tag, cl, sts, one_modes=("shs", "colours", "cov"), multi_modes=("shs", "colours", "geom"),
                misalign=False, culled=True):
    """every path against the oracle with tile culling off, twice; then with culling on: float words unchanged and
    tiles_touched the binning's culled count"""
    from gs_b200 import rasterizer as R
    prev = R.get_tile_culling()
    try:
        R.set_tile_culling(0)
        got = one_view_paths(cl, sts, one_modes)
        got.update(multi_paths(cl, sts, multi_modes))
        if misalign:
            got.update(multi_paths(cl, sts, [m for m in multi_modes if m != "colours"], True))
        for path, recs in got.items():
            for v, st in enumerate(sts):
                want = expected(cl, st, colours="colours" in path)
                assert_records(f"{tag} {path} view {v}", recs[v], want)
        if culled and multi_modes:
            R.set_tile_culling(2)
            tight = one_view_paths(cl, sts, one_modes[:1])
            tight.update(multi_paths(cl, sts, multi_modes[:1]))
            bins = R.bin_views(_dev(views_of(sts)), sts[0].image_height, sts[0].image_width, sts[0].sh_degree,
                               sts[0].scale_modifier, *(_dev(cl[k]) for k in ("means3D", "shs", "opacities", "scales",
                                                                               "rotations")), True, lists=False)
            for path, recs in tight.items():
                base = got[path]
                for v in range(len(sts)):
                    assert_records(f"{tag} {path} view {v} (tile culling)", recs[v], base[v], range(11))
                    t = bins["tiles_touched"][v].cpu().numpy().astype(np.uint32)
                    assert np.array_equal(recs[v][:, 11], t), f"{tag} {path} view {v}: tiles word != culled count"
    finally:
        R.set_tile_culling(prev)
    return got


gpu = pytest.mark.gpu


@gpu
def test_f1_near_plane_and_projection():
    cl, sts = f1_scene()
    check_scene("F1", cl, sts)


@gpu
def test_f2_frustum_clamp():
    cl, sts, _ = f2_scene()
    check_scene("F2", cl, sts)


@gpu
@pytest.mark.parametrize("mod", F3_MODS)
def test_f3_scales_and_rotations(mod):
    cl, sts = f3_sr_scene(mod)
    check_scene(f"F3 mod {mod}", cl, sts)


@gpu
def test_f3_precomputed_covariance():
    cl, sts, _ = f3_precomp_scene()
    check_scene("F3 precomp", cl, sts, one_modes=("shs", "colours"), multi_modes=(), culled=False)


@gpu
@pytest.mark.parametrize("deg,M", f4_cases())
def test_f4_sh_colour(deg, M):
    cl, sts = f4_sh_scene(deg, M)
    check_scene(f"F4 deg {deg} M {M}", cl, sts, one_modes=("shs", "colours", "cov"))


@gpu
def test_f4_precomputed_colours():
    cl, sts = f4_colour_scene()
    got = check_scene("F4 colours", cl, sts, one_modes=("colours",), multi_modes=("colours",), culled=False)
    neg0 = np.float32(-0.0).view(np.uint32)
    for path, recs in got.items():
        rgb = recs[0][:, 8:11]
        assert (rgb == neg0).any(), f"F4 colours {path}: -0 did not pass through"


@gpu
@pytest.mark.parametrize("V", F5_V)
@pytest.mark.parametrize("N", F5_N)
def test_f5_launch_shape(N, V):
    cl, sts = f5_scene(N, V)
    got = check_scene(f"F5 N {N} V {V}", cl, sts, one_modes=("shs", "colours"), misalign=True)
    ref = got["multi shs"]
    for path in ("one-view shs", "multi geom", "multi shs misaligned", "multi geom misaligned"):
        for v in range(V):
            assert np.array_equal(got[path][v], ref[v]), f"F5 N {N} V {V}: {path} differs from multi shs, view {v}"
