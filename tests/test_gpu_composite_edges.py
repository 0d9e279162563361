"""Composite kernels against a float64 evaluation of the same operation, on scenes built in pixel units at the edges
where the kernels go wrong: tile lists of exactly L records around the 128-record ring stages (S1), pixels that
terminate at chosen list positions (S2), large thin rotated splats whose alpha = 1/255 level set crosses quadrant
corners and tile rows (S3), and frames whose edge tiles are mostly outside the image (S4).  Two runs of the same scenes
in one process must agree bit for bit.

Reference.  `oracle/gs_oracle.py`'s composite in float64, run on the records the kernels work on: the fp32 oracle's
preprocess outputs (which reproduce the library's; its integer outputs are checked bit for bit) cast to double.  The
input gradients chain the fp64 composite's derivatives through the fp64 preprocess.  This isolates the composite: the
fp32 projection alone moves a mean near x = 2000 px by ~1e-4 px, which would dominate any composite bar.  The kernels
make discrete decisions (power <= 0, alpha >= 1/255, T (1 - alpha) < 1e-4) where fp32 and fp64 may legitimately disagree
when a value sits on a threshold; `pair_analysis` gives every (record, pixel) pair an fp32 error scale rho (units of
u = 2^-24) and excludes a pixel when any pair it considers lies within EXCL_Z u rho (relative) of a threshold.  (The
0.99 clamp needs no exclusion: min() is continuous and its gradient is straight-through on both sides.)  Excluded pixels
get zero upstream gradient, so they cannot move the gradients either; their count is asserted per scene.

Bars (derivation).  rho_j = 8 + 10 S bounds the relative fp32 error of alpha_j in units of u: 8 for the opacity product,
ex2.approx (<= 2 ulp) and the record's log2 scaling; 10 S for the power's five roundings and those of dx, dy, each
<= u S, where S is the sum of |terms| of the quadratic form.  T_j's relative error scale is R_j = sum over earlier
contributors of (alpha/(1-alpha)) rho + 2.  An image value is a recursive sum, so its bound is u (sum_j |term_j|
(rho_j + R_j + 2) + sum_j |running sum_j| + |bg| T (R + 1)); the bar is IMG_K times that.  A gradient element is a
linear image (|J|, fp64 autograd of the preprocess) of the ten per-splat sums, whose per-pixel terms get the scale
rho_j + R_N + 16 + (contributors behind j): R_N because the backward rebuilds T from final_T by division, 16 for the
per-quadrant fp32 sums over <= 64 pixels, the count for the `behind` recurrence; moments are taken against the quadrant
centre (|LX| <= 3.5), so dx enters as |dx| + 8; the preprocess backward adds 8 + 4 cond (cond = (|a c| + b^2) / det of
the 2D covariance) per derivative.  The bar is GRAD_K times that.  These worst-case bars are loose for the geometry
gradients, so every gradient is also held to GRAD_REL (1e-4) norm- and element-relative, ten times tighter than the
suite's 1e-3, and every image error to IMG_CAP (3e-5), whichever bar is smaller.  The test prints each bar's size, the
worst error / bar ratio and the worst error per quantity."""
import math
from functools import lru_cache

import numpy as np
import pytest
import torch

from oracle import gs_oracle as O

NAMES = ("means3D", "shs", "opacities", "scales", "rotations")
GRADS = NAMES + ("means2D",)
FOVY, RADIUS, DEG = 49.1, 1.75, 1
U = 2.0 ** -24
EXCL_Z = 2.0                # exclusion: a threshold within twice the error bound u rho (relative) of the value
IMG_K = 4.0
GRAD_K = 4.0
IMG_CAP = 3e-5              # whatever the derived image bar, no image error may exceed this (the suite allows 1e-4)
GRAD_REL = 1e-4             # gradients: norm- and element-relative, ten times tighter than the suite's 1e-3
S1_LENGTHS = (0, 1, 31, 32, 33, 127, 128, 129, 255, 256, 257, 383, 384, 385, 512, 513, 641)


# ---------------------------------------------------------------------------------------------------------------------
# scenes in pixel units: a camera on the +z axis looks at the origin; a splat at depth `dep` with centre (px, py) and
# standard deviations (sx, sy) in pixels, rotated by theta in the image plane
# ---------------------------------------------------------------------------------------------------------------------
def splats(W, H, px, py, dep, sx, sy, theta, op, seed):
    px, py, dep, sx, sy, theta = (torch.as_tensor(np.asarray(v, dtype=np.float64)) for v in (px, py, dep, sx, sy, theta))
    k = math.tan(math.radians(FOVY) / 2) * dep / (H / 2)               # world units per pixel at each splat's depth
    n = px.numel()
    g = torch.Generator().manual_seed(seed)
    rots = torch.stack([torch.cos(theta / 2), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64),
                        -torch.sin(theta / 2)], 1)
    return {"means3D": torch.stack([(px - (W - 1) / 2) * k, -(py - (H - 1) / 2) * k, RADIUS - dep], 1).float().contiguous(),
            "shs": (torch.rand(n, (DEG + 1) ** 2, 3, generator=g) - 0.5).contiguous(),
            "opacities": torch.as_tensor(np.asarray(op, dtype=np.float32))[:, None].contiguous(),
            "scales": torch.stack([sx * k, sy * k, torch.minimum(sx, sy) * k], 1).float().contiguous(),
            "rotations": rots.float().contiguous()}


def settings(W, H, bg=(0.1, 0.2, 0.3)):
    return O.minicam_settings(O.orbit_camera(0, 0, RADIUS), W, H, FOVY, bg=bg, sh_degree=DEG)


def upstream(W, H, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(3, H, W, generator=g) * 2 - 1, (torch.rand(1, H, W, generator=g) * 2 - 1) * 0.1,
            (torch.rand(1, H, W, generator=g) * 2 - 1) * 0.1)


def s1_scene():
    """S1: a 6 x 3 tile image; tile i holds exactly S1_LENGTHS[i] records (the 18th none).  Faint (o 0.01-0.03),
    small (sigma 0.6-1.2 px, 3-sigma radius <= 5) splats whose bounding squares stay inside their tile, centres biased
    towards quadrant (0, 0) (weights 0.5 / 0.25 / 0.15 / 0.1), so all four quadrants are hit, unevenly, at every wrap."""
    W, H = 96, 48
    rng = np.random.default_rng(11)
    px, py, sig, op = [], [], [], []
    for t, L in enumerate(S1_LENGTHS):
        tx, ty = t % 6, t // 6
        q = rng.choice(4, size=L, p=(0.5, 0.25, 0.15, 0.1))
        cx = 16 * tx + 7.5 + np.where(q & 1, 1.0, -1.0) * rng.uniform(0.0, 2.4, L)
        cy = 16 * ty + 7.5 + np.where(q & 2, 1.0, -1.0) * rng.uniform(0.0, 2.4, L)
        px += cx.tolist(); py += cy.tolist()
        sig += rng.uniform(0.6, 1.2, L).tolist(); op += rng.uniform(0.01, 0.03, L).tolist()
    n = len(px)
    dep = rng.permutation(np.linspace(1.5, 2.5, n))
    return splats(W, H, px, py, dep, sig, sig, np.zeros(n), op, seed=12), settings(W, H), upstream(W, H, 13)


# S2: single 16 x 16 tiles.  `k` is the list position of a pixel's last blended record (n_contrib).  A pixel cannot stop
# with n_contrib = 1 in exact arithmetic: T >= 0.01 after one blend and alpha <= 0.99, so T (1 - alpha) >= 1e-4 (fp32
# stops two clamped layers, 0.99f, where fp64 does not).  The ladder therefore starts at 2, and every k has a stop record
# at k + 1: n_contrib = 128 / 129 put the last contributor on a stage's last / first record, and stops at positions 128,
# 129, 130, 256-258 cover both sides of each wrap.
S2_UNIFORM = (2, 127, 128, 129, 255, 256, 257)
S2_QUAD = ((127, 128, 129, None), (255, 256, 257, 2), (None, 2, None, 129))
BEHIND = 60


def s2_scene(kind, arg):
    """Uniform tiles: three wide layers (sigma 60 px, o 0.985: alpha 0.969-0.985 over the tile) at positions k - 1,
    k, k + 1: two blend (T >= 2.2e-4 * T_fill), the third stops every pixel.  Per-quadrant tiles: three layers of a
    narrow splat (sigma 2 px, o 0.995) centred 0.25 px off pixel (3, 3) of the quadrant (alpha 0.981 there): one at
    an early free position, one at k_q, the stop at the next free position after k_q; no record between k_q and the
    stop reaches that pixel (the layers of other quadrants stay below 1/255 there, fillers keep 3 px away).  Other
    positions hold faint small fillers (o 0.01-0.03); BEHIND wide faint records follow everything."""
    W = H = 16
    rng = np.random.default_rng(100 + (arg if kind == "u" else 7 * arg))
    if kind == "u":
        special = {p: (7.5, 7.5, 60.0, 0.985) for p in (arg - 1, arg, arg + 1)}
        centres = np.array([(3.5 + 8 * (q & 1), 3.5 + 8 * (q >> 1)) for q in range(4)])
    else:
        ks = sorted((kq, q) for q, kq in enumerate(S2_QUAD[arg]) if kq is not None)
        lay = {q: (8 * (q & 1) + 3.25, 8 * (q >> 1) + 3.25, 2.0, 0.995) for _, q in ks}
        special = {}
        for kq, q in ks:
            assert kq not in special
            special[kq] = lay[q]
        for kq, q in ks:
            special[min(p for p in range(1, kq) if p not in special)] = lay[q]
        for kq, q in ks:
            special[min(p for p in range(kq + 1, 10 ** 4) if p not in special)] = lay[q]
        centres = np.array([v[:2] for v in lay.values()])
    last = max(special)
    px, py, sig, op = [], [], [], []
    for p in range(1, last + 1):
        if p in special:
            cx, cy, s, o = special[p]
        else:
            while True:
                cx, cy = rng.uniform(1.0, 14.0, 2)
                if np.min(np.hypot(*(centres - (cx, cy)).T)) >= 3.0:
                    break
            s, o = rng.uniform(0.6, 0.9), rng.uniform(0.01, 0.03)
        px.append(cx); py.append(cy); sig.append(s); op.append(o)
    for _ in range(BEHIND):
        px.append(rng.uniform(0.0, 15.0)); py.append(rng.uniform(0.0, 15.0))
        sig.append(rng.uniform(6.0, 10.0)); op.append(rng.uniform(0.05, 0.3))
    n = len(px)
    dep = np.linspace(1.2, 2.8, n)                   # list order = the order built above
    return splats(W, H, px, py, dep, sig, sig, np.zeros(n), op, seed=200 + n), settings(W, H, bg=(0.3, 0.6, 0.9)), \
        upstream(W, H, 300 + n)


S4_FRAMES = ((1, 1), (7, 5), (16, 16), (17, 33), (1, 300), (300, 1), (2000, 16))


def s4_scene(W, H):
    """S4: frames with partial edge tiles.  Background (0.3, 0.6, 0.9).  Two thirds of the splats sit just beyond the
    right / bottom edge (centres up to 6 px outside, sigma 1-4 px), so most of their footprint falls on the
    out-of-image pixels of the edge tiles; the rest are spread over the frame.  40 % of the splats are anisotropic
    (minor / major 0.25-0.7) and rotated, so the rotation gradients are compared with a non-zero fp64 reference."""
    rng = np.random.default_rng(W * 1000 + H)
    n = int(min(400, 24 + 0.3 * W * H / 16))
    edge = rng.random(n) < 2 / 3
    px = np.where(edge & (rng.random(n) < 0.5), W - 1 + rng.uniform(-2.0, 6.0, n), rng.uniform(-2.0, W + 1.0, n))
    py = np.where(edge & (px < W - 3), H - 1 + rng.uniform(-2.0, 6.0, n), rng.uniform(-2.0, H + 1.0, n))
    sig = rng.uniform(1.0, 4.0, n)
    aniso = rng.random(n) < 0.4                      # 40 %: anisotropic and rotated, so the rotation gradient is not 0
    sy = np.where(aniso, sig * rng.uniform(0.25, 0.7, n), sig)
    theta = np.where(aniso, rng.uniform(0.0, np.pi, n), 0.0)
    op = rng.uniform(0.05, 0.9, n)
    dep = rng.permutation(np.linspace(1.5, 2.5, n))
    return splats(W, H, px, py, dep, sig, sy, theta, op, seed=W + H), settings(W, H, bg=(0.3, 0.6, 0.9)), \
        upstream(W, H, W * 7 + H)


def scene(name):
    """(cloud, settings, upstream) of a scene id"""
    if name == "S1":
        return s1_scene()
    if name.startswith("S2u"):
        return s2_scene("u", int(name[3:]))
    if name.startswith("S2q"):
        return s2_scene("q", int(name[3:]))
    W, H = (int(v) for v in name[2:].split("x"))
    return s4_scene(W, H)


SCENES = ["S1"] + [f"S2u{k}" for k in S2_UNIFORM] + [f"S2q{i}" for i in range(len(S2_QUAD))] + \
    [f"S4{W}x{H}" for W, H in S4_FRAMES]
# stated upper bound on S1's excluded pixels (S2: 4 per tile, S4: max(2, W H / 500) per frame)
MAX_EXCLUDED = {"S1": 8}


# ---------------------------------------------------------------------------------------------------------------------
# float64 analysis of every (record, pixel) pair
# ---------------------------------------------------------------------------------------------------------------------
def pair_analysis(pre, point_list, ranges, st, up=None):
    """Per pixel: the excluded mask and the error scales E of colour[3], depth, alpha, final_T (units of u); with
    upstream gradients `up` also V[N, 10], the bound scales of the ten per-splat derivatives
    (px, py, a, b, c, opacity, r, g, b, depth) in units of u.  Returns dict; also the reconstructed fp64 images."""
    W, H = st.image_width, st.image_height
    gx, gy = pre["grid"]
    xy = pre["xy"].detach().double().numpy(); con = pre["conic"].detach().double().numpy()
    op = pre["opacity"].detach().double().numpy(); rgb = pre["rgb"].detach().double().numpy()
    dep = pre["depth"].detach().double().numpy()
    N = xy.shape[0]
    bg = st.bg.double().numpy()
    excl = np.zeros((H, W), bool)
    E = np.zeros((6, H, W)); img = np.zeros((6, H, W))                 # colour 3, depth, alpha, final_T
    img[:3] = bg[:, None, None]; img[5] = 1.0; E[:3] = np.abs(bg)[:, None, None]; E[5] = 1.0
    V = np.zeros((N, 10))
    if up is not None:
        gC = up[0].double().numpy(); gD = up[1].double().numpy()[0]; gA = up[2].double().numpy()[0]
    for t in range(gx * gy):
        s, e = int(ranges[t, 0]), int(ranges[t, 1])
        if e <= s:
            continue
        ids = point_list[s:e].astype(np.int64)
        ty, tx = divmod(t, gx)
        ys, xs = np.meshgrid(np.arange(ty * 16, min(ty * 16 + 16, H)), np.arange(tx * 16, min(tx * 16 + 16, W)), indexing="ij")
        ys, xs = ys.reshape(-1), xs.reshape(-1)
        dx = xy[ids, 0, None] - xs[None]; dy = xy[ids, 1, None] - ys[None]
        a, b, c = con[ids, 0, None], con[ids, 1, None], con[ids, 2, None]
        P = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
        S = 0.5 * np.abs(a) * dx * dx + 0.5 * np.abs(c) * dy * dy + np.abs(b * dx * dy)
        rho = 8 + 10 * S
        G = np.exp(P)
        araw = op[ids, None] * G
        al = np.minimum(araw, 0.99)
        valid = (P <= 0) & (al >= 1 / 255)
        ae = np.where(valid, al, 0.0)
        Tafter = np.cumprod(1 - ae, axis=0)
        Tbefore = np.vstack([np.ones_like(Tafter[:1]), Tafter[:-1]])
        stop = valid & (Tafter < 1e-4)
        nstop = np.cumsum(stop, axis=0)
        contrib = valid & (nstop == 0)
        considered = (nstop - stop) == 0                                 # up to and including the stop record
        dR = np.where(contrib, ae / (1 - ae) * rho + 2, 0.0)
        R = np.cumsum(dR, axis=0)
        Rb = np.vstack([np.zeros_like(R[:1]), R[:-1]])
        RN = R[-1]
        with np.errstate(divide="ignore"):
            mA = np.abs(np.log(np.maximum(araw, 1e-300) * 255.0)) < EXCL_Z * U * rho
            mP = np.abs(P) < EXCL_Z * U * rho
            mT = valid & (np.abs(np.log(np.maximum(Tafter, 1e-300) / 1e-4)) < EXCL_Z * U * (ae / (1 - ae) * rho + Rb + 2))
        ex = (considered & (mA | mP | mT)).any(axis=0)
        excl[ys, xs] = ex
        w = np.where(contrib, ae * Tbefore, 0.0)
        TN = np.where(contrib, 1 - ae, 1.0).prod(axis=0)
        for ch in range(5):
            v = rgb[ids, ch, None] if ch < 3 else (dep[ids, None] if ch == 3 else np.ones((len(ids), 1)))
            terms = v * w
            run = np.cumsum(terms, axis=0)
            img[ch, ys, xs] = run[-1] + (TN * bg[ch] if ch < 3 else 0.0)
            E[ch, ys, xs] = (np.abs(terms) * (rho + Rb + 2)).sum(0) + np.abs(np.where(contrib, run, 0)).sum(0) + \
                (np.abs(bg[ch]) * TN * (RN + 1) if ch < 3 else 0.0)
        img[5, ys, xs] = TN
        E[5, ys, xs] = TN * (RN + 1)
        if up is None:
            continue
        gc = gC[:, ys, xs]; gd = gD[ys, xs]; ga = gA[ys, xs]
        sj = (np.abs(rgb[ids, 0, None] * gc[0]) + np.abs(rgb[ids, 1, None] * gc[1]) + np.abs(rgb[ids, 2, None] * gc[2])
              + np.abs(dep[ids, None] * gd) + np.abs(ga))                 # bound on |s_j| = |gC.rgb_j + gD depth_j + gA|
        sw = np.where(contrib, sj * w, 0.0)
        behind = np.cumsum(sw[::-1], axis=0)[::-1] - sw                 # sum over later contributors
        bgg = np.abs(bg[:, None] * gc).sum(0)
        Aj = np.where(contrib, Tbefore * sj + (behind + TN * bgg) / (1 - ae), 0.0)   # bound on |dL/dalpha_j|
        nbehind = np.cumsum(contrib[::-1], axis=0)[::-1] - contrib
        scale = rho + RN + 16 + nbehind
        wk = araw * Aj * scale                                          # |dL/dpower| scale
        ax, ay = np.abs(dx) + 8, np.abs(dy) + 8
        Vt = np.stack([(wk * ax).sum(1), (wk * ay).sum(1), (wk * ax * ax).sum(1), (wk * ax * ay).sum(1),
                       (wk * ay * ay).sum(1), (G * Aj * scale).sum(1),
                       (np.abs(gc[0]) * w * scale).sum(1), (np.abs(gc[1]) * w * scale).sum(1),
                       (np.abs(gc[2]) * w * scale).sum(1), (np.abs(gd) * w * scale).sum(1)], 1)
        np.add.at(V, ids, Vt)
    out = dict(excluded=excl, E=E, img=img)
    if up is not None:
        a, b, c = np.abs(con[:, 0]), np.abs(con[:, 1]), np.abs(con[:, 2])
        out["V"] = np.stack([a * V[:, 0] + b * V[:, 1], b * V[:, 0] + c * V[:, 1], 0.5 * V[:, 2], V[:, 3], 0.5 * V[:, 4],
                             V[:, 5], V[:, 6], V[:, 7], V[:, 8], V[:, 9]], 1)
    return out


def preprocess_abs_jacobian(cl, st):
    """|d(px, py, a, b, c, opacity, r, g, b, depth) / d(input)| per Gaussian, in fp64 (the preprocess is per Gaussian,
    so the gradient of each summed output is the Jacobian's diagonal block)"""
    leaf = {k: cl[k].double().requires_grad_(True) for k in NAMES}
    m2 = torch.zeros_like(leaf["means3D"]).requires_grad_(True)
    pre = O.preprocess(leaf["means3D"], leaf["scales"], leaf["rotations"], leaf["opacities"], leaf["shs"], None, None, m2, st)
    outs = [pre["xy"][:, 0], pre["xy"][:, 1], pre["conic"][:, 0], pre["conic"][:, 1], pre["conic"][:, 2],
            pre["opacity"], pre["rgb"][:, 0], pre["rgb"][:, 1], pre["rgb"][:, 2], pre["depth"]]
    vis = pre["visible"].double()
    J = {}
    for kk, o in enumerate(outs):
        gs = torch.autograd.grad((o * vis).sum(), [leaf[k] for k in NAMES] + [m2], retain_graph=True, allow_unused=True)
        for name, gi in zip(GRADS, gs):
            gi = torch.zeros_like(leaf[name] if name != "means2D" else m2) if gi is None else gi
            J.setdefault(name, []).append(gi.detach().abs())
    return {k: torch.stack(v, 0) for k, v in J.items()}                # [10, N, ...]


@lru_cache(maxsize=None)
def reference(name):
    """fp32 oracle (integer outputs and the records the composite works on); the composite in fp64 on those records
    (images, final_T, derivatives by the records) with excluded pixels' upstream zeroed; the six input gradients as
    those derivatives chained through the fp64 preprocess; the bars; the excluded mask"""
    cl, st, up = scene(name)
    fp32 = O.rasterize(cl["means3D"], torch.zeros_like(cl["means3D"]), cl["shs"], None, cl["opacities"], cl["scales"],
                       cl["rotations"], None, st, return_aux=True)
    aux = fp32[4]
    pre = aux["pre"]
    rec = {k: pre[k].detach().double().requires_grad_(True) for k in ("xy", "conic", "opacity", "rgb", "depth")}
    rec["grid"] = pre["grid"]
    an = pair_analysis(rec, aux["point_list"], aux["ranges"], st)
    keep = torch.from_numpy(~an["excluded"])
    up0 = tuple(u * keep[None].float() for u in up)
    an = pair_analysis(rec, aux["point_list"], aux["ranges"], st, tuple(u.double() for u in up0))
    color, depth, alpha, n_contrib, final_T = O.composite(rec, aux["point_list"], aux["ranges"], st)
    loss = (color * up0[0].double()).sum() + (depth * up0[1].double()).sum() + (alpha * up0[2].double()).sum()
    keys2d = ("xy", "conic", "opacity", "rgb", "depth")
    d2d = torch.autograd.grad(loss, [rec[k] for k in keys2d])
    leaf = {k: cl[k].double().requires_grad_(True) for k in NAMES}
    m2 = torch.zeros_like(leaf["means3D"]).requires_grad_(True)
    p64 = O.preprocess(leaf["means3D"], leaf["scales"], leaf["rotations"], leaf["opacities"], leaf["shs"], None, None, m2, st)
    g = torch.autograd.grad([p64[k] for k in keys2d], [leaf[k] for k in NAMES] + [m2], grad_outputs=list(d2d),
                            allow_unused=True)
    g64 = {k: (torch.zeros_like(leaf[k] if k != "means2D" else m2) if gi is None else gi.detach()) for k, gi in zip(GRADS, g)}
    # bound scales of the ten derivatives: the composite's (V) plus the preprocess backward's own rounding, which works
    # on the fp32 forward values (relative 8 + 4 cond of each derivative)
    cov = pre["cov2d"].detach().double()
    det = (cov[:, 0] * cov[:, 2] - cov[:, 1] ** 2).abs()
    cond = ((cov[:, 0] * cov[:, 2]).abs() + cov[:, 1] ** 2) / torch.where(det > 0, det, torch.ones_like(det))
    d10 = torch.cat([d2d[0], d2d[1], d2d[2][:, None], d2d[3], d2d[4][:, None]], 1).abs()
    V = torch.from_numpy(an["V"]) + (8 + 4 * cond[:, None]) * d10                  # [N, 10], units of u
    J = preprocess_abs_jacobian(cl, st)
    gbar = {}
    for k in GRADS:
        shape = J[k].shape[1:]
        gbar[k] = GRAD_K * U * (J[k] * V.t().reshape(10, shape[0], *([1] * (len(shape) - 1)))).sum(0)
    # the rotation gradient of a splat with equal scales is a cancellation inside the covariance chain (its fp64 value
    # and |J| are zero); its terms are of the size of the scale gradient times the scale
    sc = cl["scales"].double()
    gbar["rotations"] = gbar["rotations"] + 8 * ((gbar["scales"] + GRAD_K * U * 16 * g64["scales"].abs()) * sc).sum(1, keepdim=True)
    out64 = dict(color=color.detach(), depth=depth.detach(), alpha=alpha.detach(), final_T=final_T.detach())
    return dict(cl=cl, st=st, up=up0, fp32=fp32, out64=out64, g64=g64, an=an, gbar=gbar)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the scenes' premises
# ---------------------------------------------------------------------------------------------------------------------
def test_pair_analysis_reconstructs_the_fp64_oracle():
    """(CPU) the per-pair reconstruction behind exclusions and bars computes the oracle's fp64 images"""
    for name in ("S1", "S2q1", "S417x33"):
        r = reference(name)
        img, o = r["an"]["img"], r["out64"]
        assert np.abs(img[:3] - o["color"].numpy()).max() < 1e-12
        assert np.abs(img[3] - o["depth"].numpy()[0]).max() < 1e-12
        assert np.abs(img[4] - o["alpha"].numpy()[0]).max() < 1e-12
        assert np.abs(img[5] - o["final_T"].numpy()).max() < 1e-12


def test_s1_premise():
    """(CPU) tile t lists exactly S1_LENGTHS[t] records, every splat is visible, no pixel gets T < 1e-4, and each
    listed tile has records hitting each of its four quadrants"""
    r = reference("S1")
    ranges = r["fp32"][4]["ranges"]
    lengths = [int(e - s) for s, e in ranges]
    assert lengths == list(S1_LENGTHS) + [0]
    assert bool((r["fp32"][1] > 0).all())
    assert float(r["out64"]["final_T"].min()) >= 1e-4 * 10
    nc = r["fp32"][4]["n_contrib"].numpy()
    for t, L in enumerate(S1_LENGTHS):
        if L < 32:
            continue
        ty, tx = divmod(t, 6)
        for qy in (0, 8):
            for qx in (0, 8):
                assert nc[16 * ty + qy:16 * ty + qy + 8, 16 * tx + qx:16 * tx + qx + 8].max() > 0
    assert int(r["an"]["excluded"].sum()) <= MAX_EXCLUDED["S1"]


def test_s2_premise():
    """(CPU) the exact n_contrib ladder from `composite_sequential` (fp64): uniform tiles stop every pixel with
    n_contrib = k; per-quadrant tiles stop pixel (3, 3) of quadrant q with n_contrib = k_q, and quadrants without a
    k run into the records behind; records behind every stop exist and contribute elsewhere"""
    def run(cl, st):
        c64 = {kk: v.double() for kk, v in cl.items()}
        pre = O.preprocess(c64["means3D"], c64["scales"], c64["rotations"], c64["opacities"], c64["shs"], None, None, None, st)
        keys, vals = O.sort_pairs(*O.duplicate_with_keys(pre))
        ranges = O.identify_tile_ranges(keys, 1)
        _, _, _, nc, T = O.composite_sequential(pre, vals, ranges, st)
        return int(ranges[0, 1]), nc, T
    for k in S2_UNIFORM:
        cl, st, _ = s2_scene("u", k)
        L, nc, T = run(cl, st)
        assert L == k + 1 + BEHIND
        assert bool((nc == k).all()), (k, nc.unique())
        assert float(T.max()) < 1e-3                    # every pixel stopped with the stop layer still ahead
    for i, ks in enumerate(S2_QUAD):
        cl, st, _ = s2_scene("q", i)
        L, nc, _ = run(cl, st)
        for q, kq in enumerate(ks):
            y, x = 3 + 8 * (q >> 1), 3 + 8 * (q & 1)
            if kq is None:
                assert int(nc[y, x]) > L - BEHIND, (i, q, int(nc[y, x]))
            else:
                assert int(nc[y, x]) == kq, (i, q, int(nc[y, x]))
        assert int(nc.max()) > L - BEHIND
    for name in [f"S2u{k}" for k in S2_UNIFORM] + [f"S2q{i}" for i in range(len(S2_QUAD))]:
        assert int(reference(name)["an"]["excluded"].sum()) <= 4, name


def test_s4_premise():
    """(CPU) every frame has partial edge tiles (except 16 x 16) with out-of-image footprint, and few exclusions"""
    for W, H in S4_FRAMES:
        r = reference(f"S4{W}x{H}")
        pre = r["fp32"][4]["pre"]
        vis = pre["visible"]
        assert int(vis.sum()) > 0, (W, H)
        xy = pre["xy"][vis]
        outside = ((xy[:, 0] > W - 1) | (xy[:, 1] > H - 1)).float().mean()
        assert float(outside) > 0.3, (W, H)
        assert int(r["an"]["excluded"].sum()) <= max(2, W * H // 500), (W, H)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the kernels against the fp64 reference
# ---------------------------------------------------------------------------------------------------------------------
def kernel_outputs(cl, st, up, dev):
    from gs_b200 import rasterizer as R
    W, H = st.image_width, st.image_height
    rs = R.GaussianRasterizationSettings(H, W, st.tanfovx, st.tanfovy, st.bg.to(dev), st.scale_modifier,
                                         st.viewmatrix.to(dev), st.projmatrix.to(dev), DEG, st.campos.to(dev), False, False)
    fs = R.forward_with_state(rs, cl["means3D"].to(dev), cl["opacities"].to(dev), shs=cl["shs"].to(dev),
                              scales=cl["scales"].to(dev), rotations=cl["rotations"].to(dev))
    out = {k: fs[k].detach().cpu().clone() for k in ("color", "depth", "alpha", "final_T", "n_contrib", "radii",
                                                     "sorted_keys", "point_list", "ranges")}
    inp = {k: cl[k].to(dev).requires_grad_(True) for k in NAMES}
    m2 = torch.zeros(cl["means3D"].shape[0], 3, device=dev, requires_grad=True)
    color, _, depth, alpha = R.GaussianRasterizer(rs)(
        means3D=inp["means3D"], means2D=m2, shs=inp["shs"], colors_precomp=None, opacities=inp["opacities"],
        scales=inp["scales"], rotations=inp["rotations"], cov3D_precomp=None)
    ((color * up[0].to(dev)).sum() + (depth * up[1].to(dev)).sum() + (alpha * up[2].to(dev)).sum()).backward()
    torch.cuda.synchronize()
    for k in NAMES:
        out["g_" + k] = inp[k].grad.cpu()
    out["g_means2D"] = m2.grad.cpu()
    return out


def check_against_fp64(name, got):
    """integer outputs bit-exact against the fp32 oracle; images, final_T and the six gradients within the fp64 bars.
    Returns the worst ratio error / bar per quantity."""
    r = reference(name)
    _, radii, _, _, aux = r["fp32"]
    an = r["an"]
    keep = ~an["excluded"]
    assert torch.equal(got["radii"], radii)
    assert np.array_equal(got["sorted_keys"].numpy().astype(np.uint64), aux["keys"])
    assert np.array_equal(got["point_list"].numpy().astype(np.uint32), aux["point_list"])
    assert np.array_equal(got["ranges"].numpy().astype(np.uint32), aux["ranges"])
    nc_bad = (got["n_contrib"].numpy() != aux["n_contrib"].numpy()) & keep
    assert int(nc_bad.sum()) == 0, f"{name}: n_contrib differs from the fp32 oracle at {int(nc_bad.sum())} pixels"
    worst = {}
    o64 = r["out64"]
    pairs = (("color", got["color"].double().numpy(), o64["color"].numpy(), an["E"][:3]),
             ("depth", got["depth"].double().numpy()[0], o64["depth"].numpy()[0], an["E"][3]),
             ("alpha", got["alpha"].double().numpy()[0], o64["alpha"].numpy()[0], an["E"][4]),
             ("final_T", got["final_T"].double().numpy(), o64["final_T"].numpy(), an["E"][5]))
    for what, a, b, E in pairs:
        bar = IMG_K * U * E
        worst[what + "_bar"] = float(bar.max())
        err = np.abs(a - b)
        m = keep if a.ndim == 2 else np.broadcast_to(keep, a.shape)
        ratio = np.where(m, err / np.maximum(bar, 1e-300), 0.0)
        worst[what] = float(ratio.max()) if ratio.size else 0.0
        worst[what + "_err"] = float(err[m].max()) if m.any() else 0.0
        assert worst[what] <= 1.0, f"{name} {what}: error {float(err[m].max())} over the bar ({worst[what]:.3g}x)"
        assert worst[what + "_err"] <= IMG_CAP, f"{name} {what}: error {worst[what + '_err']} over {IMG_CAP}"
    for k in GRADS:
        a, b, bar = got["g_" + k].double(), r["g64"][k].double(), r["gbar"][k]
        err = (a - b).abs()
        ratio = err / torch.clamp_min(bar, 1e-300)
        worst["g_" + k] = float(ratio.max()) if ratio.numel() else 0.0
        worst["g_" + k + "_relbar"] = float(bar.norm() / b.norm()) if float(b.norm()) > 0 else 0.0
        assert worst["g_" + k] <= 1.0, f"{name} grad {k}: error over the bar ({worst['g_' + k]:.3g}x, max err {float(err.max())})"
        # and 10x tighter than the suite's `_grad_close`: norm-relative GRAD_REL, element-wise GRAD_REL relative with a
        # floor of GRAD_REL / 100 of the largest component
        if float(b.norm()) > 0:
            rel = float((a - b).norm() / b.norm())
            worst["g_" + k + "_rel"] = rel
            assert rel < GRAD_REL, f"{name} grad {k}: norm-relative error {rel:.3g}"
            scale = float(b.abs().max())
            assert bool((err <= GRAD_REL * b.abs() + 1e-2 * GRAD_REL * scale).all()), f"{name} grad {k}: element-wise"
        # (a zero reference -- the rotation gradient of splats with equal scales -- is held to the derived bar alone: the
        # kernel's value is the rounding noise of an exact cancellation)
    return worst


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENES)
def test_scene_matches_fp64(dev, name):
    """the composite kernels, one scene, against the fp64 bars"""
    r = reference(name)
    got = kernel_outputs(r["cl"], r["st"], r["up"], dev)
    worst = check_against_fp64(name, got)
    print(f"{name}: excluded {int(r['an']['excluded'].sum())} px; worst " +
          " ".join(f"{k}={v:.3g}" for k, v in worst.items()))


# ---------------------------------------------------------------------------------------------------------------------
# S3: culling adversaries (forward, one splat per render, so a pixel's output alpha is that splat's alpha)
# ---------------------------------------------------------------------------------------------------------------------
S3_W, S3_H = 1920, 1080
S3_SIGMA = (20.0, 80.0, 300.0, 1000.0, 2200.0)
S3_THETA = (0.0, 0.31, 0.785398, 1.2, 1.5708, 2.5)
S3_OPACITY = (1.03 / 255, 0.05, 0.6, 1.0)


def s3_splats():
    """every (sigma_major, theta, opacity) combination, sigma_minor at the 0.3 px^2 low-pass floor (world minor scale
    ~1e-3 px); centres uniform over the frame widened by 10 % on each side, so some lie outside the image"""
    rng = np.random.default_rng(5)
    out = []
    for s in S3_SIGMA:
        for th in S3_THETA:
            for o in S3_OPACITY:
                out.append((rng.uniform(-0.1, 1.1) * S3_W, rng.uniform(-0.1, 1.1) * S3_H, s, th, o))
    return out


def s3_cloud(i):
    px, py, s, th, o = s3_splats()[i]
    return splats(S3_W, S3_H, [px], [py], [2.0], [s], [1e-3], [th], [o], seed=i)


def s3_alpha(pre):
    """fp64 alpha image of the single splat, evaluated from the fp32 preprocess record (the fp32 oracle reproduces the
    kernel's preprocess; the record's conic is the operand the composite works on), with the per-pixel error scale of
    the kernel's power in log2 units"""
    xy = pre["xy"].detach().double().numpy()[0]; con = pre["conic"].detach().double().numpy()[0]
    o = float(pre["opacity"][0])
    ys, xs = np.mgrid[0:S3_H, 0:S3_W].astype(np.float64)
    dx, dy = xy[0] - xs, xy[1] - ys
    P = -0.5 * (con[0] * dx * dx + con[2] * dy * dy) - con[1] * dx * dy
    S = (0.5 * abs(con[0]) * dx * dx + 0.5 * abs(con[2]) * dy * dy + abs(con[1]) * np.abs(dx * dy)) / math.log(2)
    araw = o * np.exp(P)
    return P, np.minimum(araw, 0.99), araw, S


S3_ERR_K = 12.0   # log2-unit error of the kernel's power <= 12 u S: five roundings, dx and dy, the record's scaling


def test_s3_premise():
    """(CPU) every splat is visible, its alpha >= 1/255 region crosses quadrant corners and tile-row boundaries
    (many 8 x 8 quadrants whose largest alpha is within [1, 1.5] / 255), opacities just above 1/255 and above the
    0.99 clamp are present, and some centres are outside the image"""
    outside = hidden = 0
    barely_corner = barely_row = 0
    for i in range(len(s3_splats())):
        cl, st = s3_cloud(i), settings(S3_W, S3_H)
        pre = O.preprocess(cl["means3D"], cl["scales"], cl["rotations"], cl["opacities"], cl["shs"], None, None, None, st)
        if int(pre["radii"][0]) == 0:              # centre too far outside for its size: no tile listed
            hidden += 1
            continue
        xy = pre["xy"][0]
        outside += int(not (0 <= float(xy[0]) < S3_W and 0 <= float(xy[1]) < S3_H))
        if i % 5:
            continue                                # the full-frame evaluation is slow on a CPU: every fifth splat
        P, al, _, _ = s3_alpha(pre)
        a = np.pad(al, ((0, 0), (0, 0)))
        q = a[:S3_H // 8 * 8].reshape(S3_H // 8, 8, S3_W // 8, 8).max(axis=(1, 3))
        barely = (q * 255 >= 1) & (q * 255 <= 1.5)
        barely_corner += int(barely.sum())
        rows = a[15::16] * 255
        barely_row += int(((rows >= 1) & (rows <= 1.5)).sum())
    assert outside >= 10 and hidden <= len(s3_splats()) // 10
    assert barely_corner > 50 and barely_row > 50
    assert min(S3_OPACITY) * 255 < 1.05 and max(S3_OPACITY) > 0.99


def s3_kernel_alpha(pre):
    """alpha image of the single splat as the composite computes it: the record's log2-scaled conic rounded to fp32
    as the preprocess writes it (c.x = fl(-0.5 log2e conA), c.y = fl(-log2e conB), c.z = fl(-0.5 log2e conC)), and the
    power in power2's operation order, t = c.x dx; t = fma(c.y, dy, t); p = t dx; p = fma(c.z dy, dy, p), in fp32
    (an fma is one fp64 operation on fp32 operands, whose products are exact in fp64, rounded to fp32).  What remains
    unemulated is ex2.approx (<= 2^-22 relative), the opacity product and the fma's rare double rounding."""
    f = np.float32
    xy = pre["xy"].detach().numpy().astype(f)[0]; con = pre["conic"].detach().numpy().astype(f)[0]
    l2e = f(1.4426950408889634)
    cx, cy, cz = f(f(-0.5) * l2e) * con[0], l2e * (-con[1]), f(f(-0.5) * l2e) * con[2]
    ys, xs = np.mgrid[0:S3_H, 0:S3_W]
    dx = (xy[0] - xs.astype(f)).astype(f); dy = (xy[1] - ys.astype(f)).astype(f)
    t = (cx * dx).astype(f)
    t = (np.float64(cy) * dy.astype(np.float64) + t.astype(np.float64)).astype(f)
    pw = (t * dx).astype(f)
    q = (cz * dy).astype(f)
    pw = (q.astype(np.float64) * dy.astype(np.float64) + pw.astype(np.float64)).astype(f)
    o = float(pre["opacity"][0])
    return pw.astype(np.float64), np.minimum(o * np.exp2(pw.astype(np.float64)), 0.99)


S3_DELTA = 2.0 ** -18      # covers ex2.approx, the opacity product and the fma double rounding (each <= 2^-21)


@pytest.mark.gpu
@pytest.mark.parametrize("culling", [0, 2])
def test_s3_every_pixel_above_the_level_set_shows_the_splat(dev, culling):
    """Observable: inside the splat's listed tiles, every pixel where the composite's own per-pixel arithmetic
    (`s3_kernel_alpha`) gives alpha >= (1 + S3_DELTA)/255 and power <= 0 shows the splat (output alpha > 0), and every
    pixel where it gives alpha < (1 - S3_DELTA)/255 does not.  The per-pixel test is emulated, so the band left
    unchecked is 2^-18 wide and the whole alpha = 1/255 level set is checked: a miss can only come from a culling test
    (quad_hit, or with culling 2 also tight_spans) rejecting a quadrant or tile the splat reaches.  Shown pixels must
    equal the emulated alpha within S3_DELTA, and the fp64 alpha within the fp32 bound of the power (S3_ERR_K u S).
    tight_spans only handles squares of at most 8 tile rows (sigma_major up to ~20 px); larger squares are listed
    whole, so for sigma_major >= 80 px only quad_hit is exercised."""
    from gs_b200 import rasterizer as R
    st = settings(S3_W, S3_H)
    rs = R.GaussianRasterizationSettings(S3_H, S3_W, st.tanfovx, st.tanfovy, st.bg.to(dev), 1.0, st.viewmatrix.to(dev),
                                         st.projmatrix.to(dev), DEG, st.campos.to(dev), False, False)
    misses, stray, worst, worst_em, band, covered = [], 0, 0.0, 0.0, 0, 0
    R.set_tile_culling(culling)
    try:
        for i in range(len(s3_splats())):
            cl = s3_cloud(i)
            pre = O.preprocess(cl["means3D"], cl["scales"], cl["rotations"], cl["opacities"], cl["shs"], None, None, None, st)
            with torch.no_grad():
                _, radii, _, alpha = R.GaussianRasterizer(rs)(
                    means3D=cl["means3D"].to(dev), means2D=torch.zeros(1, 3, device=dev), opacities=cl["opacities"].to(dev),
                    shs=cl["shs"].to(dev), scales=cl["scales"].to(dev), rotations=cl["rotations"].to(dev))
            assert int(radii[0]) == int(pre["radii"][0])
            if int(radii[0]) == 0:
                continue
            k = alpha[0].double().cpu().numpy()
            pk, ak = s3_kernel_alpha(pre)
            P, al, _, S = s3_alpha(pre)
            # the package lists a splat only in the tiles of its 3-sigma square: pixels outside it never show the splat
            (x0, y0), (x1, y1) = pre["rect_min"][0].tolist(), pre["rect_max"][0].tolist()
            rect = np.zeros_like(al, bool)
            rect[16 * y0:16 * y1, 16 * x0:16 * x1] = True
            must = (ak * 255 >= 1 + S3_DELTA) & (pk <= 0) & rect
            never = (ak * 255 < 1 - S3_DELTA) | (pk > 0) | ~rect
            in_band = rect & (al * 255 >= 1.1) & (al * 255 < 3)
            band += int(in_band.sum()); covered += int((in_band & must).sum())
            miss = must & (k == 0)
            if miss.any():
                ys, xs = np.nonzero(miss)
                misses.append((i, int(miss.sum()), float(ak[ys[0], xs[0]] * 255), int(ys[0]), int(xs[0])))
            stray += int((never & (k > 0)).sum())
            shown = must & (k > 0)
            if shown.any():
                worst_em = max(worst_em, float((np.abs(k[shown] - ak[shown]) / ak[shown]).max() / S3_DELTA))
                err = S3_ERR_K * U * S[shown]
                rel = np.abs(k[shown] - al[shown]) / al[shown]
                worst = max(worst, float((rel / (np.exp2(err) * (1 + S3_DELTA) - 1)).max()))
    finally:
        R.set_tile_culling(1)
    print(f"S3 culling {culling}: worst |alpha - alpha_emulated| / (alpha 2^-18) = {worst_em:.3g}, "
          f"worst |alpha - alpha64| / fp32 bound = {worst:.3g}; pixels with 255 alpha64 in [1.1, 3) whose fp32 alpha "
          f"is also above 1/255: {covered} of {band}")
    assert not misses, f"culling false negatives (splat, pixels, 255 alpha, y, x): {misses[:8]}"
    assert stray == 0
    assert worst_em <= 1.0 and worst <= 1.0


# ---------------------------------------------------------------------------------------------------------------------
# run-to-run determinism on the scenes above
# ---------------------------------------------------------------------------------------------------------------------
REPEAT_SCENES = ["S1", "S2u128", "S2u257", "S2q0", "S2q1", "S417x33", "S42000x16"]


def _scene_outputs(dev):
    res = {}
    for name in REPEAT_SCENES:
        cl, st, up = scene(name)
        for k, v in kernel_outputs(cl, st, up, dev).items():
            res[f"{name}/{k}"] = v.numpy()
    return res


@pytest.mark.gpu
def test_default_runs_are_bit_identical(dev):
    """every output and gradient of the scenes, run twice in one process, is bit-identical"""
    first, again = _scene_outputs(dev), _scene_outputs(dev)
    for k in first:
        assert np.array_equal(first[k], again[k], equal_nan=True), k
