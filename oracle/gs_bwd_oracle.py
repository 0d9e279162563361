"""float64 restatement of the per-Gaussian preprocess backward (csrc/gs_backward.cu), with a running bound on the error
of the kernel's fp32 evaluation of every gradient element.

Values.  The chain is restated operation by operation in float64 on the fp32 inputs, with the reference's quirks kept:
  * dL/dcov2D goes through 1/(det^2 + 1e-7f) (the exact derivative of the conic has 1/det^2); the screen-space mean
    gradient uses the exact conic cc/det, -cb/det, ca/det;
  * when |t.x / t.z| > 1.3 tanfovx (fp32), t.x gets no gradient through J and t.z differentiates J with the clamped
    value lim * t.z held fixed (same for y);
  * a colour channel whose fp32 SH colour (before the max with 0) is < 0 passes no gradient;
  * the quaternion is used as given, not normalised.
Every discrete decision is taken from fp32, as the kernels take it: the visibility (radii > 0 of the forward), the two
frustum-clamp masks (fp32 t.x / t.z against fp32 1.3 tanfov) and the SH clamp (`sh_colour32`, the forward's colour
arithmetic: explicit fp32 fmas from 0, then + 0.5).  These are inputs here; `clamp_masks32` and `sh_colour32` compute
them.

Bars.  Every value carries `e`, a first-order bound on |fp32 evaluation - exact value of the same formula on the same
fp32 inputs|: each operation adds u |result| (u = 2^-24) to the propagated input bounds (a + b: ea + eb;
a b: |a| eb + |b| ea + ea eb; a / b: (ea + |a / b| eb) / (|b| - eb); sqrt(a): ea / (2 sqrt(a))).  The bound is
therefore k u sum |terms| over the chain, evaluated in float64; FMA contraction only removes roundings, so it holds for
any contraction the compiler chooses.  A kernel gradient element g passes when |g - v| <= BAR_K e + FLOOR |v|, with
BAR_K = 2 (room for the second-order terms the first-order bound drops) and FLOOR = 1e-12 (float64 noise of v itself).
An element whose value and bound are both 0 (a culled Gaussian, a masked SH channel, an SH row above the active degree)
must be exactly 0.
"""
import numpy as np

from oracle.uvbake_oracle import fma32

f32 = np.float32
U = 2.0 ** -24
BAR_K = 2.0
FLOOR = 1e-12

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)


def _c(x):
    """a kernel literal (fp32) as an exact E"""
    return x if isinstance(x, E) else E(np.asarray(x, f32).astype(np.float64))


class E:
    """float64 value v with a bound e on the error of the kernel's fp32 evaluation"""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = np.asarray(v, dtype=np.float64)
        self.e = np.zeros_like(self.v) if e is None else np.asarray(e, dtype=np.float64)

    def __add__(self, o):
        o = _c(o); v = self.v + o.v
        return E(v, self.e + o.e + U * np.abs(v))

    __radd__ = __add__

    def __sub__(self, o):
        o = _c(o); v = self.v - o.v
        return E(v, self.e + o.e + U * np.abs(v))

    def __rsub__(self, o):
        return _c(o) - self

    def __neg__(self):
        return E(-self.v, self.e)

    def __mul__(self, o):
        o = _c(o); v = self.v * o.v
        return E(v, np.abs(self.v) * o.e + np.abs(o.v) * self.e + self.e * o.e + U * np.abs(v))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = _c(o)
        with np.errstate(all="ignore"):
            v = self.v / o.v
            e = (self.e + np.abs(v) * o.e) / np.maximum(np.abs(o.v) - o.e, 1e-300) + U * np.abs(v)
        return E(v, e)

    def __rtruediv__(self, o):
        return _c(o) / self

    def where(self, mask, other):
        other = _c(other)
        return E(np.where(mask, self.v, other.v), np.where(mask, self.e, other.e))


def sqrt(a):
    with np.errstate(all="ignore"):
        v = np.sqrt(a.v)
        return E(v, a.e / np.maximum(2.0 * v, 1e-300) + U * v)


def zeros(n):
    return E(np.zeros(n))


def add_where(acc, term, mask):
    """acc + term where mask (one fp32 add), acc untouched elsewhere"""
    s = acc + term
    return E(np.where(mask, s.v, acc.v), np.where(mask, s.e, acc.e))


# ---------------------------------------------------------------------------------------------------------------------
# fp32 decisions
# ---------------------------------------------------------------------------------------------------------------------
def sh_colour32(deg, sh, d):
    """The forward's SH colour before the max with 0, bit for bit (gs_common.cuh gs_sh_colour): sh [N, M, 3] fp32,
    d [N, 3] = mean - campos in fp32.  Returns rgb [N, 3] fp32."""
    sh = np.asarray(sh, f32); d = np.asarray(d, f32)
    with np.errstate(all="ignore"):
        inv = f32(1.0) / np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
        x, y, z = d[:, 0] * inv, d[:, 1] * inv, d[:, 2] * inv
        bas = [np.full_like(x, f32(SH_C0))]
        if deg > 0:
            bas += [f32(-SH_C1) * y, f32(SH_C1) * z, f32(-SH_C1) * x]
        if deg > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            c2 = [f32(v) for v in SH_C2]
            bas += [c2[0] * xy, c2[1] * yz, c2[2] * (f32(2) * zz - xx - yy), c2[3] * xz, c2[4] * (xx - yy)]
        if deg > 2:
            c3 = [f32(v) for v in SH_C3]
            bas += [c3[0] * y * (f32(3) * xx - yy), c3[1] * xy * z, c3[2] * y * (f32(4) * zz - xx - yy),
                    c3[3] * z * (f32(2) * zz - f32(3) * xx - f32(3) * yy), c3[4] * x * (f32(4) * zz - xx - yy),
                    c3[5] * z * (xx - yy), c3[6] * x * (xx - f32(3) * yy)]
        out = np.zeros((len(x), 3), f32)
        for ch in range(3):
            r = np.zeros_like(x)
            for k, b in enumerate(bas):
                r = fma32(b, sh[:, k, ch], r)
            out[:, ch] = r + f32(0.5)
    return out


def view_t32(m, means):
    """t = W mean + t_w in fp32, the kernels' left-to-right order (exact for an axis-aligned view matrix, whatever the
    contraction)"""
    m = np.asarray(m, f32).reshape(16); x, y, z = (np.asarray(means, f32)[:, i] for i in range(3))
    tx = m[0] * x + m[4] * y + m[8] * z + m[12]
    ty = m[1] * x + m[5] * y + m[9] * z + m[13]
    tz = m[2] * x + m[6] * y + m[10] * z + m[14]
    return tx, ty, tz


def clamp_masks32(m, means, tanfovx, tanfovy):
    """(in_x, in_y): t.x / t.z and t.y / t.z within [-1.3 tanfov, 1.3 tanfov] in fp32"""
    tx, ty, tz = view_t32(m, means)
    limx, limy = f32(1.3) * f32(tanfovx), f32(1.3) * f32(tanfovy)
    with np.errstate(all="ignore"):
        txtz, tytz = tx / tz, ty / tz
    return (txtz >= -limx) & (txtz <= limx), (tytz >= -limy) & (tytz <= limy)


# ---------------------------------------------------------------------------------------------------------------------
# the chain
# ---------------------------------------------------------------------------------------------------------------------
def _cov3d_fwd(scales, rots, mod):
    sc = [_c(mod) * E(scales[:, k]) for k in range(3)]
    r, qx, qy, qz = (E(rots[:, k]) for k in range(4))
    R = [1.0 - 2.0 * (qy * qy + qz * qz), 2.0 * (qx * qy - r * qz), 2.0 * (qx * qz + r * qy),
         2.0 * (qx * qy + r * qz), 1.0 - 2.0 * (qx * qx + qz * qz), 2.0 * (qy * qz - r * qx),
         2.0 * (qx * qz - r * qy), 2.0 * (qy * qz + r * qx), 1.0 - 2.0 * (qx * qx + qy * qy)]
    Mm = [R[3 * i + k] * sc[k] for i in range(3) for k in range(3)]
    c = [Mm[0] * Mm[0] + Mm[1] * Mm[1] + Mm[2] * Mm[2], Mm[0] * Mm[3] + Mm[1] * Mm[4] + Mm[2] * Mm[5],
         Mm[0] * Mm[6] + Mm[1] * Mm[7] + Mm[2] * Mm[8], Mm[3] * Mm[3] + Mm[4] * Mm[4] + Mm[5] * Mm[5],
         Mm[3] * Mm[6] + Mm[4] * Mm[7] + Mm[5] * Mm[8], Mm[6] * Mm[6] + Mm[7] * Mm[7] + Mm[8] * Mm[8]]
    return c, R, sc


def _cov3d_bwd(dcv, R, sc, mod, rots):
    Gxx, Gxy, Gxz, Gyy, Gyz, Gzz = dcv[0], 0.5 * dcv[1], 0.5 * dcv[2], dcv[3], 0.5 * dcv[4], dcv[5]
    dsc, dR = [None] * 3, [None] * 9
    for k in range(3):
        M0, M1, M2 = R[k] * sc[k], R[3 + k] * sc[k], R[6 + k] * sc[k]
        d0 = 2.0 * (Gxx * M0 + Gxy * M1 + Gxz * M2)
        d1 = 2.0 * (Gxy * M0 + Gyy * M1 + Gyz * M2)
        d2 = 2.0 * (Gxz * M0 + Gyz * M1 + Gzz * M2)
        dsc[k] = _c(mod) * (d0 * R[k] + d1 * R[3 + k] + d2 * R[6 + k])
        dR[k], dR[3 + k], dR[6 + k] = d0 * sc[k], d1 * sc[k], d2 * sc[k]
    r, qx, qy, qz = (E(rots[:, k]) for k in range(4))
    dq = [2.0 * (qz * (dR[3] - dR[1]) + qy * (dR[2] - dR[6]) + qx * (dR[7] - dR[5])),
          2.0 * (qy * (dR[1] + dR[3]) + qz * (dR[2] + dR[6]) + r * (dR[7] - dR[5])) - 4.0 * qx * (dR[4] + dR[8]),
          2.0 * (qx * (dR[1] + dR[3]) + r * (dR[2] - dR[6]) + qz * (dR[5] + dR[7])) - 4.0 * qy * (dR[0] + dR[8]),
          2.0 * (r * (dR[3] - dR[1]) + qx * (dR[2] + dR[6]) + qy * (dR[5] + dR[7])) - 4.0 * qz * (dR[0] + dR[4])]
    return dsc, dq


def _sh_basis(deg, dx, dy, dz):
    n = dx.v.shape
    z0 = E(np.zeros(n))
    bas, bx, by, bz = [E(np.full(n, np.float64(f32(SH_C0))))], [z0], [z0], [z0]
    if deg > 0:
        c1 = _c(SH_C1)
        bas += [-c1 * dy, c1 * dz, -c1 * dx]
        bx += [z0, z0, -c1]; by += [-c1, z0, z0]; bz += [z0, c1, z0]
    if deg > 1:
        c = [_c(v) for v in SH_C2]
        xx, yy, zz, xy, yz, xz = dx * dx, dy * dy, dz * dz, dx * dy, dy * dz, dx * dz
        bas += [c[0] * xy, c[1] * yz, c[2] * (2.0 * zz - xx - yy), c[3] * xz, c[4] * (xx - yy)]
        bx += [c[0] * dy, z0, c[2] * -2.0 * dx, c[3] * dz, c[4] * 2.0 * dx]
        by += [c[0] * dx, c[1] * dz, c[2] * -2.0 * dy, z0, c[4] * -2.0 * dy]
        bz += [z0, c[1] * dy, c[2] * 4.0 * dz, c[3] * dx, z0]
    if deg > 2:
        c = [_c(v) for v in SH_C3]
        bas += [c[0] * dy * (3.0 * xx - yy), c[1] * xy * dz, c[2] * dy * (4.0 * zz - xx - yy),
                c[3] * dz * (2.0 * zz - 3.0 * xx - 3.0 * yy), c[4] * dx * (4.0 * zz - xx - yy), c[5] * dz * (xx - yy),
                c[6] * dx * (xx - 3.0 * yy)]
        bx += [c[0] * 6.0 * xy, c[1] * yz, c[2] * -2.0 * xy, c[3] * -6.0 * xz, c[4] * (4.0 * zz - 3.0 * xx - yy),
               c[5] * 2.0 * xz, c[6] * (3.0 * xx - 3.0 * yy)]
        by += [c[0] * (3.0 * xx - 3.0 * yy), c[1] * xz, c[2] * (4.0 * zz - xx - 3.0 * yy), c[3] * -6.0 * yz,
               c[4] * -2.0 * xy, c[5] * -2.0 * yz, c[6] * -6.0 * xy]
        bz += [z0, c[1] * xy, c[2] * 8.0 * yz, c[3] * (6.0 * zz - 3.0 * xx - 3.0 * yy), c[4] * 8.0 * xz,
               c[5] * (xx - yy), z0]
    return bas, bx, by, bz


def view_backward(view, deg, means, c, sg, shs=None, rgb_mask=None, in_xy=None):
    """One view's contribution of every Gaussian (the kernels' backward_view), evaluated for all rows; the caller masks
    the invisible ones.  view: dict m[16], p[16], cam[3], tanfovx, tanfovy, fx, fy, W, H (fp32 values).  c: cov3D
    (6 E).  sg [N, 12] fp32.  shs [N, M, 3] or None (colours precomputed).  rgb_mask [N, 3]: the fp32 SH colour is
    < 0.  in_xy: clamp_masks32.  Returns a dict of E (and lists of E)."""
    m = [_c(v) for v in np.asarray(view["m"], f32).reshape(16)]
    p = [_c(v) for v in np.asarray(view["p"], f32).reshape(16)]
    x, y, z = (E(np.asarray(means, f32)[:, i]) for i in range(3))
    sg = np.asarray(sg, f32).astype(np.float64)
    gg, gc, gk = [E(sg[:, i]) for i in range(4)], [E(sg[:, 4 + i]) for i in range(4)], [E(sg[:, 8 + i]) for i in range(4)]
    tx = m[0] * x + m[4] * y + m[8] * z + m[12]
    ty = m[1] * x + m[5] * y + m[9] * z + m[13]
    tz = m[2] * x + m[6] * y + m[10] * z + m[14]
    hx = p[0] * x + p[4] * y + p[8] * z + p[12]
    hy = p[1] * x + p[5] * y + p[9] * z + p[13]
    hw = p[3] * x + p[7] * y + p[11] * z + p[15]
    pw = 1.0 / (hw + 1e-7)
    dmx, dmy, dmz = m[2] * gg[2], m[6] * gg[2], m[10] * gg[2]
    out = {"dop": gc[3]}
    if shs is not None:
        shs = np.asarray(shs, f32)
        cam = [_c(v) for v in np.asarray(view["cam"], f32)]
        vx, vy, vz = x - cam[0], y - cam[1], z - cam[2]
        inv = 1.0 / sqrt(vx * vx + vy * vy + vz * vz)
        dx, dy, dz = vx * inv, vy * inv, vz * inv
        bas, bx, by, bz = _sh_basis(deg, dx, dy, dz)
        dcol = [gk[ch].where(~rgb_mask[:, ch], 0.0) for ch in range(3)]
        ddx = ddy = ddz = zeros(len(x.v))
        dsh = []
        for k in range(len(bas)):
            s = dcol[0] * E(shs[:, k, 0]) + dcol[1] * E(shs[:, k, 1]) + dcol[2] * E(shs[:, k, 2])
            ddx, ddy, ddz = ddx + bx[k] * s, ddy + by[k] * s, ddz + bz[k] * s
            dsh.append([bas[k] * dcol[ch] for ch in range(3)])
        dot = dx * ddx + dy * ddy + dz * ddz
        dmx, dmy, dmz = dmx + (ddx - dx * dot) * inv, dmy + (ddy - dy * dot) * inv, dmz + (ddz - dz * dot) * inv
        out["dsh"] = dsh
    else:
        out["dcol"] = gk[:3]
    fx, fy = _c(view["fx"]), _c(view["fy"])
    limx, limy = f32(1.3) * f32(view["tanfovx"]), f32(1.3) * f32(view["tanfovy"])
    inx, iny = in_xy
    txtz, tytz = tx / tz, ty / tz
    cx = txtz.where(inx, np.clip(txtz.v, -limx, limx)) * tz
    cy = tytz.where(iny, np.clip(tytz.v, -limy, limy)) * tz
    xmul, ymul = E(inx.astype(np.float64)), E(iny.astype(np.float64))
    itz = 1.0 / tz
    itz2 = itz * itz
    itz3 = itz2 * itz
    J00, J02, J11, J12 = fx * itz, -(fx * cx) * itz2, fy * itz, -(fy * cy) * itz2
    T00, T01, T02 = J00 * m[0] + J02 * m[2], J00 * m[4] + J02 * m[6], J00 * m[8] + J02 * m[10]
    T10, T11, T12 = J11 * m[1] + J12 * m[2], J11 * m[5] + J12 * m[6], J11 * m[9] + J12 * m[10]
    c0, c1, c2, c3, c4, c5 = c
    v00, v01, v02 = c0 * T00 + c1 * T01 + c2 * T02, c1 * T00 + c3 * T01 + c4 * T02, c2 * T00 + c4 * T01 + c5 * T02
    v10, v11, v12 = c0 * T10 + c1 * T11 + c2 * T12, c1 * T10 + c3 * T11 + c4 * T12, c2 * T10 + c4 * T11 + c5 * T12
    ca = T00 * v00 + T01 * v01 + T02 * v02 + 0.3
    cb = T00 * v10 + T01 * v11 + T02 * v12
    cc = T10 * v10 + T11 * v11 + T12 * v12 + 0.3
    denom = ca * cc - cb * cb
    d2i = 1.0 / (denom * denom + 1e-7)
    gA, gB, gC = -0.5 * gc[0], -gc[1], -0.5 * gc[2]
    di = 1.0 / denom
    cA, cB, cC = cc * di, -cb * di, ca * di
    dpx, dpy = -(cA * gg[0] + cB * gg[1]), -(cB * gg[0] + cC * gg[1])
    g2x, g2y = dpx * (0.5 * _c(view["W"])), dpy * (0.5 * _c(view["H"]))
    out["g2x"], out["g2y"] = g2x, g2y
    mul1, mul2 = hx * pw * pw, hy * pw * pw
    dmx = dmx + ((p[0] * pw - p[3] * mul1) * g2x + (p[1] * pw - p[3] * mul2) * g2y)
    dmy = dmy + ((p[4] * pw - p[7] * mul1) * g2x + (p[5] * pw - p[7] * mul2) * g2y)
    dmz = dmz + ((p[8] * pw - p[11] * mul1) * g2x + (p[9] * pw - p[11] * mul2) * g2y)
    ga = d2i * (-cc * cc * gA + cb * cc * gB - cb * cb * gC)
    gb = d2i * (2.0 * cb * cc * gA - (denom + 2.0 * cb * cb) * gB + 2.0 * ca * cb * gC)
    gcc = d2i * (-cb * cb * gA + ca * cb * gB - ca * ca * gC)
    out["dcv"] = [T00 * T00 * ga + T00 * T10 * gb + T10 * T10 * gcc,
                  2.0 * T00 * T01 * ga + (T00 * T11 + T01 * T10) * gb + 2.0 * T10 * T11 * gcc,
                  2.0 * T00 * T02 * ga + (T00 * T12 + T02 * T10) * gb + 2.0 * T10 * T12 * gcc,
                  T01 * T01 * ga + T01 * T11 * gb + T11 * T11 * gcc,
                  2.0 * T01 * T02 * ga + (T01 * T12 + T02 * T11) * gb + 2.0 * T11 * T12 * gcc,
                  T02 * T02 * ga + T02 * T12 * gb + T12 * T12 * gcc]
    dT00, dT01, dT02 = 2.0 * ga * v00 + gb * v10, 2.0 * ga * v01 + gb * v11, 2.0 * ga * v02 + gb * v12
    dT10, dT11, dT12 = 2.0 * gcc * v10 + gb * v00, 2.0 * gcc * v11 + gb * v01, 2.0 * gcc * v12 + gb * v02
    dJ00 = m[0] * dT00 + m[4] * dT01 + m[8] * dT02
    dJ02 = m[2] * dT00 + m[6] * dT01 + m[10] * dT02
    dJ11 = m[1] * dT10 + m[5] * dT11 + m[9] * dT12
    dJ12 = m[2] * dT10 + m[6] * dT11 + m[10] * dT12
    dtx = xmul * (-fx * itz2) * dJ02
    dty = ymul * (-fy * itz2) * dJ12
    dtz = -fx * itz2 * dJ00 - fy * itz2 * dJ11 + (2.0 * fx * cx) * itz3 * dJ02 + (2.0 * fy * cy) * itz3 * dJ12
    out["dm"] = [dmx + (m[0] * dtx + m[1] * dty + m[2] * dtz), dmy + (m[4] * dtx + m[5] * dty + m[6] * dtz),
                 dmz + (m[8] * dtx + m[9] * dty + m[10] * dtz)]
    out["denom"] = denom
    return out


def preprocess_backward(views, deg, M, means, sg, radii, shs=None, colors_precomp=None, scales=None, rots=None,
                        cov3D_precomp=None, mod=1.0, chunk=1, bounds=None):
    """Gradients of every Gaussian summed over `views` (dicts as view_backward's, each with `rgb_mask` and `in_xy`
    when needed; see `decisions`), in the kernels' order: chunk = 1 is the one-view kernel called once per view with
    the later calls accumulating; otherwise the multi-view kernel over view chunks of `chunk` views, or over the chunks
    [bounds[k], bounds[k + 1]) when given (views summed per Gaussian inside a chunk, the cov3D chain run once per
    chunk, later chunks accumulating).  sg [V, N, 12], radii [V, N].  Returns a dict name ->
    E over the flattened gradient array of that input (means3D [N*3], means2D [N*3], shs [N*M*3], colors, opacities,
    scales, rotations, cov3D)."""
    means = np.asarray(means, f32)
    N = len(means)
    if cov3D_precomp is not None:
        cp = np.asarray(cov3D_precomp, f32)
        c, R, sc = [E(cp[:, k]) for k in range(6)], None, None
    else:
        scales, rots = np.asarray(scales, f32), np.asarray(rots, f32)
        c, R, sc = _cov3d_fwd(scales, rots, mod)
    z = lambda: zeros(N)            # noqa: E731
    G = {"dm": [z() for _ in range(3)], "g2": [z(), z()], "dop": z(), "dsc": [z() for _ in range(3)],
         "dq": [z() for _ in range(4)], "dcv": [z() for _ in range(6)], "dcol": [z() for _ in range(3)],
         "dsh": [[z() for _ in range(3)] for _ in range(M)]}
    V = len(views)
    if bounds is None:
        bounds = list(range(0, V, chunk)) + [V]
    for k0, k1 in zip(bounds[:-1], bounds[1:]):
        A = {"dm": [z() for _ in range(3)], "g2": [z(), z()], "dop": z(), "dcv": [z() for _ in range(6)],
             "dcol": [z() for _ in range(3)], "dsh": [[z() for _ in range(3)] for _ in range(M)]}
        any_vis = np.zeros(N, bool)
        for v in range(k0, k1):
            vis = np.asarray(radii[v]) > 0
            any_vis |= vis
            vw = views[v]
            o = view_backward(vw, deg, means, c, sg[v], shs, vw.get("rgb_mask"), vw["in_xy"])
            for i in range(3):
                A["dm"][i] = add_where(A["dm"][i], o["dm"][i], vis)
            A["g2"][0] = add_where(A["g2"][0], o["g2x"], vis)
            A["g2"][1] = add_where(A["g2"][1], o["g2y"], vis)
            A["dop"] = add_where(A["dop"], o["dop"], vis)
            for i in range(6):
                A["dcv"][i] = add_where(A["dcv"][i], o["dcv"][i], vis)
            if shs is not None:
                for k in range(len(o["dsh"])):
                    for ch in range(3):
                        A["dsh"][k][ch] = add_where(A["dsh"][k][ch], o["dsh"][k][ch], vis)
            else:
                for ch in range(3):
                    A["dcol"][ch] = add_where(A["dcol"][ch], o["dcol"][ch], vis)
        if cov3D_precomp is None:
            dsc, dq = _cov3d_bwd(A["dcv"], R, sc, mod, rots)
        first = k0 == 0
        upd = (lambda g, a: a.where(any_vis, 0.0)) if first else (lambda g, a: add_where(g, a, any_vis))
        for key in ("dm", "g2", "dcv", "dcol"):
            G[key] = [upd(g, a) for g, a in zip(G[key], A[key])]
        G["dop"] = upd(G["dop"], A["dop"])
        if cov3D_precomp is None:
            G["dsc"] = [upd(g, a) for g, a in zip(G["dsc"], dsc)]
            G["dq"] = [upd(g, a) for g, a in zip(G["dq"], dq)]
        for k in range(M):      # SH rows are written (chunk 0) or added (later chunks) for every Gaussian
            for ch in range(3):
                a = A["dsh"][k][ch]
                G["dsh"][k][ch] = a if first else G["dsh"][k][ch] + a

    def flat(lst, cols):
        return E(np.stack([g.v for g in lst], 1).reshape(-1), np.stack([g.e for g in lst], 1).reshape(-1)) \
            if cols else None
    out = {"means3D": flat(G["dm"], 3), "means2D": flat(G["g2"] + [z()], 3), "opacities": flat([G["dop"]], 1)}
    if shs is not None:
        rows = [G["dsh"][k][ch] for k in range(M) for ch in range(3)]
        out["shs"] = flat(rows, 1)
    else:
        out["colors"] = flat(G["dcol"], 3)
    if cov3D_precomp is None:
        out["scales"], out["rotations"] = flat(G["dsc"], 3), flat(G["dq"], 4)
    else:
        out["cov3D"] = flat(G["dcv"], 6)
    return out


def decisions(view, deg, means, shs=None):
    """The fp32 decisions of one view for view_backward: rgb_mask (SH colour < 0) and in_xy (clamp masks)"""
    d = {"in_xy": clamp_masks32(view["m"], means, view["tanfovx"], view["tanfovy"])}
    if shs is not None:
        dirs = np.asarray(means, f32) - np.asarray(view["cam"], f32)[None]
        d["rgb_mask"] = sh_colour32(deg, shs, dirs) < 0
    return d


def check(name, got, ref, exact_zero=True):
    """(worst |got - v| / bar, number of elements) for one gradient; raises AssertionError naming the worst element
    when any element is outside BAR_K e + FLOOR |v|, or (exact_zero) nonzero where v and e are both 0"""
    got = np.asarray(got, np.float64).reshape(-1)
    bar = BAR_K * ref.e + FLOOR * np.abs(ref.v)
    err = np.abs(got - ref.v)
    if exact_zero:
        zero = bar == 0
        bad = np.flatnonzero(zero & (got != 0))
        assert bad.size == 0, f"{name}: {bad.size} elements nonzero where the oracle is exactly 0, e.g. [{bad[0]}] = " \
            f"{got[bad[0]]!r}"
    with np.errstate(all="ignore"):
        ratio = np.where(bar > 0, err / bar, np.where(err > 0, np.inf, 0.0))
    assert np.all(np.isfinite(got)), f"{name}: non-finite kernel gradient"
    i = int(np.argmax(ratio)) if ratio.size else 0
    assert ratio.size == 0 or ratio[i] <= 1.0, \
        f"{name}[{i}]: kernel {got[i]!r}, oracle {ref.v[i]!r}, |err| {err[i]:.3e} > bar {bar[i]:.3e}"
    return (float(ratio[i]) if ratio.size else 0.0), ratio.size
