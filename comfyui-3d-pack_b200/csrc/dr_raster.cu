// Mesh rasterizer: clip-space triangles -> (u, v, z/w, id+1) + barycentric pixel derivatives.
//
// Replaces nvdiffrast's dr.rasterize (CudaRaster path; diff_mesh_renderer.py:97, flexicubes_renderer.py:49,
// mesh_utils.py:531).  GPU-first design instead of a port of the bin/coarse/fine software pipeline:
//   1. one thread per triangle evaluates 2-D HOMOGENEOUS edge functions (rows of adj([x;y;w])) over its pixel
//      bounding box — no clipping needed for vertices behind the eye — and resolves visibility with ONE 64-bit
//      atomicMin per covered pixel on (ordered z/w bits << 32 | triangle id): nearest wins, ties -> lowest id,
//      independent of scheduling order (deterministic).  Meshes here are dense (500k triangles at 1080p are
//      ~1.5 px each), so the work per triangle is a handful of pixels and the z-buffer (16 B/pixel) lives in L2;
//   2. triangles whose box exceeds 256 pixels go to a queue drained by CTA-wide loops (persistent grid);
//   3. a per-pixel resolve pass recomputes barycentrics / derivatives for the winner and writes rast, rast_db.
// Coverage is decided by the EXACT signs of the edge functions (see "exact coverage signs" below): the per-pixel loop
// evaluates them in fp64 (at 1080p the fp32 values are within their rounding error of 0 for a sizeable share of the
// pixels next to an edge), and the rare (triangle, pixel) pairs still inside the fp64 error band, in practice exact
// zeros, are deferred to a second pass that decides them exactly.
// THIS TU IS COMPILED WITH -fmad=false: z/w (and u, v) use the exact fp32 operation order of oracle/dr_oracle.py, so
// triangle ids are bit-exact against the oracle.
#include "../../include/dr_b200.h"
#include "gs_common.cuh"

namespace {

struct TriSetup { float a0, b0, c0, a1, b1, c1, a2, b2, c2, det, z0, z1, z2, sgn; };

__device__ __forceinline__ bool tri_setup(const float4 p0, const float4 p1, const float4 p2, TriSetup& t) {
    t.a0 = p1.y * p2.w - p2.y * p1.w; t.b0 = p2.x * p1.w - p1.x * p2.w; t.c0 = p1.x * p2.y - p2.x * p1.y;
    t.a1 = p2.y * p0.w - p0.y * p2.w; t.b1 = p0.x * p2.w - p2.x * p0.w; t.c1 = p2.x * p0.y - p0.x * p2.y;
    t.a2 = p0.y * p1.w - p1.y * p0.w; t.b2 = p1.x * p0.w - p0.x * p1.w; t.c2 = p0.x * p1.y - p1.x * p0.y;
    t.det = p0.x * t.a0 + p1.x * t.a1 + p2.x * t.a2;
    t.z0 = p0.z; t.z1 = p1.z; t.z2 = p2.z;
    t.sgn = (t.det < 0.f) ? -1.f : 1.f;
    return t.det != 0.f;
}

// ---- exact coverage signs ------------------------------------------------------------------------------------------
// A pixel centre P = (X, Y, 1) is inside when sign(det) e_i > 0 for all i, e_i = det[[x_j, x_k, X], [y_j, y_k, Y],
// [w_j, w_k, 1]] = (a_i X + b_i Y) + c_i.  An exact 0 is decided by the signs of (a_i, b_i), i.e. P is moved by
// (eps, eps^2): a consistent symbolic perturbation, under which a closed fan around a vertex on a pixel centre, and a
// shared edge through pixel centres, cover every point exactly once.  The fp32 e_i (the one z/w is computed from) has a
// rounding error below gamma_5 times the sum of its |terms|, which over |X|, |Y| <= 1 is at most edge_err (a 3x slack
// covers the fp32 evaluation of the bound and subnormal products); outside that band its sign is exact.  Inside it, an
// fp64 evaluation (exact products, four roundings: error <= 2^-51 sum |terms|, against err >= 2^-20 of it) decides, and
// when that too is inside its band (in practice an exact zero) the 12 triple-product terms are summed as a
// nonoverlapping expansion (fma TwoProduct, Shewchuk's Grow-Expansion).  The orientation sign(det) is settled the same
// way when the fp32 det is inside its band.

__device__ __forceinline__ float edge_err(const float4 pj, const float4 pk) {
    return ((fabsf(pj.y * pk.w) + fabsf(pk.y * pj.w)) + (fabsf(pk.x * pj.w) + fabsf(pj.x * pk.w)) +
            (fabsf(pj.x * pk.y) + fabsf(pk.x * pj.y))) * 0x1p-20f + 1.0e-37f;
}

__device__ __forceinline__ float tri_err(const float4 p0, const float4 p1, const float4 p2) {
    return fmaxf(edge_err(p1, p2), fmaxf(edge_err(p2, p0), edge_err(p0, p1)));
}

__device__ __forceinline__ float det_err(const float4 p0, const float4 p1, const float4 p2) {
    return (fabsf(p0.x) * (fabsf(p1.y * p2.w) + fabsf(p2.y * p1.w)) + fabsf(p1.x) * (fabsf(p2.y * p0.w) + fabsf(p0.y * p2.w)) +
            fabsf(p2.x) * (fabsf(p0.y * p1.w) + fabsf(p1.y * p0.w))) * 0x1p-20f + 1.0e-37f;
}

// sign of det[[x0, x1, x2], [y0, y1, y2], [w0, w1, w2]], exactly
__device__ __noinline__ int det3_sign_exact(float x0, float y0, float w0, float x1, float y1, float w1, float x2, float y2, float w2) {
    double h[12];
    int n = 0;
    const double tp[6] = {(double)x0 * y1, -((double)x0 * y2), -((double)x1 * y0), (double)x1 * y2, (double)x2 * y0, -((double)x2 * y1)};
    const float tw[6] = {w2, w1, w2, w0, w1, w0};
    for (int k = 0; k < 12; k++) {
        const double hi = tp[k >> 1] * (double)tw[k >> 1];
        double q = (k & 1) ? fma(tp[k >> 1], (double)tw[k >> 1], -hi) : hi;
        int m = 0;
        for (int i = 0; i < n; i++) {                  // Grow-Expansion with zero elimination
            const double s = q + h[i], bv = s - q, err = (q - (s - bv)) + (h[i] - bv);
            q = s;
            if (err != 0.0) h[m++] = err;
        }
        h[m++] = q;
        n = m;
    }
    for (int i = n - 1; i >= 0; i--)                    // components grow in magnitude: the largest nonzero one decides
        if (h[i] != 0.0) return h[i] > 0.0 ? 1 : -1;
    return 0;
}

// orientation sign: +-1, or 0 for a triangle of exactly zero area
__device__ float tri_orientation(const float4 p0, const float4 p1, const float4 p2, float det) {
    if (fabsf(det) > det_err(p0, p1, p2)) return det < 0.f ? -1.f : 1.f;
    return (float)det3_sign_exact(p0.x, p0.y, p0.w, p1.x, p1.y, p1.w, p2.x, p2.y, p2.w);
}

// exact coverage decision for the edge j -> k (fp32 value e, band err) of a triangle with orientation sgn
__device__ bool edge_inside_exact(float e, float err, const float4 pj, const float4 pk, float X, float Y, float sgn) {
    if (fabsf(e) > err) return e * sgn > 0.f;
    const double a = (double)pj.y * pk.w - (double)pk.y * pj.w, b = (double)pk.x * pj.w - (double)pj.x * pk.w;
    const double e64 = (a * X + b * Y) + ((double)pj.x * pk.y - (double)pk.x * pj.y);
    if (fabs(e64) > (double)err * 0x1p-28) return e64 * sgn > 0.0;
    const int s = det3_sign_exact(pj.x, pj.y, pj.w, pk.x, pk.y, pk.w, X, Y, 1.0f) * (int)sgn;
    if (s != 0) return s > 0;
    const double as = a * sgn, bs = b * sgn;
    return (as > 0.0) || ((as == 0.0) && (bs > 0.0));
}

__device__ __forceinline__ uint32_t ordered_bits(float f) {
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ void depth_write(const TriSetup& t, float e0, float e1, float e2, int tri_id, unsigned long long* zp) {
    const float zw = ((t.z0 * e0 + t.z1 * e1) + t.z2 * e2) / t.det;
    if (!(zw >= -1.0f && zw <= 1.0f)) return;
    const unsigned long long key = ((unsigned long long)ordered_bits(zw) << 32) | (unsigned long long)(uint32_t)tri_id;
    atomicMin(zp, key);
}

// Deferred work: (gid << 32) | pixel, or (gid << 32) | 0xFFFFFFFF for a triangle whose orientation is inside its band.
struct Deferred { unsigned long long* list; uint32_t* count; uint32_t cap; };

__device__ __forceinline__ void defer(const Deferred& d, uint32_t gid, uint32_t pix) {
    const uint32_t slot = atomicAdd(d.count, 1u);
    if (slot < d.cap) d.list[slot] = ((unsigned long long)gid << 32) | pix;    // overflow: the fallback pass redoes all
}

// fp64 edge coefficients (each one rounding of a difference of exact products): the per-pixel coverage filter
struct Edge64 { double a0, b0, c0, a1, b1, c1, a2, b2, c2, err; };

__device__ __forceinline__ void edge64_setup(const float4 p0, const float4 p1, const float4 p2, float err32, Edge64& g) {
    g.a0 = (double)p1.y * p2.w - (double)p2.y * p1.w; g.b0 = (double)p2.x * p1.w - (double)p1.x * p2.w; g.c0 = (double)p1.x * p2.y - (double)p2.x * p1.y;
    g.a1 = (double)p2.y * p0.w - (double)p0.y * p2.w; g.b1 = (double)p0.x * p2.w - (double)p2.x * p0.w; g.c1 = (double)p2.x * p0.y - (double)p0.x * p2.y;
    g.a2 = (double)p0.y * p1.w - (double)p1.y * p0.w; g.b2 = (double)p1.x * p0.w - (double)p0.x * p1.w; g.c2 = (double)p0.x * p1.y - (double)p1.x * p0.y;
    g.err = (double)err32 * 0x1p-28;                   // >= 2^-48 sum |terms| >= 8x the fp64 evaluation error
}

__device__ __forceinline__ void shade_pixel(const TriSetup& t, const Edge64& g, uint32_t gid, int tri_id, int px, int py, float sx,
                                            float sy, int W, unsigned long long* __restrict__ zrow, const Deferred& d) {
    const float X = ((float)px + 0.5f) * sx - 1.0f;
    const float Y = ((float)py + 0.5f) * sy - 1.0f;
    const double Xd = X, Yd = Y, sg = t.sgn;
    const double s0 = ((g.a0 * Xd + g.b0 * Yd) + g.c0) * sg, s1 = ((g.a1 * Xd + g.b1 * Yd) + g.c1) * sg,
                 s2 = ((g.a2 * Xd + g.b2 * Yd) + g.c2) * sg;
    if (s0 < -g.err || s1 < -g.err || s2 < -g.err) return;                  // surely outside
    if (!(s0 > g.err && s1 > g.err && s2 > g.err)) {                        // an exact zero (or next to one): decide later
        defer(d, gid, (uint32_t)(py * W + px));
        return;
    }
    const float e0 = (t.a0 * X + t.b0 * Y) + t.c0;                          // z/w in the fp32 contract order
    const float e1 = (t.a1 * X + t.b1 * Y) + t.c1;
    const float e2 = (t.a2 * X + t.b2 * Y) + t.c2;
    depth_write(t, e0, e1, e2, tri_id, zrow + px);
}

// the exact decision for one (triangle, pixel): the deferred pass and the overflow fallback
__device__ void shade_pixel_exact(const TriSetup& t, const float4 p0, const float4 p1, const float4 p2, float err, int tri_id,
                                  int px, int py, float sx, float sy, unsigned long long* __restrict__ zrow) {
    const float X = ((float)px + 0.5f) * sx - 1.0f;
    const float Y = ((float)py + 0.5f) * sy - 1.0f;
    const float e0 = (t.a0 * X + t.b0 * Y) + t.c0;
    const float e1 = (t.a1 * X + t.b1 * Y) + t.c1;
    const float e2 = (t.a2 * X + t.b2 * Y) + t.c2;
    if (!(edge_inside_exact(e0, err, p1, p2, X, Y, t.sgn) && edge_inside_exact(e1, err, p2, p0, X, Y, t.sgn) &&
          edge_inside_exact(e2, err, p0, p1, X, Y, t.sgn))) return;
    depth_write(t, e0, e1, e2, tri_id, zrow + px);
}

// pixel bounding box (inclusive); full screen when a vertex is behind the eye
__device__ __forceinline__ void tri_bbox(const float4 p0, const float4 p1, const float4 p2, int W, int H, int& x0,
                                         int& y0, int& x1, int& y1) {
    if (p0.w > 0.f && p1.w > 0.f && p2.w > 0.f) {
        const float ax = (p0.x / p0.w + 1.f) * (0.5f * W), bx = (p1.x / p1.w + 1.f) * (0.5f * W), cx = (p2.x / p2.w + 1.f) * (0.5f * W);
        const float ay = (p0.y / p0.w + 1.f) * (0.5f * H), by = (p1.y / p1.w + 1.f) * (0.5f * H), cy = (p2.y / p2.w + 1.f) * (0.5f * H);
        const float mnx = fminf(ax, fminf(bx, cx)), mxx = fmaxf(ax, fmaxf(bx, cx));
        const float mny = fminf(ay, fminf(by, cy)), mxy = fmaxf(ay, fmaxf(by, cy));
        // pixel i has its centre at i+0.5; one pixel of slack against rounding
        x0 = max(0, (int)floorf(fmaxf(mnx, -1.0e6f) - 0.5f) - 1); x1 = min(W - 1, (int)ceilf(fminf(mxx, 1.0e6f) - 0.5f) + 1);
        y0 = max(0, (int)floorf(fmaxf(mny, -1.0e6f) - 0.5f) - 1); y1 = min(H - 1, (int)ceilf(fminf(mxy, 1.0e6f) - 0.5f) + 1);
    } else {
        x0 = 0; y0 = 0; x1 = W - 1; y1 = H - 1;
    }
}

constexpr int LARGE_AREA = 256;

__global__ void __launch_bounds__(256)
raster_small_kernel(const float4* __restrict__ pos, const int32_t* __restrict__ tri, int B, int V, int F, int H, int W,
                    float sx, float sy, unsigned long long* __restrict__ zbuf, uint32_t* __restrict__ queue,
                    uint32_t* __restrict__ qcount, Deferred d) {
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (long long)B * F) return;
    const int b = (int)(gid / F), f = (int)(gid - (long long)b * F);
    const int i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
    if ((unsigned)i0 >= (unsigned)V || (unsigned)i1 >= (unsigned)V || (unsigned)i2 >= (unsigned)V) return;
    const float4 p0 = pos[(size_t)b * V + i0], p1 = pos[(size_t)b * V + i1], p2 = pos[(size_t)b * V + i2];
    TriSetup t;
    if (!tri_setup(p0, p1, p2, t)) return;
    if (!(fabsf(t.det) > det_err(p0, p1, p2))) {          // orientation inside its band: the whole triangle goes exact
        defer(d, (uint32_t)gid, 0xFFFFFFFFu);
        return;
    }
    int x0, y0, x1, y1;
    tri_bbox(p0, p1, p2, W, H, x0, y0, x1, y1);
    if (x1 < x0 || y1 < y0) return;
    if ((x1 - x0 + 1) * (y1 - y0 + 1) > LARGE_AREA) {
        const uint32_t slot = atomicAdd(qcount, 1u);
        queue[slot] = (uint32_t)gid;                    // capacity B*F
        return;
    }
    Edge64 g;
    edge64_setup(p0, p1, p2, tri_err(p0, p1, p2), g);
    unsigned long long* zb = zbuf + (size_t)b * H * W;
    for (int py = y0; py <= y1; py++)
        for (int px = x0; px <= x1; px++) shade_pixel(t, g, (uint32_t)gid, f, px, py, sx, sy, W, zb + (size_t)py * W, d);
}

__global__ void __launch_bounds__(256)
raster_large_kernel(const float4* __restrict__ pos, const int32_t* __restrict__ tri, int B, int V, int F, int H, int W,
                    float sx, float sy, unsigned long long* __restrict__ zbuf, const uint32_t* __restrict__ queue,
                    const uint32_t* __restrict__ qcount, Deferred d) {
    const uint32_t n = *qcount;
    for (uint32_t q = blockIdx.x; q < n; q += gridDim.x) {
        const uint32_t gid = queue[q];
        const int b = (int)(gid / (uint32_t)F), f = (int)(gid - (uint32_t)b * (uint32_t)F);
        const int i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
        const float4 p0 = pos[(size_t)b * V + i0], p1 = pos[(size_t)b * V + i1], p2 = pos[(size_t)b * V + i2];
        TriSetup t;
        tri_setup(p0, p1, p2, t);
        Edge64 g;
        edge64_setup(p0, p1, p2, tri_err(p0, p1, p2), g);
        int x0, y0, x1, y1;
        tri_bbox(p0, p1, p2, W, H, x0, y0, x1, y1);
        const int bw = x1 - x0 + 1, total = bw * (y1 - y0 + 1);
        unsigned long long* zb = zbuf + (size_t)b * H * W;
        for (int i = threadIdx.x; i < total; i += blockDim.x) {
            const int py = y0 + i / bw, px = x0 + i - (i / bw) * bw;
            shade_pixel(t, g, gid, f, px, py, sx, sy, W, zb + (size_t)py * W, d);
        }
    }
}

// exact set-up of triangle gid (false: out of range or zero area)
__device__ __forceinline__ bool exact_setup(const float4* __restrict__ pos, const int32_t* __restrict__ tri, int V, int F, uint32_t gid,
                                            TriSetup& t, float4& p0, float4& p1, float4& p2, float& err, int& b, int& f) {
    b = (int)(gid / (uint32_t)F); f = (int)(gid - (uint32_t)b * (uint32_t)F);
    const int i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
    if ((unsigned)i0 >= (unsigned)V || (unsigned)i1 >= (unsigned)V || (unsigned)i2 >= (unsigned)V) return false;
    p0 = pos[(size_t)b * V + i0]; p1 = pos[(size_t)b * V + i1]; p2 = pos[(size_t)b * V + i2];
    if (!tri_setup(p0, p1, p2, t)) return false;
    t.sgn = tri_orientation(p0, p1, p2, t.det);
    err = tri_err(p0, p1, p2);
    return t.sgn != 0.f;
}

// the deferred (triangle, pixel) pairs, and the triangles whose orientation needed the exact sign (whole box)
__global__ void __launch_bounds__(256)
raster_deferred_kernel(const float4* __restrict__ pos, const int32_t* __restrict__ tri, int B, int V, int F, int H, int W,
                       float sx, float sy, unsigned long long* __restrict__ zbuf, Deferred d) {
    const uint32_t n = min(*d.count, d.cap);
    for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < n; q += gridDim.x * blockDim.x) {
        const unsigned long long e = d.list[q];
        TriSetup t; float4 p0, p1, p2; float err; int b, f;
        if (!exact_setup(pos, tri, V, F, (uint32_t)(e >> 32), t, p0, p1, p2, err, b, f)) continue;
        unsigned long long* zb = zbuf + (size_t)b * H * W;
        const uint32_t pix = (uint32_t)(e & 0xFFFFFFFFull);
        if (pix != 0xFFFFFFFFu) {
            const int py = (int)(pix / (uint32_t)W), px = (int)(pix - (uint32_t)py * (uint32_t)W);
            shade_pixel_exact(t, p0, p1, p2, err, f, px, py, sx, sy, zb + (size_t)py * W);
            continue;
        }
        int x0, y0, x1, y1;
        tri_bbox(p0, p1, p2, W, H, x0, y0, x1, y1);
        for (int py = y0; py <= y1; py++)
            for (int px = x0; px <= x1; px++) shade_pixel_exact(t, p0, p1, p2, err, f, px, py, sx, sy, zb + (size_t)py * W);
    }
}

// only when the deferred list overflowed: every triangle, exactly, over its whole box (atomicMin makes redoing the
// pixels already written harmless)
__global__ void __launch_bounds__(256)
raster_overflow_kernel(const float4* __restrict__ pos, const int32_t* __restrict__ tri, int B, int V, int F, int H, int W,
                       float sx, float sy, unsigned long long* __restrict__ zbuf, Deferred d) {
    if (*d.count <= d.cap) return;
    for (long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x; gid < (long long)B * F; gid += (long long)gridDim.x * blockDim.x) {
        TriSetup t; float4 p0, p1, p2; float err; int b, f;
        if (!exact_setup(pos, tri, V, F, (uint32_t)gid, t, p0, p1, p2, err, b, f)) continue;
        int x0, y0, x1, y1;
        tri_bbox(p0, p1, p2, W, H, x0, y0, x1, y1);
        unsigned long long* zb = zbuf + (size_t)b * H * W;
        for (int py = y0; py <= y1; py++)
            for (int px = x0; px <= x1; px++) shade_pixel_exact(t, p0, p1, p2, err, f, px, py, sx, sy, zb + (size_t)py * W);
    }
}

__global__ void __launch_bounds__(256)
raster_resolve_kernel(const float4* __restrict__ pos, const int32_t* __restrict__ tri, int B, int V, int H, int W,
                      float sx, float sy, const unsigned long long* __restrict__ zbuf, float4* __restrict__ rast,
                      float4* __restrict__ rast_db) {
    const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t npix = (size_t)B * H * W;
    if (pix >= npix) return;
    const unsigned long long key = zbuf[pix];
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f), d = make_float4(0.f, 0.f, 0.f, 0.f);
    if (key != 0xFFFFFFFFFFFFFFFFull) {
        const int f = (int)(uint32_t)(key & 0xFFFFFFFFull);
        const int b = (int)(pix / ((size_t)H * W));
        const int rem = (int)(pix - (size_t)b * H * W);
        const int py = rem / W, px = rem - py * W;
        const int i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
        const float4 p0 = pos[(size_t)b * V + i0], p1 = pos[(size_t)b * V + i1], p2 = pos[(size_t)b * V + i2];
        TriSetup t;
        tri_setup(p0, p1, p2, t);
        const float X = ((float)px + 0.5f) * sx - 1.0f, Y = ((float)py + 0.5f) * sy - 1.0f;
        const float e0 = (t.a0 * X + t.b0 * Y) + t.c0, e1 = (t.a1 * X + t.b1 * Y) + t.c1, e2 = (t.a2 * X + t.b2 * Y) + t.c2;
        const float S = e0 + e1 + e2;
        const float zw = ((t.z0 * e0 + t.z1 * e1) + t.z2 * e2) / t.det;
        // coverage is exact, so at a pixel within rounding of an edge the fp32 e_i may have the sign opposite to the
        // triangle's: it is then replaced by 0 (which is closer to the exact value) so that u, v, 1 - u - v >= 0
        const float sg = S < 0.f ? -1.f : 1.f;
        const float c0 = e0 * sg < 0.f ? 0.f : e0, c1 = e1 * sg < 0.f ? 0.f : e1, c2 = e2 * sg < 0.f ? 0.f : e2;
        const float Sc = c0 + c1 + c2;
        r = Sc != 0.f ? make_float4(c0 / Sc, c1 / Sc, zw, (float)(f + 1)) : make_float4(e0 / S, e1 / S, zw, (float)(f + 1));
        const float sa = t.a0 + t.a1 + t.a2, sb = t.b0 + t.b1 + t.b2, iS2 = 1.0f / (S * S);
        d = make_float4((t.a0 * S - e0 * sa) * iS2 * sx, (t.b0 * S - e0 * sb) * iS2 * sy,
                        (t.a1 * S - e1 * sa) * iS2 * sx, (t.b1 * S - e1 * sb) * iS2 * sy);
    }
    rast[pix] = r;
    rast_db[pix] = d;
}

// dL/dpos through u,v:  dL/dM[r][c] = -e_c/(S^2 det) * [ gu (A0r S - e0 SA_r) + gv (A1r S - e1 SA_r) ],
// M = [[x0,x1,x2],[y0,y1,y2],[w0,w1,w2]], A_kr = (a_k,b_k,c_k)[r], SA_r = sum_k A_kr.
__global__ void __launch_bounds__(256)
raster_backward_kernel(const float4* __restrict__ pos, const int32_t* __restrict__ tri, int B, int V, int H, int W,
                       float sx, float sy, const float4* __restrict__ rast, const float4* __restrict__ g,
                       float* __restrict__ dpos) {
    const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t npix = (size_t)B * H * W;
    if (pix >= npix) return;
    const float4 r = rast[pix];
    const int f = (int)r.w - 1;
    if (f < 0) return;
    const float gu = g[pix].x, gv = g[pix].y;
    if (gu == 0.f && gv == 0.f) return;
    const int b = (int)(pix / ((size_t)H * W));
    const int rem = (int)(pix - (size_t)b * H * W);
    const int py = rem / W, px = rem - py * W;
    const int vi[3] = {tri[3 * f], tri[3 * f + 1], tri[3 * f + 2]};
    const float4 p0 = pos[(size_t)b * V + vi[0]], p1 = pos[(size_t)b * V + vi[1]], p2 = pos[(size_t)b * V + vi[2]];
    TriSetup t;
    tri_setup(p0, p1, p2, t);
    const float X = ((float)px + 0.5f) * sx - 1.0f, Y = ((float)py + 0.5f) * sy - 1.0f;
    const float e[3] = {(t.a0 * X + t.b0 * Y) + t.c0, (t.a1 * X + t.b1 * Y) + t.c1, (t.a2 * X + t.b2 * Y) + t.c2};
    const float S = e[0] + e[1] + e[2];
    const float A0[3] = {t.a0, t.b0, t.c0}, A1[3] = {t.a1, t.b1, t.c1};
    const float SA[3] = {t.a0 + t.a1 + t.a2, t.b0 + t.b1 + t.b2, t.c0 + t.c1 + t.c2};
    const float k = -1.0f / (S * S * t.det);
    float br[3];
#pragma unroll
    for (int r3 = 0; r3 < 3; r3++) br[r3] = k * (gu * (A0[r3] * S - e[0] * SA[r3]) + gv * (A1[r3] * S - e[1] * SA[r3]));
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float* d = dpos + ((size_t)b * V + vi[c]) * 4;
        atomicAdd(d + 0, e[c] * br[0]);
        atomicAdd(d + 1, e[c] * br[1]);
        atomicAdd(d + 3, e[c] * br[2]);
    }
}

}  // namespace

// deferred-list capacity: two (triangle, pixel) pairs per triangle, far above what meshes need (the pairs are the
// pixels within rounding of an edge); beyond it the overflow pass stays correct, only slower
static size_t deferred_cap(int B, int F) { return (size_t)2 * B * F + 4096; }

extern "C" {

size_t dr_b200_rasterize_scratch_bytes(int32_t B, int32_t F, int32_t H, int32_t W) {
    return (size_t)B * H * W * 8 + 256 + deferred_cap(B, F) * 8 + (size_t)B * F * 4;
}

int32_t dr_b200_rasterize_fwd(const float* pos, const int32_t* tri, int32_t B, int32_t V, int32_t F, int32_t H, int32_t W,
                              float* rast, float* rast_db, void* scratch, void* stream) {
    GS_REQ(B >= 0 && V >= 0 && F >= 0 && H > 0 && W > 0, "bad sizes");
    GS_REQ(rast && rast_db && scratch && (F == 0 || (pos && tri)), "NULL pointer");
    GS_REQ(((size_t)pos & 15) == 0 && ((size_t)rast & 15) == 0 && ((size_t)rast_db & 15) == 0, "pos/rast must be 16-byte aligned");
    const cudaStream_t s = (cudaStream_t)stream;
    if (B <= 0 || H <= 0 || W <= 0) return 0;
    const size_t npix = (size_t)B * H * W;
    unsigned long long* zbuf = (unsigned long long*)scratch;
    uint32_t* qcount = (uint32_t*)((char*)scratch + npix * 8);
    Deferred d;
    d.count = qcount + 1;
    d.cap = (uint32_t)deferred_cap(B, F);
    d.list = (unsigned long long*)((char*)scratch + npix * 8 + 256);
    uint32_t* queue = (uint32_t*)(d.list + d.cap);
    GS_CUDA_CHECK(cudaMemsetAsync(zbuf, 0xFF, npix * 8, s));
    GS_CUDA_CHECK(cudaMemsetAsync(qcount, 0, 256, s));
    const float sx = (float)(2.0 / (double)W), sy = (float)(2.0 / (double)H);
    if (F > 0) {
        const long long nt = (long long)B * F;
        raster_small_kernel<<<(unsigned)((nt + 255) / 256), 256, 0, s>>>((const float4*)pos, tri, B, V, F, H, W, sx, sy, zbuf, queue, qcount, d);
        raster_large_kernel<<<GS_NUM_SMS * 4, 256, 0, s>>>((const float4*)pos, tri, B, V, F, H, W, sx, sy, zbuf, queue, qcount, d);
        raster_deferred_kernel<<<GS_NUM_SMS * 4, 256, 0, s>>>((const float4*)pos, tri, B, V, F, H, W, sx, sy, zbuf, d);
        raster_overflow_kernel<<<GS_NUM_SMS * 4, 256, 0, s>>>((const float4*)pos, tri, B, V, F, H, W, sx, sy, zbuf, d);
        gs_count_launches(4);
    }
    raster_resolve_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, s>>>((const float4*)pos, tri, B, V, H, W, sx, sy, zbuf,
                                                                          (float4*)rast, (float4*)rast_db);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int32_t dr_b200_rasterize_bwd(const float* pos, const int32_t* tri, int32_t B, int32_t V, int32_t F, int32_t H, int32_t W,
                              const float* rast, const float* dL_drast, float* dL_dpos, void* stream) {
    GS_REQ(pos && tri && rast && dL_drast && dL_dpos, "NULL pointer");
    const cudaStream_t s = (cudaStream_t)stream;
    if (B <= 0 || F <= 0) return 0;
    const size_t npix = (size_t)B * H * W;
    const float sx = (float)(2.0 / (double)W), sy = (float)(2.0 / (double)H);
    raster_backward_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, s>>>((const float4*)pos, tri, B, V, H, W, sx, sy,
                                                                           (const float4*)rast, (const float4*)dL_drast, dL_dpos);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

}  // extern "C"
