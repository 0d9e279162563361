// StableFast3D's UV texture baker (sf3d/texture_baker.py's TextureBaker over texture_baker.slang: bake_uv and
// interpolate), with every output bit identical to the reference's own kernels, i.e. the CUDA slangtorch generates from
// texture_baker.slang as nvcc 12.9 compiles it for sm_90a with default flags (FMA contraction on, IEEE division).
//
// Contract, read off that build's SASS (INTEGRATION §3).  out[res,res,4]; the launched region is rows x cols texels.
//   Texel (row, col):  x = sat(fl(col / res)),  y = 1 - sat(fl(row / res))      (IEEE division, no half-texel offset)
//   Face i, vertices a = uv[f.x], b = uv[f.y], c = uv[f.z]:
//     e1 = b - a,  e2 = c - a,  q = (x, y) - a                                  (one rounding each)
//     dot(s, t) = fma(s.y, t.y, fma(s.x, t.x, +0))  -- a zero product is +0, never -0
//     d00 = dot(e1, e1), d01 = dot(e1, e2), d11 = dot(e2, e2), d20 = dot(q, e1), d21 = dot(q, e2)
//     denom = fma(d00, d11, -(d01*d01))
//     v = fma(d11, d20, -(d01*d21)) / denom,  w = fma(d00, d21, -(d01*d20)) / denom   (IEEE division)
//     u = (1 - v) - w;  hit iff v >= 0 && w >= 0 && v + w <= 1
//   The smallest hitting face index wins (the reference loops i = 0.. and stops at the first hit): out = (u, v, w,
//   (float)i), i converted round-to-nearest, so i is inexact above 2^24.  No hit: (0, 0, 0, -1).
//   interpolate: i = (int)rast.w (truncating; NaN gives 0, out-of-range saturates); i < 0 gives 0; otherwise per
//   channel fma(rast.z, attr[f.z], fma(rast.x, attr[f.x], rast.y * attr[f.y])).
//   Texels outside the launched region are not written.
// Deviations, where the reference is undefined: a face with a vertex id out of range is skipped; an interpolate whose
// face or vertex id is out of range writes 0; a region larger than the texture is clipped to it.
// THIS TU IS COMPILED WITH -fmad=false: the contractions above are spelled out with __fmaf_rn, every other operation
// is rounded once, in the order written.
//
// Algorithm: one thread per face computes a conservative candidate-texel box (below) and rasterizes it itself or queues
// the face for a warp or a CTA by the box's size; every candidate texel runs the exact test above and a hit does
// atomicMin(winner[texel], i), so the result does not depend on the order the atomics land in.  A per-texel resolve
// recomputes (u, v, w) for the winner with the same arithmetic.  4 B of scratch per texel plus 8 B per face.
//
// The candidate box.  Write E1, E2, Q for the exact differences (e1, e2, q are them rounded), D = (E1 x E2)^2 for the
// exact denominator and P = |E1|^2 |E2|^2 >= D.  Standard error bounds (u = 2^-24, one rounding per operation) give
//   d00 = |E1|^2 (1 + t), |t| <= 4.01u (likewise d11);  |d01 - E1.E2| <= 4.01u |E1||E2|;  |d20 - Q.E1| <= 4.01u |Q||E1|
//   |denom - D| <= 18.1u P,  so with K = d00 d11 / denom (computed):  |denom/D - 1| <= 19u K  when u K << 1;
//   |vnum - (E1 x E2)(Q x E2)| <= 18.1u |E1||E2|^2 |Q|,  |wnum - ...| <= 18.1u |E1|^2 |E2| |Q|.
// An accepted texel has v, w >= -0 and v + w <= 1 + u, so |v| <= 1 + u, and then (K <= 2^14 keeps 19uK <= 0.019)
//   |v - v*| <= 1.05 (u + 19u K + 18.4u K |Q|/|E1|) <= 22u K (1 + R/|E1|) =: ev,   likewise ew with |E2|,
// where v*, w* are p's exact barycentrics and R >= |Q| bounds the distance from a to any point of [0,1]^2 (x and y are
// always in [0,1]).  So an accepted p = a + v* E1 + w* E2 has v* >= -ev, w* >= -ew, v* + w* <= 1 + u + ev + ew: it lies
// in the triangle grown by at most et = 2(ev + ew) + u times |E1.x| + |E2.x| in x (|E1.y| + |E2.y| in y).  The kernel
// uses 64u K instead of 22u K, which also covers the roundings of the bound itself, adds 2^-60 for underflow in the dot
// products (d00, d11 >= 2^-60 are required), and pads the texel range by 2 for the rounding of x and y.
// Every face this does not cover goes to a whole-texture path, which tests every texel of the region: K > 2^14 (an
// angle at a below ~0.45 degrees), denom < 0, d00 or d11 outside [2^-60, 2^60], or a non-finite bound.  A face with
// denom == 0 or NaN, or a non-finite UV (which makes denom NaN), can never hit (v or w is then NaN or +-inf, or
// v + w = +inf) and is dropped.
#include "gs_common.cuh"

namespace {

constexpr uint32_t UB_EMPTY = 0xffffffffu;
constexpr long long UB_WARP_AREA = 256;     // boxes above this go to the warp queue
constexpr long long UB_CTA_AREA = 8192;     // ... and above this to the CTA queue
constexpr float UB_U = 5.9604644775390625e-8f;      // 2^-24
constexpr float UB_KMAX = 16384.0f;                 // 2^14
constexpr float UB_TINY = 8.673617379884035e-19f;   // 2^-60
constexpr float UB_HUGE = 1.152921504606847e18f;    // 2^60

struct Face {
    float ax, ay, e1x, e1y, e2x, e2y, d00, d01, d11, denom;
};

__device__ __forceinline__ float dot2(float sx, float sy, float tx, float ty) {
    return __fmaf_rn(sy, ty, __fmaf_rn(sx, tx, 0.0f));
}

// false: a vertex id is out of range
__device__ __forceinline__ bool face_setup(const float2* __restrict__ uv, int NV, const int32_t* __restrict__ T, uint32_t f,
                                           Face& s) {
    const int i0 = T[3 * (size_t)f], i1 = T[3 * (size_t)f + 1], i2 = T[3 * (size_t)f + 2];
    if ((unsigned)i0 >= (unsigned)NV || (unsigned)i1 >= (unsigned)NV || (unsigned)i2 >= (unsigned)NV) return false;
    const float2 a = uv[i0], b = uv[i1], c = uv[i2];
    s.ax = a.x; s.ay = a.y;
    s.e1x = b.x - a.x; s.e1y = b.y - a.y;
    s.e2x = c.x - a.x; s.e2y = c.y - a.y;
    s.d00 = dot2(s.e1x, s.e1y, s.e1x, s.e1y);
    s.d01 = dot2(s.e1x, s.e1y, s.e2x, s.e2y);
    s.d11 = dot2(s.e2x, s.e2y, s.e2x, s.e2y);
    s.denom = __fmaf_rn(s.d00, s.d11, -(s.d01 * s.d01));
    return true;
}

__device__ __forceinline__ float texel_x(int col, int res) { return __saturatef(__fdiv_rn((float)col, (float)res)); }
__device__ __forceinline__ float texel_y(int row, int res) { return 1.0f - __saturatef(__fdiv_rn((float)row, (float)res)); }

// the reference's barycentric test at (x, y); v and w as it computes them
__device__ __forceinline__ bool bary(const Face& s, float x, float y, float& v, float& w) {
    const float qx = x - s.ax, qy = y - s.ay;
    const float d20 = dot2(qx, qy, s.e1x, s.e1y), d21 = dot2(qx, qy, s.e2x, s.e2y);
    v = __fdiv_rn(__fmaf_rn(s.d11, d20, -(s.d01 * d21)), s.denom);
    w = __fdiv_rn(__fmaf_rn(s.d00, d21, -(s.d01 * d20)), s.denom);
    return v >= 0.0f && w >= 0.0f && v + w <= 1.0f;
}

__device__ __forceinline__ void shade(const Face& s, uint32_t f, int row, int col, int res, int cols,
                                      uint32_t* __restrict__ winner) {
    float v, w;
    if (bary(s, texel_x(col, res), texel_y(row, res), v, w)) atomicMin(winner + (size_t)row * cols + col, f);
}

enum { UB_DROP = 0, UB_BOX = 1, UB_WHOLE = 2 };

// the candidate texels [r0, r1] x [c0, c1] of a face (header), clipped to the region; UB_DROP when it can never hit
__device__ __forceinline__ int face_box(const Face& s, const float2* __restrict__ uv, const int32_t* __restrict__ T,
                                        uint32_t f, int res, int rows, int cols, int& r0, int& r1, int& c0, int& c1) {
    r0 = 0; r1 = rows - 1; c0 = 0; c1 = cols - 1;
    const float2 b = uv[T[3 * (size_t)f + 1]], c = uv[T[3 * (size_t)f + 2]];
    if (!(isfinite(s.ax) && isfinite(s.ay) && isfinite(b.x) && isfinite(b.y) && isfinite(c.x) && isfinite(c.y)))
        return UB_DROP;
    if (!(s.denom != 0.0f)) return UB_DROP;                             // 0 or NaN
    if (!(s.denom > 0.0f && s.d00 >= UB_TINY && s.d11 >= UB_TINY && s.d00 <= UB_HUGE && s.d11 <= UB_HUGE))
        return UB_WHOLE;
    const float K = s.d00 * s.d11 / s.denom;
    if (!(K <= UB_KMAX)) return UB_WHOLE;
    const float rx = fmaxf(fabsf(s.ax), fabsf(1.0f - s.ax)), ry = fmaxf(fabsf(s.ay), fabsf(1.0f - s.ay));
    const float R = sqrtf(rx * rx + ry * ry);
    const float ev = 64.0f * UB_U * K * (1.0f + R / sqrtf(s.d00)) + UB_TINY;
    const float ew = 64.0f * UB_U * K * (1.0f + R / sqrtf(s.d11)) + UB_TINY;
    const float et = 2.0f * (ev + ew) + 4.0f * UB_U;
    const float mx = et * (fabsf(s.e1x) + fabsf(s.e2x)) * 1.01f + UB_TINY;
    const float my = et * (fabsf(s.e1y) + fabsf(s.e2y)) * 1.01f + UB_TINY;
    if (!(mx < 2.0f && my < 2.0f)) return UB_WHOLE;                     // covers [0,1]^2 anyway (and catches inf)
    const float xlo = fmaxf(fminf(s.ax, fminf(b.x, c.x)) - mx, 0.0f), xhi = fminf(fmaxf(s.ax, fmaxf(b.x, c.x)) + mx, 1.0f);
    const float ylo = fmaxf(fminf(s.ay, fminf(b.y, c.y)) - my, 0.0f), yhi = fminf(fmaxf(s.ay, fmaxf(b.y, c.y)) + my, 1.0f);
    if (xlo > xhi || ylo > yhi) return UB_DROP;                         // no point of [0,1]^2 can be accepted
    const float fr = (float)res;
    c0 = max(c0, (int)floorf(xlo * fr) - 2);
    c1 = min(c1, (int)ceilf(xhi * fr) + 2);
    r0 = max(r0, (int)floorf((1.0f - yhi) * fr) - 2);                   // y = 1 - row/res, decreasing in row
    r1 = min(r1, (int)ceilf((1.0f - ylo) * fr) + 2);
    return (c0 <= c1 && r0 <= r1) ? UB_BOX : UB_DROP;
}

__global__ void __launch_bounds__(256) ub_init_kernel(uint32_t* __restrict__ winner, size_t n, uint32_t* __restrict__ counts) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 4) counts[i] = 0u;
    if (i < n) winner[i] = UB_EMPTY;
}

// one thread per face: small boxes are rasterized here, larger ones queued (whole-texture faces with the CTA queue)
__global__ void __launch_bounds__(256)
ub_small_kernel(const float2* __restrict__ uv, int NV, const int32_t* __restrict__ T, int NF, int res, int rows, int cols,
                uint32_t* __restrict__ winner, uint32_t* __restrict__ qwarp, uint32_t* __restrict__ qcta,
                uint32_t* __restrict__ counts) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= (uint32_t)NF) return;
    Face s;
    if (!face_setup(uv, NV, T, f, s)) return;
    int r0, r1, c0, c1;
    const int kind = face_box(s, uv, T, f, res, rows, cols, r0, r1, c0, c1);
    if (kind == UB_DROP) return;
    const long long area = (long long)(r1 - r0 + 1) * (c1 - c0 + 1);
    if (kind == UB_WHOLE) atomicAdd(counts + 2, 1u);
    if (kind == UB_WHOLE || area > UB_CTA_AREA) { qcta[atomicAdd(counts + 1, 1u)] = f; return; }
    if (area > UB_WARP_AREA) { qwarp[atomicAdd(counts, 1u)] = f; return; }
    for (int row = r0; row <= r1; row++)
        for (int col = c0; col <= c1; col++) shade(s, f, row, col, res, cols, winner);
}

// persistent grid: each warp drains faces of the warp queue; then the CTAs share the faces of the CTA queue.  With
// fewer such faces than CTAs each face gets gridDim.x / n CTAs, which split its box; otherwise each CTA takes whole
// faces in turn.  The split is decided on the device from the queue's length.
__global__ void __launch_bounds__(256)
ub_large_kernel(const float2* __restrict__ uv, int NV, const int32_t* __restrict__ T, int res, int rows, int cols,
                uint32_t* __restrict__ winner, const uint32_t* __restrict__ qwarp, const uint32_t* __restrict__ qcta,
                const uint32_t* __restrict__ counts) {
    const uint32_t nwarp = counts[0], ncta = counts[1];
    const int lane = threadIdx.x & 31;
    const uint32_t warps = gridDim.x * (blockDim.x >> 5);
    for (uint32_t q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); q < nwarp; q += warps) {
        const uint32_t f = qwarp[q];
        Face s;
        face_setup(uv, NV, T, f, s);
        int r0, r1, c0, c1;
        face_box(s, uv, T, f, res, rows, cols, r0, r1, c0, c1);
        const int bw = c1 - c0 + 1, total = bw * (r1 - r0 + 1);
        for (int i = lane; i < total; i += 32) {
            const int r = i / bw;
            shade(s, f, r0 + r, c0 + i - r * bw, res, cols, winner);
        }
    }
    if (ncta == 0) return;
    uint32_t q0 = blockIdx.x, qstep = gridDim.x, part = 0, parts = 1;
    if (ncta <= gridDim.x) {
        parts = gridDim.x / ncta;
        q0 = blockIdx.x % ncta; part = blockIdx.x / ncta; qstep = ncta;
        if (part >= parts) return;
    }
    for (uint32_t q = q0; q < ncta; q += qstep) {
        const uint32_t f = qcta[q];
        Face s;
        face_setup(uv, NV, T, f, s);
        int r0, r1, c0, c1;
        face_box(s, uv, T, f, res, rows, cols, r0, r1, c0, c1);
        const long long bw = c1 - c0 + 1, total = bw * (r1 - r0 + 1);
        const long long stride = (long long)parts * blockDim.x;
        for (long long i = (long long)part * blockDim.x + threadIdx.x; i < total; i += stride) {
            const long long r = i / bw;
            shade(s, f, r0 + (int)r, c0 + (int)(i - r * bw), res, cols, winner);
        }
    }
}

// per texel of the region: the winner's (u, v, w, i), recomputed with the test's arithmetic, or (0, 0, 0, -1)
__global__ void __launch_bounds__(256)
ub_resolve_kernel(const float2* __restrict__ uv, int NV, const int32_t* __restrict__ T, int res, int rows, int cols,
                  const uint32_t* __restrict__ winner, float4* __restrict__ out) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)rows * cols) return;
    const int row = (int)(t / cols), col = (int)(t - (size_t)row * cols);
    const uint32_t f = winner[t];
    float4 o = make_float4(0.0f, 0.0f, 0.0f, -1.0f);
    if (f != UB_EMPTY) {
        Face s;
        face_setup(uv, NV, T, f, s);
        float v, w;
        bary(s, texel_x(col, res), texel_y(row, res), v, w);
        o = make_float4((1.0f - v) - w, v, w, (float)(int)f);
    }
    out[(size_t)row * res + col] = o;
}

// per texel of the region: the reference's interpolate, with out-of-range face or vertex ids giving 0
__global__ void __launch_bounds__(256)
ub_interp_kernel(const float* __restrict__ attr, int NV, const int32_t* __restrict__ T, int NF, const float4* __restrict__ rast,
                 int res, int rows, int cols, float* __restrict__ out) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)rows * cols) return;
    const int row = (int)(t / cols), col = (int)(t - (size_t)row * cols);
    const size_t texel = (size_t)row * res + col;
    const float4 r = rast[texel];
    const int i = __float2int_rz(r.w);                  // cvt.rzi: NaN gives 0, out-of-range saturates
    float* o = out + 3 * texel;
    int v0 = -1, v1 = -1, v2 = -1;
    if (i >= 0 && i < NF) { v0 = T[3 * (size_t)i]; v1 = T[3 * (size_t)i + 1]; v2 = T[3 * (size_t)i + 2]; }
    if ((unsigned)v0 >= (unsigned)NV || (unsigned)v1 >= (unsigned)NV || (unsigned)v2 >= (unsigned)NV) {
        o[0] = 0.0f; o[1] = 0.0f; o[2] = 0.0f;
        return;
    }
    const float *a1 = attr + 3 * (size_t)v0, *a2 = attr + 3 * (size_t)v1, *a3 = attr + 3 * (size_t)v2;
#pragma unroll
    for (int c = 0; c < 3; c++) o[c] = __fmaf_rn(r.z, a3[c], __fmaf_rn(r.x, a1[c], r.y * a2[c]));
}

}  // namespace

size_t ub_scratch_bytes(int F, int res) { return 256 + (size_t)res * res * 4 + (size_t)F * 8; }

int ub_launch_rasterize(const float* uv, int NV, const int32_t* T, int NF, float* out, int res, int rows, int cols,
                        void* scratch, cudaStream_t s) {
    if (rows <= 0 || cols <= 0) return 0;
    const size_t n = (size_t)rows * cols;
    uint32_t* counts = (uint32_t*)scratch;
    uint32_t* winner = (uint32_t*)((char*)scratch + 256);
    uint32_t* qwarp = winner + (size_t)res * res;
    uint32_t* qcta = qwarp + NF;
    ub_init_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(winner, n, counts);
    if (NF > 0) {
        ub_small_kernel<<<(unsigned)((NF + 255) / 256), 256, 0, s>>>((const float2*)uv, NV, T, NF, res, rows, cols, winner,
                                                                     qwarp, qcta, counts);
        ub_large_kernel<<<GS_NUM_SMS * 8, 256, 0, s>>>((const float2*)uv, NV, T, res, rows, cols, winner, qwarp, qcta, counts);
        gs_count_launches(2);
    }
    ub_resolve_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>((const float2*)uv, NV, T, res, rows, cols, winner,
                                                                   (float4*)out);
    gs_count_launches(2);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int ub_launch_interpolate(const float* attr, int NV, const int32_t* T, int NF, const float* rast, float* out, int res,
                          int rows, int cols, cudaStream_t s) {
    if (rows <= 0 || cols <= 0) return 0;
    const size_t n = (size_t)rows * cols;
    ub_interp_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(attr, NV, T, NF, (const float4*)rast, res, rows, cols, out);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
