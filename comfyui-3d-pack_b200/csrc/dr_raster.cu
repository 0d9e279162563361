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
// THIS TU IS COMPILED WITH -fmad=false: coverage and z/w use the exact fp32 operation order of
// oracle/dr_oracle.py, so triangle ids are bit-exact against the oracle.
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

__device__ __forceinline__ bool edge_inside(float e, float a, float b, float sgn) {
    const float es = e * sgn, as = a * sgn, bs = b * sgn;
    return (es > 0.f) || ((es == 0.f) && ((as > 0.f) || ((as == 0.f) && (bs > 0.f))));
}

__device__ __forceinline__ uint32_t ordered_bits(float f) {
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ void shade_pixel(const TriSetup& t, int tri_id, int px, int py, float sx, float sy,
                                            unsigned long long* __restrict__ zrow) {
    const float X = ((float)px + 0.5f) * sx - 1.0f;
    const float Y = ((float)py + 0.5f) * sy - 1.0f;
    const float e0 = (t.a0 * X + t.b0 * Y) + t.c0;
    const float e1 = (t.a1 * X + t.b1 * Y) + t.c1;
    const float e2 = (t.a2 * X + t.b2 * Y) + t.c2;
    if (!(edge_inside(e0, t.a0, t.b0, t.sgn) && edge_inside(e1, t.a1, t.b1, t.sgn) && edge_inside(e2, t.a2, t.b2, t.sgn))) return;
    const float zw = ((t.z0 * e0 + t.z1 * e1) + t.z2 * e2) / t.det;
    if (!(zw >= -1.0f && zw <= 1.0f)) return;
    const unsigned long long key = ((unsigned long long)ordered_bits(zw) << 32) | (unsigned long long)(uint32_t)tri_id;
    atomicMin(zrow + px, key);
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
                    uint32_t* __restrict__ qcount) {
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (long long)B * F) return;
    const int b = (int)(gid / F), f = (int)(gid - (long long)b * F);
    const int i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
    if ((unsigned)i0 >= (unsigned)V || (unsigned)i1 >= (unsigned)V || (unsigned)i2 >= (unsigned)V) return;
    const float4 p0 = pos[(size_t)b * V + i0], p1 = pos[(size_t)b * V + i1], p2 = pos[(size_t)b * V + i2];
    TriSetup t;
    if (!tri_setup(p0, p1, p2, t)) return;
    int x0, y0, x1, y1;
    tri_bbox(p0, p1, p2, W, H, x0, y0, x1, y1);
    if (x1 < x0 || y1 < y0) return;
    if ((x1 - x0 + 1) * (y1 - y0 + 1) > LARGE_AREA) {
        const uint32_t slot = atomicAdd(qcount, 1u);
        queue[slot] = (uint32_t)gid;                    // capacity B*F
        return;
    }
    unsigned long long* zb = zbuf + (size_t)b * H * W;
    for (int py = y0; py <= y1; py++)
        for (int px = x0; px <= x1; px++) shade_pixel(t, f, px, py, sx, sy, zb + (size_t)py * W);
}

__global__ void __launch_bounds__(256)
raster_large_kernel(const float4* __restrict__ pos, const int32_t* __restrict__ tri, int B, int V, int F, int H, int W,
                    float sx, float sy, unsigned long long* __restrict__ zbuf, const uint32_t* __restrict__ queue,
                    const uint32_t* __restrict__ qcount) {
    const uint32_t n = *qcount;
    for (uint32_t q = blockIdx.x; q < n; q += gridDim.x) {
        const uint32_t gid = queue[q];
        const int b = (int)(gid / (uint32_t)F), f = (int)(gid - (uint32_t)b * (uint32_t)F);
        const int i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
        const float4 p0 = pos[(size_t)b * V + i0], p1 = pos[(size_t)b * V + i1], p2 = pos[(size_t)b * V + i2];
        TriSetup t;
        tri_setup(p0, p1, p2, t);
        int x0, y0, x1, y1;
        tri_bbox(p0, p1, p2, W, H, x0, y0, x1, y1);
        const int bw = x1 - x0 + 1, total = bw * (y1 - y0 + 1);
        unsigned long long* zb = zbuf + (size_t)b * H * W;
        for (int i = threadIdx.x; i < total; i += blockDim.x) {
            const int py = y0 + i / bw, px = x0 + i - (i / bw) * bw;
            shade_pixel(t, f, px, py, sx, sy, zb + (size_t)py * W);
        }
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
        r = make_float4(e0 / S, e1 / S, zw, (float)(f + 1));
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

size_t dr_rasterize_scratch_bytes(int B, int F, int H, int W) {
    return (size_t)B * H * W * 8 + (size_t)B * F * 4 + 256;
}

int dr_launch_rasterize_fwd(const float* pos, const int32_t* tri, int B, int V, int F, int H, int W, float* rast,
                            float* rast_db, void* scratch, cudaStream_t s) {
    if (B <= 0 || H <= 0 || W <= 0) return 0;
    const size_t npix = (size_t)B * H * W;
    unsigned long long* zbuf = (unsigned long long*)scratch;
    uint32_t* qcount = (uint32_t*)((char*)scratch + npix * 8);
    uint32_t* queue = qcount + 64;
    GS_CUDA_CHECK(cudaMemsetAsync(zbuf, 0xFF, npix * 8, s));
    GS_CUDA_CHECK(cudaMemsetAsync(qcount, 0, 256, s));
    const float sx = (float)(2.0 / (double)W), sy = (float)(2.0 / (double)H);
    if (F > 0) {
        const long long nt = (long long)B * F;
        raster_small_kernel<<<(unsigned)((nt + 255) / 256), 256, 0, s>>>((const float4*)pos, tri, B, V, F, H, W, sx, sy, zbuf, queue, qcount);
        raster_large_kernel<<<GS_NUM_SMS * 4, 256, 0, s>>>((const float4*)pos, tri, B, V, F, H, W, sx, sy, zbuf, queue, qcount);
        gs_count_launches(2);
    }
    raster_resolve_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, s>>>((const float4*)pos, tri, B, V, H, W, sx, sy, zbuf,
                                                                          (float4*)rast, (float4*)rast_db);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int dr_launch_rasterize_bwd(const float* pos, const int32_t* tri, int B, int V, int F, int H, int W, const float* rast,
                            const float* dL_drast, float* dL_dpos, cudaStream_t s) {
    if (B <= 0 || F <= 0) return 0;
    const size_t npix = (size_t)B * H * W;
    const float sx = (float)(2.0 / (double)W), sy = (float)(2.0 / (double)H);
    raster_backward_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, s>>>((const float4*)pos, tri, B, V, H, W, sx, sy,
                                                                           (const float4*)rast, (const float4*)dL_drast, dL_dpos);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
