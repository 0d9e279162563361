// Forward per-Gaussian preprocess: project + cull + EWA cov2D + extent + tile
// rect + SH->RGB, fused into one pass that emits the 48 B splat record.
//
// Replaces preprocessCUDA of diff_gaussian_rasterization (called from
// main_3DGS_renderer.py:927-936).  Algorithm per SURVEY.md App. A.1.1-4.
//
// THIS TRANSLATION UNIT IS COMPILED WITH -fmad=false: every value that decides
// an integer output (cull, radius, rect, depth bits -> keys) is computed with the
// exact IEEE fp32 operation order of oracle/gs_oracle.py::preprocess, so keys,
// radii and tile lists are bit-exact against the oracle.  The kernel is HBM
// bound (reads 4*(3+3+4+1+3M) B, writes 64 B per Gaussian), so losing FMA
// contraction here costs nothing.
#include "gs_common.cuh"

namespace {

__device__ __forceinline__ void sh_to_rgb(int deg, const float* __restrict__ sh, float dx, float dy, float dz, float& r,
                                          float& g, float& b) {
    // sh: [M,3] of this Gaussian.  Basis as shared_utils/sh_utils.py:57-112; gs_sh_colour is shared with the backward
    float rgb[3];
    gs_sh_colour(deg, sh, dx, dy, dz, rgb);
    r = fmaxf(rgb[0], 0.f); g = fmaxf(rgb[1], 0.f); b = fmaxf(rgb[2], 0.f);
}

constexpr int PP_THREADS = 128;

struct ViewK {                      // per-view constants, matrices in shared memory
    const float* m; const float* p; const float* cam;
    float tanfovx, tanfovy, fx, fy;
    int W, H, tiles_x, tiles_y;
};

// Sigma = R diag(s^2) R^T packed [xx,xy,xz,yy,yz,zz]; order of operations is part of the bit-exactness contract.
__device__ __forceinline__ void cov3d_of(const float* __restrict__ scales, const float* __restrict__ rotations,
                                         const float* __restrict__ cov3D_precomp, float mod, int idx, float c[6]) {
    if (cov3D_precomp != nullptr) {
        const float* cp = cov3D_precomp + 6 * (size_t)idx;
#pragma unroll
        for (int k = 0; k < 6; k++) c[k] = cp[k];
        return;
    }
    const float s0 = mod * scales[3 * idx + 0], s1 = mod * scales[3 * idx + 1], s2 = mod * scales[3 * idx + 2];
    const float* q = rotations + 4 * (size_t)idx;
    const float r = q[0], qx = q[1], qy = q[2], qz = q[3];
    const float R00 = 1.0f - 2.0f * (qy * qy + qz * qz), R01 = 2.0f * (qx * qy - r * qz), R02 = 2.0f * (qx * qz + r * qy);
    const float R10 = 2.0f * (qx * qy + r * qz), R11 = 1.0f - 2.0f * (qx * qx + qz * qz), R12 = 2.0f * (qy * qz - r * qx);
    const float R20 = 2.0f * (qx * qz - r * qy), R21 = 2.0f * (qy * qz + r * qx), R22 = 1.0f - 2.0f * (qx * qx + qy * qy);
    const float M00 = R00 * s0, M01 = R01 * s1, M02 = R02 * s2;
    const float M10 = R10 * s0, M11 = R11 * s1, M12 = R12 * s2;
    const float M20 = R20 * s0, M21 = R21 * s1, M22 = R22 * s2;
    c[0] = M00 * M00 + M01 * M01 + M02 * M02;
    c[1] = M00 * M10 + M01 * M11 + M02 * M12;
    c[2] = M00 * M20 + M01 * M21 + M02 * M22;
    c[3] = M10 * M10 + M11 * M11 + M12 * M12;
    c[4] = M10 * M20 + M11 * M21 + M12 * M22;
    c[5] = M20 * M20 + M21 * M21 + M22 * M22;
}

// Optional tight tile list ("tile culling").  The package lists every tile of the 3-sigma bounding square; most of
// those (tile, splat) pairs cannot reach alpha >= 1/255 anywhere in the tile and only cost sort / staging work.
// Here the exact level set  q(u) = 0.5(A ux^2 + C uy^2) + B ux uy <= log2(255 o)  (log2-scaled conic, same
// conservative slack as the composite's sub-rect mask) is intersected with each tile row of the square:
// x-extent of the ellipse inside the row's y-strip -> a span of tiles.  Result: 8 rows x (start-x0 | count<<8)
// packed in a uint4, or spans.x = 0xFFFFFFFF for "whole square" (big squares, degenerate conics).
// Pruned pairs contribute to no pixel, so images are bit-identical; only list positions (n_contrib) shift.
__device__ __forceinline__ void tight_spans(float px, float py, const float4 cq, int x0, int y0, int x1, int y1,
                                            uint32_t& count, uint4& spans) {
    spans = make_uint4(0xFFFFFFFFu, 0u, 0u, 0u);
    const int w = x1 - x0, h = y1 - y0;
    if (w > 255 || h > 8) return;
    const float o = cq.w;
    if (!(o * 255.0f >= 1.0f)) { count = 0; spans = make_uint4(0u, 0u, 0u, 0u); return; }
    const float tau = log2f(o * 255.0f) * 1.001f + 0.03f;
    const float A = -2.0f * cq.x, B = -cq.y, C = -2.0f * cq.z;
    const float det = A * C - B * B;
    if (!(A > 0.f && det > 0.f)) return;
    const float inv_det = 1.0f / det, invA = 1.0f / A;
    const float k2 = 2.0f * tau * A;
    const float Ymax = sqrtf(k2 * inv_det), Xmax = sqrtf(2.0f * tau * C * inv_det);
    const float uyR = -(B * Xmax) / C;                      // y offset of the right-most point of the ellipse
    if (!(isfinite(Ymax) && isfinite(Xmax) && isfinite(uyR) && isfinite(px) && isfinite(py))) return;
    // rows beyond h are never visited (typical squares are 2-4 tiles high); entries are packed with 64-bit shifts so
    // the loop needs no dynamically indexed array
    unsigned long long lo64 = 0ull, hi64 = 0ull;
    uint32_t total = 0;
    for (int r = 0; r < h; r++) {
        uint32_t cnt = 0, start = 0;
        const float a = (float)((y0 + r) * GS_TILE) - py, b = a + (float)(GS_TILE - 1);
        const float lo = fmaxf(a, -Ymax), hi = fminf(b, Ymax);
        if (lo <= hi) {
            const float yr = fminf(fmaxf(uyR, lo), hi), yl = fminf(fmaxf(-uyR, lo), hi);
            float xr = (-(B * yr) + sqrtf(fmaxf(k2 - det * yr * yr, 0.f))) * invA;
            float xl = (-(B * yl) - sqrtf(fmaxf(k2 - det * yl * yl, 0.f))) * invA;
            xr += 0.01f + 1e-4f * fabsf(xr);
            xl -= 0.01f + 1e-4f * fabsf(xl);
            const int ta = max(x0, (int)ceilf((px + xl - (float)(GS_TILE - 1)) * (1.0f / GS_TILE)));
            const int tb = min(x1 - 1, (int)floorf((px + xr) * (1.0f / GS_TILE)));
            if (tb >= ta) { cnt = (uint32_t)(tb - ta + 1); start = (uint32_t)(ta - x0); }
        }
        const unsigned long long e = (unsigned long long)(start | (cnt << 8));
        if (r < 4) lo64 |= e << (16 * r); else hi64 |= e << (16 * (r - 4));
        total += cnt;
    }
    uint32_t packed[4] = {(uint32_t)lo64, (uint32_t)(lo64 >> 32), (uint32_t)hi64, (uint32_t)(hi64 >> 32)};
    count = total;
    spans = make_uint4(packed[0], packed[1], packed[2], packed[3]);
}

// View-dependent part for one Gaussian: cull, project, EWA cov2D, extent, rect, colour -> record.
__device__ __forceinline__ void project_view(const ViewK& vk, int deg, int M, float x, float y, float z,
                                             const float c[6], float opacity, const float* __restrict__ sh_row,
                                             const float* __restrict__ col, SplatRec& rec, int& my_radius,
                                             uint32_t& tiles, uint32_t& dkey, bool tight, uint4& spans) {
    const float* m = vk.m;
    const float* p = vk.p;
    rec.g = make_float4(0.f, 0.f, 0.f, 0.f);
    rec.c = make_float4(0.f, 0.f, 0.f, 0.f);
    rec.k = make_float4(0.f, 0.f, 0.f, 0.f);
    my_radius = 0; tiles = 0; dkey = 0xFFFFFFFFu;
    spans = make_uint4(0u, 0u, 0u, 0u);
    const float tx = m[0] * x + m[4] * y + m[8] * z + m[12];
    const float ty = m[1] * x + m[5] * y + m[9] * z + m[13];
    const float tz = m[2] * x + m[6] * y + m[10] * z + m[14];
    if (!(tz > 0.2f)) return;
    const float hx = p[0] * x + p[4] * y + p[8] * z + p[12];
    const float hy = p[1] * x + p[5] * y + p[9] * z + p[13];
    const float hw = p[3] * x + p[7] * y + p[11] * z + p[15];
    const float pw = 1.0f / (hw + 0.0000001f);
    const float ndcx = hx * pw, ndcy = hy * pw;
    const float c0 = c[0], c1 = c[1], c2 = c[2], c3 = c[3], c4 = c[4], c5 = c[5];
    const float fx = vk.fx, fy = vk.fy;
    const float limx = 1.3f * vk.tanfovx, limy = 1.3f * vk.tanfovy;
    const float txtz = tx / tz, tytz = ty / tz;
    const float cx = fminf(limx, fmaxf(-limx, txtz)) * tz;
    const float cy = fminf(limy, fmaxf(-limy, tytz)) * tz;
    const float J00 = fx / tz, J02 = -(fx * cx) / (tz * tz);
    const float J11 = fy / tz, J12 = -(fy * cy) / (tz * tz);
    const float T00 = J00 * m[0] + J02 * m[2], T01 = J00 * m[4] + J02 * m[6], T02 = J00 * m[8] + J02 * m[10];
    const float T10 = J11 * m[1] + J12 * m[2], T11 = J11 * m[5] + J12 * m[6], T12 = J11 * m[9] + J12 * m[10];
    const float v00 = c0 * T00 + c1 * T01 + c2 * T02;
    const float v01 = c1 * T00 + c3 * T01 + c4 * T02;
    const float v02 = c2 * T00 + c4 * T01 + c5 * T02;
    const float v10 = c0 * T10 + c1 * T11 + c2 * T12;
    const float v11 = c1 * T10 + c3 * T11 + c4 * T12;
    const float v12 = c2 * T10 + c4 * T11 + c5 * T12;
    const float ca = T00 * v00 + T01 * v01 + T02 * v02 + 0.3f;
    const float cb = T00 * v10 + T01 * v11 + T02 * v12;
    const float cc = T10 * v10 + T11 * v11 + T12 * v12 + 0.3f;
    const float det = ca * cc - cb * cb;
    if (det == 0.0f) return;
    const float det_inv = 1.0f / det;
    const float mid = 0.5f * (ca + cc);
    const float disc = sqrtf(fmaxf(mid * mid - det, 0.1f));
    const float lam1 = mid + disc, lam2 = mid - disc;
    const float radf = ceilf(3.0f * sqrtf(fmaxf(lam1, lam2)));
    // A NaN extent (a NaN or non-positive-definite covariance: an overflowed scale, a bad cov3D_precomp) is culled.
    // Converted, it would be radius 0 with a one-tile rect that the emit (radius > 0 only) never fills.  Finite
    // extents are >= 1 here; +inf, like any extent past INT_MAX, saturates to INT_MAX: a full-screen square.
    if (!(radf > 0.0f)) return;
    const float px = ((ndcx + 1.0f) * (float)vk.W - 1.0f) * 0.5f;
    const float py = ((ndcy + 1.0f) * (float)vk.H - 1.0f) * 0.5f;
    const int rad_i = __float2int_rz(radf);
    int x0, y0, x1, y1;
    get_rect(px, py, rad_i, vk.tiles_x, vk.tiles_y, x0, y0, x1, y1);
    const int area = (x1 - x0) * (y1 - y0);
    if (area <= 0) return;
    my_radius = rad_i;
    tiles = (uint32_t)area;
    dkey = __float_as_uint(tz);
    float cr, cg, cbl;
    if (col != nullptr) { cr = col[0]; cg = col[1]; cbl = col[2]; }
    else if (sh_row != nullptr) sh_to_rgb(deg, sh_row, x - vk.cam[0], y - vk.cam[1], z - vk.cam[2], cr, cg, cbl);
    else { cr = 0.f; cg = 0.f; cbl = 0.f; }       // geometry-only pass: sh_colour_multi_kernel fills the colour in later
    rec.g = make_float4(px, py, tz, __int_as_float(rad_i));
    // conic pre-scaled to log2 units for the composite: a' = -0.5*log2e*A, b' = -log2e*B, c' = -0.5*log2e*C
    const float L2E = 1.4426950408889634f;
    rec.c = make_float4(-0.5f * L2E * (cc * det_inv), L2E * (cb * det_inv), -0.5f * L2E * (ca * det_inv), opacity);
    if (tight) tight_spans(px, py, rec.c, x0, y0, x1, y1, tiles, spans);
    rec.k = make_float4(cr, cg, cbl, __uint_as_float(tiles));
}

// One thread per Gaussian.  SH coefficients of the CTA's 128 Gaussians are one contiguous span of global
// memory (128*M*12 B): staged into shared memory with coalesced 128-bit loads, then each thread reads its
// own row (row stride padded to an odd word count -> bank-conflict free).
__global__ void __launch_bounds__(PP_THREADS)
preprocess_kernel(ViewArgs va, int N, int M, const float* __restrict__ means3D, const float* __restrict__ shs,
                  const float* __restrict__ colors_precomp, const float* __restrict__ opacities,
                  const float* __restrict__ scales, const float* __restrict__ rotations,
                  const float* __restrict__ cov3D_precomp, SplatRec* __restrict__ recs,
                  int32_t* __restrict__ radii, uint32_t* __restrict__ tiles_touched,
                  uint32_t* __restrict__ depth_keys, uint32_t* __restrict__ ids, uint32_t* __restrict__ min_key,
                  uint4* __restrict__ spans) {
    extern __shared__ __align__(16) float s_sh[];
    __shared__ float s_view[16], s_proj[16], s_cam[3];
    __shared__ uint32_t s_min;
    const int tid = threadIdx.x;
    const int base = blockIdx.x * PP_THREADS;
    if (tid == 0) s_min = 0xFFFFFFFFu;
    if (tid < 16) { s_view[tid] = __ldg(va.view + tid); s_proj[tid] = __ldg(va.proj + tid); }
    if (tid < 3) s_cam[tid] = __ldg(va.campos + tid);
    const int row = 3 * M;
    const int rowp = gs_rowp(row);
    if (shs != nullptr)
        gs_stage_rows_in(s_sh, shs + (size_t)base * row, min(PP_THREADS, N - base), row, tid, PP_THREADS);
    __syncthreads();

    const bool live = base + tid < N;
    const int idx = live ? base + tid : N - 1;      // tail threads redo the last Gaussian, stores are guarded
    const float x = means3D[3 * idx + 0], y = means3D[3 * idx + 1], z = means3D[3 * idx + 2];
    float c[6];
    cov3d_of(scales, rotations, cov3D_precomp, va.scale_modifier, idx, c);
    ViewK vk{s_view, s_proj, s_cam, va.tanfovx, va.tanfovy, va.focal_x, va.focal_y, va.W, va.H, va.tiles_x, va.tiles_y};
    SplatRec rec; int my_radius; uint32_t tiles, dkey; uint4 sp;
    project_view(vk, va.sh_degree, M, x, y, z, c, opacities[idx], s_sh + (idx - base) * rowp,
                 colors_precomp ? colors_precomp + 3 * (size_t)idx : nullptr, rec, my_radius, tiles, dkey,
                 spans != nullptr, sp);
    if (live) {
        if (spans) spans[idx] = sp;
        recs[idx] = rec;
        radii[idx] = my_radius;
        tiles_touched[idx] = tiles;
        depth_keys[idx] = dkey;
        ids[idx] = (uint32_t)idx;
        if (dkey != 0xFFFFFFFFu) atomicMin(&s_min, dkey);
    }
    // minimum visible depth key of the view -> bias of the depth sort (see gs_sort.cu)
    __syncthreads();
    if (tid == 0 && s_min != 0xFFFFFFFFu) atomicMin(min_key, s_min);
}

// All V views of a multi-view step in ONE pass over the Gaussians: parameters (236 B each at SH 3) are read
// once instead of V times, cov3D is computed once; per view only the 64 B of outputs are written.
// views: V x 40 floats (viewmatrix 16 | projmatrix 16 | campos 3 | bg 3 | tanfovx | tanfovy), outputs [V][N].
constexpr int PP_MAXV = 16;
__global__ void __launch_bounds__(PP_THREADS)
preprocess_multi_kernel(const float* __restrict__ views, int V, int W, int H, int sh_degree, float scale_modifier,
                        int N, int M, const float* __restrict__ means3D, const float* __restrict__ shs,
                        const float* __restrict__ colors_precomp /* [N,3] instead of shs (forward-only callers) */,
                        const float* __restrict__ opacities, const float* __restrict__ scales,
                        const float* __restrict__ rotations, SplatRec* __restrict__ recs,
                        int32_t* __restrict__ radii, uint32_t* __restrict__ tiles_touched,
                        uint32_t* __restrict__ depth_keys, uint32_t* __restrict__ ids,
                        uint32_t* __restrict__ min_keys /* [V] stride 2 words */, uint4* __restrict__ spans) {
    extern __shared__ __align__(16) float s_sh[];
    __shared__ float s_views[PP_MAXV * 40];
    __shared__ uint32_t s_min[PP_MAXV];
    const int tid = threadIdx.x;
    const int base = blockIdx.x * PP_THREADS;
    for (int i = tid; i < V * 40; i += PP_THREADS) s_views[i] = __ldg(views + i);
    if (tid < V) s_min[tid] = 0xFFFFFFFFu;
    const int row = 3 * M;
    const int rowp = gs_rowp(row);
    if (shs != nullptr) gs_stage_rows_in(s_sh, shs + (size_t)base * row, min(PP_THREADS, N - base), row, tid, PP_THREADS);
    __syncthreads();
    const bool live = base + tid < N;
    const int idx = live ? base + tid : N - 1;
    const float x = means3D[3 * idx + 0], y = means3D[3 * idx + 1], z = means3D[3 * idx + 2];
    const float opacity = opacities[idx];
    const float* col = colors_precomp ? colors_precomp + 3 * (size_t)idx : nullptr;
    float c[6];
    cov3d_of(scales, rotations, nullptr, scale_modifier, idx, c);
    const int tiles_x = (W + GS_TILE - 1) / GS_TILE, tiles_y = (H + GS_TILE - 1) / GS_TILE;
    for (int v = 0; v < V; v++) {
        const float* vw = s_views + v * 40;
        const float tfx = vw[38], tfy = vw[39];
        ViewK vk{vw, vw + 16, vw + 32, tfx, tfy, (float)W / (2.0f * tfx), (float)H / (2.0f * tfy), W, H, tiles_x, tiles_y};
        SplatRec rec; int my_radius; uint32_t tiles, dkey; uint4 sp;
        project_view(vk, sh_degree, M, x, y, z, c, opacity, shs ? s_sh + (idx - base) * rowp : nullptr, col, rec, my_radius,
                     tiles, dkey, spans != nullptr, sp);
        if (live) {
            const size_t o = (size_t)v * N + idx;
            if (spans) spans[o] = sp;
            recs[o] = rec;
            radii[o] = my_radius;
            tiles_touched[o] = tiles;
            depth_keys[o] = dkey;
            ids[o] = (uint32_t)idx;
            if (dkey != 0xFFFFFFFFu) atomicMin(&s_min[v], dkey);
        }
    }
    __syncthreads();
    if (tid < V && s_min[tid] != 0xFFFFFFFFu) atomicMin(min_keys + 2 * tid, s_min[tid]);
}


// Colour of every visible (view, Gaussian) pair written into records that a geometry-only preprocess_multi pass left
// with zero colour: the host-buffer step starts projecting, sorting and binning while the SH block (81 % of the
// parameter bytes) is still on its way over PCIe.  Same sh_to_rgb, same operands -> the same bits as the one-pass path.
__global__ void __launch_bounds__(PP_THREADS)
sh_colour_multi_kernel(const float* __restrict__ views, int V, int sh_degree, int N, int M,
                       const float* __restrict__ means3D, const float* __restrict__ shs,
                       const int32_t* __restrict__ radii, SplatRec* __restrict__ recs) {
    extern __shared__ __align__(16) float s_sh[];
    __shared__ float s_cam[PP_MAXV * 3];
    const int tid = threadIdx.x;
    const int base = blockIdx.x * PP_THREADS;
    if (tid < V * 3) s_cam[tid] = __ldg(views + (tid / 3) * 40 + 32 + tid % 3);
    const int row = 3 * M;
    const int rowp = gs_rowp(row);
    gs_stage_rows_in(s_sh, shs + (size_t)base * row, min(PP_THREADS, N - base), row, tid, PP_THREADS);
    __syncthreads();
    const int idx = base + tid;
    if (idx >= N) return;
    const float x = means3D[3 * idx + 0], y = means3D[3 * idx + 1], z = means3D[3 * idx + 2];
    for (int v = 0; v < V; v++) {
        const size_t o = (size_t)v * N + idx;
        if (radii[o] <= 0) continue;
        float cr, cg, cb;
        sh_to_rgb(sh_degree, s_sh + tid * rowp, x - s_cam[3 * v], y - s_cam[3 * v + 1], z - s_cam[3 * v + 2], cr, cg, cb);
        float* k = reinterpret_cast<float*>(&recs[o].k);
        *reinterpret_cast<float2*>(k) = make_float2(cr, cg);
        k[2] = cb;
    }
}

}  // namespace

int gs_launch_preprocess(const ViewArgs& va, int N, int M, const float* means3D, const float* shs,
                         const float* colors_precomp, const float* opacities, const float* scales,
                         const float* rotations, const float* cov3D_precomp, SplatRec* recs, int32_t* radii,
                         uint32_t* tiles_touched, uint32_t* depth_keys, uint32_t* ids, uint32_t* min_key,
                         uint4* spans, cudaStream_t s) {
    if (N <= 0) return 0;
    size_t smem = shs ? (size_t)PP_THREADS * ((3 * M) | 1) * sizeof(float) : 0;
    if (smem > 48 * 1024) {
        GS_CUDA_CHECK(cudaFuncSetAttribute(preprocess_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    int blocks = (N + PP_THREADS - 1) / PP_THREADS;
    preprocess_kernel<<<blocks, PP_THREADS, smem, s>>>(va, N, M, means3D, shs, colors_precomp, opacities, scales,
                                                       rotations, cov3D_precomp, recs, radii, tiles_touched,
                                                       depth_keys, ids, min_key, spans);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int gs_preprocess_multi_max_views() { return PP_MAXV; }

int gs_launch_preprocess_multi(const float* views_dev, int V, int W, int H, int sh_degree, float scale_modifier, int N,
                               int M, const float* means3D, const float* shs, const float* colors_precomp,
                               const float* opacities, const float* scales, const float* rotations, SplatRec* recs,
                               int32_t* radii, uint32_t* tiles_touched, uint32_t* depth_keys, uint32_t* ids,
                               uint32_t* min_keys, uint4* spans, cudaStream_t s, int geom_only) {
    if (N <= 0 || V <= 0) return 0;
    if (V > PP_MAXV) { gs_set_error("preprocess_multi: V=%d > %d", V, PP_MAXV); return 1; }
    if (geom_only) { shs = nullptr; colors_precomp = nullptr; }      // colours follow from gs_launch_sh_colour_multi
    else if ((shs == nullptr) == (colors_precomp == nullptr)) { gs_set_error("preprocess_multi: exactly one of shs / colors_precomp"); return 1; }
    size_t smem = shs ? (size_t)PP_THREADS * ((3 * M) | 1) * sizeof(float) : 0;
    if (smem > 48 * 1024)
        GS_CUDA_CHECK(cudaFuncSetAttribute(preprocess_multi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int blocks = (N + PP_THREADS - 1) / PP_THREADS;
    preprocess_multi_kernel<<<blocks, PP_THREADS, smem, s>>>(views_dev, V, W, H, sh_degree, scale_modifier, N, M, means3D,
                                                             shs, colors_precomp, opacities, scales, rotations, recs, radii,
                                                             tiles_touched, depth_keys, ids, min_keys, spans);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int gs_launch_sh_colour_multi(const float* views_dev, int V, int sh_degree, int N, int M, const float* means3D,
                              const float* shs, const int32_t* radii, SplatRec* recs, cudaStream_t s) {
    if (N <= 0 || V <= 0) return 0;
    if (V > PP_MAXV || !shs) { gs_set_error("sh_colour_multi: bad argument"); return 1; }
    const size_t smem = (size_t)PP_THREADS * ((3 * M) | 1) * sizeof(float);
    if (smem > 48 * 1024)
        GS_CUDA_CHECK(cudaFuncSetAttribute(sh_colour_multi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    sh_colour_multi_kernel<<<(N + PP_THREADS - 1) / PP_THREADS, PP_THREADS, smem, s>>>(views_dev, V, sh_degree, N, M, means3D, shs,
                                                                                      radii, recs);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
