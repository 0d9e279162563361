// pytorch3d's point rasterizer and TriplaneGaussian's points_projection on the GPU (gs_b200_pts.h, which states every
// rule): project through cameras_from_opencv_projection's camera, keep the K nearest covering points per pixel, and lift
// a feature map onto the points, with the lift's backward.
//
// Built with -fmad=false: the projection, the pixel centres and every squared distance are one rounding per operation
// in the order the header states, so a numpy float32 restatement gives the same bits.
//
// Rasterization is binned by point, not by pixel: each point walks only the pixels its radius box touches.  A candidate
// is the 64-bit key (z bits << 32) | packed index; z > 0, so the keys order as (z, index) and every pixel's selection is
// a minimum over a set, independent of the order the atomics land in.  Slot k of a pixel is filled by pass k, a 64-bit
// atomicMin over the candidates strictly greater than slot k - 1, so K passes give the K smallest keys, sorted.
#include "../../include/gs_b200_pts.h"
#include "gs_common.cuh"

#include <math.h>
#include <stdint.h>

namespace {

constexpr int TPB = 256;
constexpr uint64_t EMPTY = ~0ull;
inline unsigned nblocks(int64_t n, int per = TPB) { return (unsigned)((n + per - 1) / per); }
inline size_t al(size_t b) { return (b + 255) & ~(size_t)255; }

// pytorch3d's NonSquareNdcRange / PixToNonSquareNdc: the centre of pixel i (counted from the +X / +Y end) on a side of
// S1 pixels when the other side has S2.  The shorter side spans [-1, 1].
__device__ __forceinline__ float ndc_range(int S1, int S2) { return S1 > S2 ? ((float)S1 * 2.0f) / (float)S2 : 2.0f; }
__device__ __forceinline__ float pix_ndc(int i, int S1, int S2) {
    const float range = ndc_range(S1, S2), offset = range / 2.0f;
    return -offset + (range * (float)i + offset) / (float)S1;
}

// The pixels (counted from the +X end) whose centres can lie within r of p along one axis, widened by one pixel on each
// side so rounding cannot drop one; the exact test decides.  Empty (lo > hi) when the span misses the image.
__device__ __forceinline__ void pix_span(float p, float r, int S1, int S2, int& lo, int& hi) {
    const float range = ndc_range(S1, S2), offset = range / 2.0f;
    float a = ((p - r + offset) * (float)S1 - offset) / range, b = ((p + r + offset) * (float)S1 - offset) / range;
    if (!(b >= -2.0f) || !(a <= (float)S1 + 1.0f)) { lo = 0; hi = -1; return; }
    a = fmaxf(a, -2.0f); b = fminf(b, (float)S1 + 1.0f);
    lo = max(0, (int)floorf(a) - 1);
    hi = min(S1 - 1, (int)ceilf(b) + 1);
}

__device__ __forceinline__ int cloud_of(int64_t p, int N, int64_t P, const int64_t* first) {
    if (!first) return (int)(p / (P / N));
    int lo = 0, hi = N - 1;                       // the last n with first[n] <= p
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (first[mid] <= p) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// ---- projection: one thread per packed point -> (x_ndc, y_ndc, z_view, cloud) ----------------------------------------
__global__ void __launch_bounds__(TPB) k_project(int64_t P, int N, int ncam, const float* __restrict__ pts,
                                                 const int64_t* __restrict__ first, const float* __restrict__ R,
                                                 const float* __restrict__ T, const float* __restrict__ Km,
                                                 const float* __restrict__ hw, int H, int W, float4* __restrict__ ndc) {
    const int64_t p = (int64_t)blockIdx.x * TPB + threadIdx.x;
    if (p >= P) return;
    const int n = cloud_of(p, N, P, first), c = ncam > 1 ? n : 0;
    const float x = pts[3 * p], y = pts[3 * p + 1], z = pts[3 * p + 2];
    const float* r = R + 9 * c;
    const float xc = ((r[0] * x + r[1] * y) + r[2] * z) + T[3 * c];
    const float yc = ((r[3] * x + r[4] * y) + r[5] * z) + T[3 * c + 1];
    const float zc = ((r[6] * x + r[7] * y) + r[8] * z) + T[3 * c + 2];
    const float* k = Km + 9 * c;
    const float h = hw ? hw[2 * c] : (float)H, w = hw ? hw[2 * c + 1] : (float)W;
    const float s = fminf(h, w) * 0.5f;
    const float u = (k[0] * xc) / zc + k[2], v = (k[4] * yc) / zc + k[5];
    ndc[p] = make_float4((w * 0.5f - u) / s, (h * 0.5f - v) / s, zc, __int_as_float(n));
}

// ---- pass k of the rasterizer: one thread per packed point ----------------------------------------------------------
__global__ void __launch_bounds__(TPB) k_cover(int64_t P, int H, int W, int K, int pass, float radius,
                                               const float4* __restrict__ ndc, unsigned long long* __restrict__ keys) {
    const int64_t p = (int64_t)blockIdx.x * TPB + threadIdx.x;
    if (p >= P) return;
    const float4 q = ndc[p];
    if (!(q.z > 0.0f) || !isfinite(q.x) || !isfinite(q.y)) return;     // z <= 0, NaN or off to infinity: never drawn
    const int n = __float_as_int(q.w);
    const float r2 = radius * radius;
    int xlo, xhi, ylo, yhi;
    pix_span(q.x, radius, W, H, xlo, xhi);
    pix_span(q.y, radius, H, W, ylo, yhi);
    const unsigned long long key = ((unsigned long long)__float_as_uint(q.z) << 32) | (unsigned long long)(uint32_t)p;
    for (int yi = ylo; yi <= yhi; yi++) {
        const float dy = pix_ndc(yi, H, W) - q.y;
        const int64_t row = ((int64_t)n * H + (H - 1 - yi)) * W;
        for (int xi = xlo; xi <= xhi; xi++) {
            const float dx = pix_ndc(xi, W, H) - q.x;
            if (!(dx * dx + dy * dy < r2)) continue;
            unsigned long long* slot = keys + (row + (W - 1 - xi)) * K + pass;
            if (pass > 0 && key <= slot[-1]) continue;                    // already in an earlier slot
            atomicMin(slot, key);
        }
    }
}

// ---- keys -> idx / zbuf / dists: one thread per (pixel, slot) --------------------------------------------------------
__global__ void __launch_bounds__(TPB) k_fragments(int64_t total, int H, int W, int K, const float4* __restrict__ ndc,
                                                   const unsigned long long* __restrict__ keys, int32_t* __restrict__ idx,
                                                   float* __restrict__ zbuf, float* __restrict__ dists) {
    const int64_t e = (int64_t)blockIdx.x * TPB + threadIdx.x;
    if (e >= total) return;
    const unsigned long long key = keys[e];
    if (key == EMPTY) {
        idx[e] = -1;
        if (zbuf) zbuf[e] = -1.0f;
        if (dists) dists[e] = -1.0f;
        return;
    }
    const int32_t p = (int32_t)(uint32_t)key;
    idx[e] = p;
    if (zbuf) zbuf[e] = __uint_as_float((uint32_t)(key >> 32));
    if (dists) {
        const int64_t pix = e / K;
        const int x = (int)(pix % W), y = (int)((pix / W) % H);
        const float4 q = ndc[p];
        const float dx = pix_ndc(W - 1 - x, W, H) - q.x, dy = pix_ndc(H - 1 - y, H, W) - q.y;
        dists[e] = dx * dx + dy * dy;
    }
}

// ---- lift: each point's winner is the largest (pixel, slot) index that selected it -----------------------------------
__global__ void __launch_bounds__(TPB) k_winner(int32_t total, const int32_t* __restrict__ idx, int32_t* __restrict__ winner) {
    const int32_t e = blockIdx.x * TPB + threadIdx.x;
    if (e >= total) return;
    const int32_t p = idx[e];
    if (p >= 0) atomicMax(winner + p, e);
}

// out [P, C]: one thread per element, channels fastest (coalesced writes; the feature map is read in place)
__global__ void __launch_bounds__(TPB) k_lift(int64_t total, int C, int HW, int W, int K, const int32_t* __restrict__ winner,
                                              const float* __restrict__ f, int64_t s0, int64_t s1, int64_t s2, int64_t s3,
                                              float* __restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * TPB + threadIdx.x;
    if (t >= total) return;
    const int64_t p = t / C;
    const int c = (int)(t - p * C);
    const int32_t w = winner[p];
    float v = 0.0f;
    if (w >= 0) {
        const int32_t pix = w / K, n = pix / HW, yx = pix - n * HW, y = yx / W, x = yx - y * W;
        v = f[n * s0 + c * s1 + y * s2 + x * s3];
    }
    out[t] = v;
}

// grad_features [N, C, H, W]: one thread per element; the sum over the pixel's slots whose point it won, in slot order
__global__ void __launch_bounds__(TPB) k_lift_bwd(int64_t total, int C, int HW, int K, const int32_t* __restrict__ idx,
                                                  const int32_t* __restrict__ winner, const float* __restrict__ go,
                                                  float* __restrict__ grad) {
    const int64_t t = (int64_t)blockIdx.x * TPB + threadIdx.x;
    if (t >= total) return;
    const int64_t nc = t / HW;
    const int yx = (int)(t - nc * HW);
    const int n = (int)(nc / C), c = (int)(nc - (int64_t)n * C);
    const int32_t e0 = (n * HW + yx) * K;
    float acc = 0.0f;
    for (int k = 0; k < K; k++) {
        const int32_t p = idx[e0 + k];
        if (p >= 0 && winner[p] == e0 + k) acc += go[(int64_t)p * C + c];
    }
    grad[t] = acc;
}

bool bad_dims(const char* fn, int32_t N, int64_t P, int32_t H, int32_t W, int32_t K) {
    if (N < 0 || P < 0 || H < 1 || W < 1 || K < 1 || K > GS_B200_PTS_MAX_K || (N == 0 && P > 0)) {
        gs_set_error("%s: N %d, P %lld, H %d, W %d, K %d (need N >= 0, P >= 0, H, W >= 1, 1 <= K <= %d)", fn, N,
                     (long long)P, H, W, K, GS_B200_PTS_MAX_K);
        return true;
    }
    if ((double)N * H * W * K >= 2147483648.0 || P >= 2147483648LL) {
        gs_set_error("%s: N*H*W*K and P must be below 2^31", fn);
        return true;
    }
    return false;
}

}  // namespace

size_t gs_b200_pts_scratch_bytes(int32_t N, int64_t P, int32_t H, int32_t W, int32_t K) {
    if (bad_dims("pts_scratch_bytes", N, P, H, W, K)) return 0;
    return al((size_t)N * H * W * K * 8) + al((size_t)P * 16) + 256;
}

int32_t gs_b200_pts_rasterize(int32_t N, int64_t P, int32_t H, int32_t W, int32_t K, float radius, int32_t ncam,
                              const float* points, const int64_t* first, const float* R, const float* T,
                              const float* camera_matrix, const float* image_hw, int32_t* idx, float* zbuf,
                              float* dists, void* scratch, void* stream) {
    static const char* fn = "pts_rasterize";
    if (bad_dims(fn, N, P, H, W, K)) return 1;
    if (N > 0 && ncam != 1 && ncam != N) { gs_set_error("%s: %d cameras for %d clouds (need 1 or N)", fn, ncam, N); return 1; }
    if (!(radius >= 0.0f)) { gs_set_error("%s: radius %g (need >= 0)", fn, (double)radius); return 1; }
    const int64_t total = (int64_t)N * H * W * K;
    if (total == 0) return 0;
    if (!idx || !scratch || (P > 0 && (!points || !R || !T || !camera_matrix))) { gs_set_error("%s: NULL pointer", fn); return 1; }
    if (!first && P % N) { gs_set_error("%s: P %lld is not a multiple of N %d and `first` is NULL", fn, (long long)P, N); return 1; }
    cudaStream_t s = (cudaStream_t)stream;
    char* scr = (char*)(((uintptr_t)scratch + 255) & ~(uintptr_t)255);
    unsigned long long* keys = (unsigned long long*)scr;
    float4* ndc = (float4*)(scr + al((size_t)total * 8));
    GS_CUDA_CHECK(cudaMemsetAsync(keys, 0xff, (size_t)total * 8, s));
    if (P > 0) {
        k_project<<<nblocks(P), TPB, 0, s>>>(P, N, ncam, points, first, R, T, camera_matrix, image_hw, H, W, ndc);
        for (int k = 0; k < K; k++) k_cover<<<nblocks(P), TPB, 0, s>>>(P, H, W, K, k, radius, ndc, keys);
        gs_count_launches(1 + K);
    }
    k_fragments<<<nblocks(total), TPB, 0, s>>>(total, H, W, K, ndc, keys, idx, zbuf, dists);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int32_t gs_b200_pts_lift(int32_t N, int64_t P, int32_t H, int32_t W, int32_t K, int32_t C, const int32_t* idx,
                         const float* features, const int64_t* feature_strides_host, int32_t* winner, float* out,
                         void* stream) {
    static const char* fn = "pts_lift";
    if (bad_dims(fn, N, P, H, W, K)) return 1;
    if (C < 0 || (double)P * C >= 9.2e18) { gs_set_error("%s: C %d", fn, C); return 1; }
    if (P == 0) return 0;
    const int64_t total = (int64_t)N * H * W * K;
    if (!winner || (C > 0 && (!out || !features || !feature_strides_host)) || (total > 0 && !idx)) {
        gs_set_error("%s: NULL pointer", fn);
        return 1;
    }
    cudaStream_t s = (cudaStream_t)stream;
    GS_CUDA_CHECK(cudaMemsetAsync(winner, 0xff, (size_t)P * 4, s));
    if (total > 0) { k_winner<<<nblocks(total), TPB, 0, s>>>((int32_t)total, idx, winner); gs_count_launches(1); }
    if (C > 0) {
        const int64_t* st = feature_strides_host;
        k_lift<<<nblocks(P * C), TPB, 0, s>>>(P * C, C, H * W, W, K, winner, features, st[0], st[1], st[2], st[3], out);
        gs_count_launches(1);
    }
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int32_t gs_b200_pts_lift_backward(int32_t N, int64_t P, int32_t H, int32_t W, int32_t K, int32_t C, const int32_t* idx,
                                  const int32_t* winner, const float* grad_out, float* grad_features, void* stream) {
    static const char* fn = "pts_lift_backward";
    if (bad_dims(fn, N, P, H, W, K)) return 1;
    if (C < 0 || (double)N * C * H * W >= 9.2e18) { gs_set_error("%s: C %d", fn, C); return 1; }
    const int64_t total = (int64_t)N * C * H * W;
    if (total == 0) return 0;
    if (!grad_features || !idx || (P > 0 && (!winner || !grad_out))) { gs_set_error("%s: NULL pointer", fn); return 1; }
    k_lift_bwd<<<nblocks(total), TPB, 0, (cudaStream_t)stream>>>(total, C, H * W, K, idx, winner, grad_out, grad_features);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
