// pointnet2_ops' point-cloud operators on the GPU (include/gs_b200.h, "pointnet2" section): farthest point sampling,
// ball query, three-NN, gather / grouping and three-interpolate, forward, and the gather / three-interpolate
// backward as a deterministic scatter-sum.
//
// Built with -fmad=false: every squared distance is ((dx*dx + dy*dy) + dz*dz), one rounding per operation, and the
// three-interpolate forward is ((w0*f0 + w1*f1) + w2*f2), so a numpy float32 restatement in the same order gives the
// same bits.  Ties are broken by the smallest index everywhere, so no result depends on the launch shape.
#include "../../include/gs_b200.h"
#include "gs_common.cuh"

#include <float.h>
#include <limits.h>
#include <algorithm>

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int TPB = 256;
inline unsigned nblocks(int64_t n, int per = TPB) { return (unsigned)((n + per - 1) / per); }

__device__ __forceinline__ float dist2(float ax, float ay, float az, float bx, float by, float bz) {
    const float dx = ax - bx, dy = ay - by, dz = az - bz;
    return (dx * dx + dy * dy) + dz * dz;
}

// pointnet2_ops' FPS never updates nor picks a point with x^2 + y^2 + z^2 <= 1e-3 (fp32 magnitude against the double
// literal).  Such points carry the running distance -1, which fminf keeps and which never beats a real candidate.
__device__ __forceinline__ bool fps_skipped(float x, float y, float z) {
    const float mag = (x * x + y * y) + z * z;
    return (double)mag <= 1e-3;
}

// ---- farthest point sampling: one CTA of 1024 threads per batch item -----------------------------------------------
// A candidate is the pair (running distance, index); the step's pick is the largest distance, smallest index on ties.
// Running distances are >= -1 and <= 1e10, so key = bits(d) + 1 for d >= 0 and 0 for the skipped marker orders them
// as unsigned integers.  Each warp reduces with one redux.max over the keys and one redux.min over the indices that
// hold the maximum; every warp then reduces the 32 warp winners itself, so one __syncthreads per step suffices
// (the winner slots are double-buffered by step parity).  Max with a smallest-index tie-break is associative and
// commutative, so the pick does not depend on the reduction tree.
constexpr int FPS_T = 1024;

__device__ __forceinline__ unsigned fps_key(float d) { return d < 0.f ? 0u : __float_as_uint(d) + 1u; }

__device__ __forceinline__ void fps_warp_argmax(unsigned& key, int& idx) {
    const unsigned kmax = __reduce_max_sync(FULL, key);
    idx = (int)__reduce_min_sync(FULL, key == kmax ? (unsigned)idx : (unsigned)INT_MAX);
    key = kmax;
}

// PPT > 0: coordinates staged in shared memory as SoA (12 B per point), PPT running distances per thread in
// registers (points tid, tid + 1024, ...).  PPT == 0: coordinates read from global memory (they stay in L2) and running
// distances kept in `gtemp` [B, N].
template <int PPT>
__global__ void __launch_bounds__(FPS_T, 1) k_fps(int N, int npoint, const float* __restrict__ xyz,
                                                  int32_t* __restrict__ out, float* __restrict__ gtemp) {
    extern __shared__ float s_xyz[];
    __shared__ unsigned s_key[2][32];
    __shared__ int s_idx[2][32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* p = xyz + (size_t)blockIdx.x * N * 3;
    int32_t* o = out + (size_t)blockIdx.x * npoint;
    float temp[PPT > 0 ? PPT : 1];
    float* gt = gtemp + (size_t)blockIdx.x * N;
    if (PPT > 0) {
        float* sx = s_xyz; float* sy = s_xyz + N; float* sz = s_xyz + 2 * N;
#pragma unroll
        for (int j = 0; j < PPT; j++) {
            const int k = tid + j * FPS_T;
            temp[j] = -1.f;
            if (k < N) {
                const float x = p[3 * k], y = p[3 * k + 1], z = p[3 * k + 2];
                sx[k] = x; sy[k] = y; sz[k] = z;
                temp[j] = fps_skipped(x, y, z) ? -1.f : 1e10f;
            }
        }
    } else {
        for (int k = tid; k < N; k += FPS_T) gt[k] = fps_skipped(p[3 * k], p[3 * k + 1], p[3 * k + 2]) ? -1.f : 1e10f;
    }
    if (tid == 0 && npoint > 0) o[0] = 0;
    __syncthreads();
    int last = 0;
    for (int s = 1; s < npoint; s++) {
        unsigned key = 0;
        int idx = 0;
        if (PPT > 0) {
            const float lx = s_xyz[last], ly = s_xyz[N + last], lz = s_xyz[2 * N + last];
            const float* bx = s_xyz + tid;             // this thread's points sit at constant offsets j * FPS_T
            const int rem = N - tid;
#pragma unroll
            for (int j = 0; j < PPT; j++) {
                if (j * FPS_T < rem) {
                    const float t = fminf(dist2(bx[j * FPS_T], bx[N + j * FPS_T], bx[2 * N + j * FPS_T], lx, ly, lz), temp[j]);
                    temp[j] = t;
                    const unsigned kk = fps_key(t);
                    if (kk > key) { key = kk; idx = j; }
                }
            }
            idx = key ? tid + idx * FPS_T : 0;          // no candidate: (key 0, index 0)
        } else {
            const float lx = p[3 * last], ly = p[3 * last + 1], lz = p[3 * last + 2];
            for (int k = tid; k < N; k += FPS_T) {
                const float t = fminf(dist2(p[3 * k], p[3 * k + 1], p[3 * k + 2], lx, ly, lz), gt[k]);
                gt[k] = t;
                const unsigned kk = fps_key(t);
                if (kk > key) { key = kk; idx = k; }
            }
        }
        fps_warp_argmax(key, idx);
        if (lane == 0) { s_key[s & 1][warp] = key; s_idx[s & 1][warp] = idx; }
        __syncthreads();
        key = s_key[s & 1][lane];
        idx = s_idx[s & 1][lane];
        fps_warp_argmax(key, idx);
        last = idx;
        if (tid == 0) o[s] = last;
    }
}

// ---- ball query: one warp per query ----------------------------------------------------------------------------------
// 32 consecutive candidates per round; hits are appended in index order (ballot + popc) until nsample are found.
// Slots past the last hit repeat the first hit (0 when there is none).
__global__ void __launch_bounds__(TPB) k_ball_query(int nq, int N, int P, int S, float r2, const float* __restrict__ xyz,
                                                    const float* __restrict__ new_xyz, int32_t* __restrict__ out) {
    const int q = (int)((blockIdx.x * (unsigned)TPB + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (q >= nq) return;
    const float* p = xyz + (size_t)(q / P) * N * 3;
    const float qx = new_xyz[3 * (size_t)q], qy = new_xyz[3 * (size_t)q + 1], qz = new_xyz[3 * (size_t)q + 2];
    int32_t* o = out + (size_t)q * S;
    int cnt = 0, first = 0;
    for (int base = 0; base < N && cnt < S; base += 32) {
        const int k = base + lane;
        bool hit = false;
        if (k < N) hit = dist2(qx, qy, qz, p[3 * k], p[3 * k + 1], p[3 * k + 2]) < r2;
        const unsigned m = __ballot_sync(FULL, hit);
        if (!m) continue;
        if (cnt == 0) first = base + __ffs(m) - 1;
        const int pos = cnt + __popc(m & ((1u << lane) - 1u));
        if (hit && pos < S) o[pos] = k;
        cnt += __popc(m);
    }
    for (int l = min(cnt, S) + lane; l < S; l += 32) o[l] = first;
}

// ---- three-NN: one warp per query --------------------------------------------------------------------------------------
// Each lane keeps a sorted top 3 of its strided candidates under strict-< insertion in ascending index (NaN and +inf
// never enter); three argmin rounds over the lanes' heads, by (d^2, index), merge them.  d^2 >= +0, so its bits order
// as unsigned integers.
__global__ void __launch_bounds__(TPB) k_three_nn(int nq, int n, int m, const float* __restrict__ unknown,
                                                  const float* __restrict__ known, float* __restrict__ dist,
                                                  int32_t* __restrict__ idx) {
    const int q = (int)((blockIdx.x * (unsigned)TPB + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (q >= nq) return;
    const float* kp = known + (size_t)(q / n) * m * 3;
    const float ux = unknown[3 * (size_t)q], uy = unknown[3 * (size_t)q + 1], uz = unknown[3 * (size_t)q + 2];
    float d0 = INFINITY, d1 = INFINITY, d2 = INFINITY;
    int i0 = INT_MAX, i1 = INT_MAX, i2 = INT_MAX;
    for (int k = lane; k < m; k += 32) {
        const float d = dist2(ux, uy, uz, kp[3 * k], kp[3 * k + 1], kp[3 * k + 2]);
        if (d < d0) { d2 = d1; i2 = i1; d1 = d0; i1 = i0; d0 = d; i0 = k; }
        else if (d < d1) { d2 = d1; i2 = i1; d1 = d; i1 = k; }
        else if (d < d2) { d2 = d; i2 = k; }
    }
#pragma unroll
    for (int r = 0; r < 3; r++) {
        const unsigned key = __float_as_uint(d0);
        const unsigned kmin = __reduce_min_sync(FULL, key);
        const int wi = (int)__reduce_min_sync(FULL, key == kmin ? (unsigned)i0 : (unsigned)INT_MAX);
        if (lane == 0) {
            const bool none = wi == INT_MAX;
            dist[3 * (size_t)q + r] = none ? INFINITY : __fsqrt_rn(__uint_as_float(kmin));
            idx[3 * (size_t)q + r] = none ? 0 : wi;
        }
        if (key == kmin && i0 == wi) { d0 = d1; i0 = i1; d1 = d2; i1 = i2; d2 = INFINITY; i2 = INT_MAX; }
    }
}

// ---- gathers and three-interpolate: one thread per output element, coalesced along the last dimension ---------------
__global__ void __launch_bounds__(TPB) k_gather(uint32_t total, int C, int N, int M, const float* __restrict__ f,
                                                const int32_t* __restrict__ idx, float* __restrict__ out) {
    const uint32_t t = blockIdx.x * TPB + threadIdx.x;
    if (t >= total) return;
    const uint32_t bc = t / M, j = t - bc * M, b = bc / C;
    const int32_t v = idx[(size_t)b * M + j];
    out[t] = (uint32_t)v < (uint32_t)N ? f[(size_t)bc * N + v] : 0.f;
}

__device__ __forceinline__ float feat_or_zero(const float* f, int32_t v, int m) {
    return (uint32_t)v < (uint32_t)m ? f[v] : 0.f;
}

__global__ void __launch_bounds__(TPB) k_three_interp(uint32_t total, int C, int m, int n, const float* __restrict__ f,
                                                      const int32_t* __restrict__ idx, const float* __restrict__ w,
                                                      float* __restrict__ out) {
    const uint32_t t = blockIdx.x * TPB + threadIdx.x;
    if (t >= total) return;
    const uint32_t bc = t / n, i = t - bc * n, b = bc / C;
    const size_t r = ((size_t)b * n + i) * 3;
    const float* fr = f + (size_t)bc * m;
    const float f0 = feat_or_zero(fr, idx[r], m), f1 = feat_or_zero(fr, idx[r + 1], m), f2 = feat_or_zero(fr, idx[r + 2], m);
    out[t] = (w[r] * f0 + w[r + 1] * f1) + w[r + 2] * f2;
}

// backward values of three-interpolate: vals[b, c, 3i + k] = grad_out[b, c, i] * w[b, i, k]
__global__ void __launch_bounds__(TPB) k_three_interp_vals(uint32_t total, int C, int n, const float* __restrict__ go,
                                                           const float* __restrict__ w, float* __restrict__ vals) {
    const uint32_t t = blockIdx.x * TPB + threadIdx.x;
    if (t >= total) return;
    const uint32_t r = t / 3, bc = r / n, i = r - bc * n, b = bc / C;
    vals[t] = go[r] * w[((size_t)b * n + i) * 3 + (t - r * 3)];
}

// int32 index -> int64 scatter index; values outside [0, N) go to the discard slot N
__global__ void __launch_bounds__(TPB) k_widen(uint32_t total, int N, const int32_t* __restrict__ idx, int64_t* __restrict__ out) {
    const uint32_t t = blockIdx.x * TPB + threadIdx.x;
    if (t >= total) return;
    const int32_t v = idx[t];
    out[t] = (uint32_t)v < (uint32_t)N ? v : N;
}

inline size_t al(size_t b) { return (b + 255) & ~(size_t)255; }

bool too_big(const char* fn, double a, double b = 0, double c = 0) {
    if (a < 2147483648.0 && b < 2147483648.0 && c < 2147483648.0) return false;
    gs_set_error("%s: fewer than 2^31 elements per tensor are supported", fn);
    return true;
}

// the backward's scatter-sum of src [B, C, M] (contiguous) through idx [B, M] into grad [B, C, N + 1]
int scatter_shape(int B, int C, int N, int64_t M, int64_t (&shape)[3], int64_t (&istr)[3]) {
    shape[0] = B; shape[1] = C; shape[2] = M;
    istr[0] = M; istr[1] = 0; istr[2] = 1;
    return N + 1;
}

size_t scatter_bytes(int B, int C, int N, int64_t M) {
    int64_t shape[3], istr[3];
    const int dim_size = scatter_shape(B, C, N, M, shape, istr);
    const size_t sb = gs_b200_scatter_scratch_bytes(GS_B200_SCATTER_SUM, GS_B200_SCATTER_F32, 3, shape, 2, istr, dim_size);
    return sb ? al((size_t)B * M * 8) + sb : 0;
}

int scatter_fold(const char* fn, int B, int C, int N, int64_t M, const float* src, const int32_t* idx, float* grad,
                 char* scratch, cudaStream_t s) {
    int64_t shape[3], istr[3];
    const int dim_size = scatter_shape(B, C, N, M, shape, istr);
    if ((double)B * M >= 1073741824.0) { gs_set_error("%s: fewer than 2^30 index elements are supported", fn); return 1; }
    int64_t* wide = (int64_t*)scratch;
    const uint32_t ni = (uint32_t)(B * M);
    if (ni) { k_widen<<<nblocks(ni), TPB, 0, s>>>(ni, N, idx, wide); gs_count_launches(1); }
    const int64_t sstr[3] = {(int64_t)C * M, M, 1}, ostr[3] = {(int64_t)C * dim_size, dim_size, 1};
    if (gs_b200_scatter_forward(GS_B200_SCATTER_SUM, GS_B200_SCATTER_F32, 3, shape, 2, dim_size, src, sstr, wide, istr,
                                grad, ostr, 0, nullptr, scratch + al((size_t)B * M * 8), s))
        return 1;
    return 0;
}

template <int PPT>
int launch_fps(int B, int N, int npoint, const float* xyz, int32_t* out, float* temp, cudaStream_t s) {
    const size_t smem = PPT > 0 ? (size_t)N * 12 : 0;
    if (smem > 48 * 1024) GS_CUDA_CHECK(cudaFuncSetAttribute(k_fps<PPT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_fps<PPT><<<B, FPS_T, smem, s>>>(N, npoint, xyz, out, temp);
    gs_count_launches(1);
    return 0;
}

}  // namespace

int32_t gs_b200_pn2_furthest_point_sample(int32_t B, int32_t N, int32_t npoint, const float* xyz, int32_t* idx_out,
                                          float* temp, void* stream) {
    static const char* fn = "pn2_furthest_point_sample";
    if (B < 0 || N < 1 || npoint < 0) { gs_set_error("%s: B %d, N %d, npoint %d (need B >= 0, N >= 1, npoint >= 0)", fn, B, N, npoint); return 1; }
    if (too_big(fn, (double)B * N * 3, (double)B * npoint)) return 1;
    if (B == 0 || npoint == 0) return 0;
    if (!xyz || !idx_out || (N > GS_B200_PN2_FPS_ONCHIP_MAX && !temp)) { gs_set_error("%s: NULL pointer", fn); return 1; }
    cudaStream_t s = (cudaStream_t)stream;
    int rc;
    if (N <= FPS_T) rc = launch_fps<1>(B, N, npoint, xyz, idx_out, temp, s);
    else if (N <= 2 * FPS_T) rc = launch_fps<2>(B, N, npoint, xyz, idx_out, temp, s);
    else if (N <= 4 * FPS_T) rc = launch_fps<4>(B, N, npoint, xyz, idx_out, temp, s);
    else if (N <= 8 * FPS_T) rc = launch_fps<8>(B, N, npoint, xyz, idx_out, temp, s);
    else if (N <= GS_B200_PN2_FPS_ONCHIP_MAX) rc = launch_fps<16>(B, N, npoint, xyz, idx_out, temp, s);
    else rc = launch_fps<0>(B, N, npoint, xyz, idx_out, temp, s);
    if (rc) return rc;
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int32_t gs_b200_pn2_ball_query(int32_t B, int32_t N, int32_t npoint, int32_t nsample, float radius, const float* xyz,
                               const float* new_xyz, int32_t* idx_out, void* stream) {
    static const char* fn = "pn2_ball_query";
    if (B < 0 || N < 1 || npoint < 0 || nsample < 0) { gs_set_error("%s: B %d, N %d, npoint %d, nsample %d", fn, B, N, npoint, nsample); return 1; }
    if (too_big(fn, (double)B * N * 3, (double)B * npoint * 3, (double)B * npoint * nsample)) return 1;
    const int nq = B * npoint;
    if (nq == 0 || nsample == 0) return 0;
    if (!xyz || !new_xyz || !idx_out) { gs_set_error("%s: NULL pointer", fn); return 1; }
    k_ball_query<<<nblocks((int64_t)nq * 32), TPB, 0, (cudaStream_t)stream>>>(nq, N, npoint, nsample, radius * radius, xyz,
                                                                             new_xyz, idx_out);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int32_t gs_b200_pn2_three_nn(int32_t B, int32_t n, int32_t m, const float* unknown, const float* known, float* dist,
                             int32_t* idx, void* stream) {
    static const char* fn = "pn2_three_nn";
    if (B < 0 || n < 0 || m < 1) { gs_set_error("%s: B %d, n %d, m %d (need m >= 1)", fn, B, n, m); return 1; }
    if (too_big(fn, (double)B * n * 3, (double)B * m * 3)) return 1;
    const int nq = B * n;
    if (nq == 0) return 0;
    if (!unknown || !known || !dist || !idx) { gs_set_error("%s: NULL pointer", fn); return 1; }
    k_three_nn<<<nblocks((int64_t)nq * 32), TPB, 0, (cudaStream_t)stream>>>(nq, n, m, unknown, known, dist, idx);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int32_t gs_b200_pn2_gather(int32_t B, int32_t C, int32_t N, int32_t M, const float* features, const int32_t* idx,
                           float* out, void* stream) {
    static const char* fn = "pn2_gather";
    if (B < 0 || C < 0 || N < 1 || M < 0) { gs_set_error("%s: B %d, C %d, N %d, M %d (need N >= 1)", fn, B, C, N, M); return 1; }
    if (too_big(fn, (double)B * C * N, (double)B * C * M, (double)B * M)) return 1;
    const uint32_t total = (uint32_t)((int64_t)B * C * M);
    if (total == 0) return 0;
    if (!features || !idx || !out) { gs_set_error("%s: NULL pointer", fn); return 1; }
    k_gather<<<nblocks(total), TPB, 0, (cudaStream_t)stream>>>(total, C, N, M, features, idx, out);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int32_t gs_b200_pn2_three_interpolate(int32_t B, int32_t C, int32_t m, int32_t n, const float* features,
                                      const int32_t* idx, const float* weight, float* out, void* stream) {
    static const char* fn = "pn2_three_interpolate";
    if (B < 0 || C < 0 || m < 1 || n < 0) { gs_set_error("%s: B %d, C %d, m %d, n %d (need m >= 1)", fn, B, C, m, n); return 1; }
    if (too_big(fn, (double)B * C * m, (double)B * C * n, (double)B * n * 3)) return 1;
    const uint32_t total = (uint32_t)((int64_t)B * C * n);
    if (total == 0) return 0;
    if (!features || !idx || !weight || !out) { gs_set_error("%s: NULL pointer", fn); return 1; }
    k_three_interp<<<nblocks(total), TPB, 0, (cudaStream_t)stream>>>(total, C, m, n, features, idx, weight, out);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

size_t gs_b200_pn2_backward_scratch_bytes(int32_t B, int32_t C, int32_t N, int64_t M, int32_t three) {
    if (B < 0 || C < 0 || N < 1 || M < 0) { gs_set_error("pn2_backward_scratch_bytes: B %d, C %d, N %d, M %lld", B, C, N, (long long)M); return 0; }
    const int64_t Ms = three ? M * 3 : M;
    const size_t sb = scatter_bytes(B, C, N, Ms);
    if (!sb) return 0;
    return sb + (three ? al((size_t)B * C * Ms * 4) : 0) + 256;
}

int32_t gs_b200_pn2_gather_backward(int32_t B, int32_t C, int32_t N, int64_t M, const float* grad_out,
                                    const int32_t* idx, float* grad_features, void* scratch, void* stream) {
    static const char* fn = "pn2_gather_backward";
    if (B < 0 || C < 0 || N < 1 || M < 0) { gs_set_error("%s: B %d, C %d, N %d, M %lld", fn, B, C, N, (long long)M); return 1; }
    if (too_big(fn, (double)B * C * (N + 1), (double)B * C * M)) return 1;
    if ((int64_t)B * C * (N + 1) == 0) return 0;
    if (!grad_features || !scratch || ((int64_t)B * C * M && (!grad_out || !idx))) { gs_set_error("%s: NULL pointer", fn); return 1; }
    char* scr = (char*)(((uintptr_t)scratch + 255) & ~(uintptr_t)255);
    return scatter_fold(fn, B, C, N, M, grad_out, idx, grad_features, scr, (cudaStream_t)stream);
}

int32_t gs_b200_pn2_three_interpolate_backward(int32_t B, int32_t C, int32_t m, int32_t n, const float* grad_out,
                                               const int32_t* idx, const float* weight, float* grad_features,
                                               void* scratch, void* stream) {
    static const char* fn = "pn2_three_interpolate_backward";
    if (B < 0 || C < 0 || m < 1 || n < 0) { gs_set_error("%s: B %d, C %d, m %d, n %d", fn, B, C, m, n); return 1; }
    if (too_big(fn, (double)B * C * (m + 1), (double)B * C * n * 3)) return 1;
    if ((int64_t)B * C * (m + 1) == 0) return 0;
    const int64_t M = (int64_t)n * 3;
    if (!grad_features || !scratch || ((int64_t)B * C * n && (!grad_out || !idx || !weight))) { gs_set_error("%s: NULL pointer", fn); return 1; }
    cudaStream_t s = (cudaStream_t)stream;
    char* scr = (char*)(((uintptr_t)scratch + 255) & ~(uintptr_t)255);
    float* vals = (float*)scr;
    const uint32_t nv = (uint32_t)((int64_t)B * C * M);
    if (nv) { k_three_interp_vals<<<nblocks(nv), TPB, 0, s>>>(nv, C, n, grad_out, weight, vals); gs_count_launches(1); }
    return scatter_fold(fn, B, C, m, M, vals, idx, grad_features, scr + al((size_t)nv * 4), s);
}
