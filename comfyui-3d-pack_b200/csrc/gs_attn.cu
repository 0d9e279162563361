// Variable-length multi-head attention forward (flash_attn's varlen / dense entry points, head dim 64, fp16 and bf16)
// on the GPU (include/gs_b200_attn.h): a FlashAttention-2-style kernel on mma.sync tensor cores.
//
// A CTA owns 64 query rows (4 warps x 16) of one (sequence, head) and streams the sequence's keys and values in 64-row
// tiles through a double-buffered cp.async ring; rows past the sequence's end are zero-filled.  Per tile, S = Q.K^T
// (mma.sync.m16n8k16, fp32 sums), x = S * (scale * log2 e) in fp32, keys past the end set to -inf, then the online
// softmax on exp2: m' = max(m, max x), O *= exp2(m - m'), l = l * exp2(m - m') + sum p, p = exp2(x - m').  p is rounded
// to the input dtype in registers and reused as the A fragment of O += P.V, with V read by ldmatrix.trans.  At the
// end O is divided by l once (0 for an empty key set) and rounded once.  Every sum has a fixed order that depends only
// on the row's position in its sequence, so every output has the same bits on every run, whatever the batch around it.
#include "../../include/gs_b200_attn.h"
#include "gs_common.cuh"
#include "mma_sm90.cuh"

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <algorithm>
#include <climits>
#include <cmath>

namespace {

constexpr int D = 64;          // head dim
constexpr int BM = 64;         // query rows per CTA
constexpr int BN = 64;         // keys per tile
constexpr int LDS = D + 8;     // smem row pitch in halves (144 B): ldmatrix rows land on distinct bank quads
constexpr int NT = 128;        // 4 warps x 16 query rows

struct Attn {
    const void *q, *k, *v;
    void* out;
    int64_t q_row, q_head, k_row, k_head, v_row, v_head;
    const int32_t *cu_q, *cu_k;
    int64_t total_q, total_k, Lq, Lk;  // Lq / Lk: the dense sequence lengths when cu_q / cu_k is NULL
    int B, H, nqb;
    float sl2;                         // softmax_scale * log2(e)
};

template <typename T> __device__ __forceinline__ uint32_t pack2(float a, float b);
template <> __device__ __forceinline__ uint32_t pack2<__half>(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}
template <> __device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float a, float b) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}
template <typename T> __device__ __forceinline__ void mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <> __device__ __forceinline__ void mma<__half>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    mma16816(d, a, b0, b1);
}
template <> __device__ __forceinline__ void mma<__nv_bfloat16>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    mma16816_bf16(d, a, b0, b1);
}

// [start, end) of sequence b, clamped into [0, total]: a malformed cu_seqlens cannot move an access out of the tensor
__device__ __forceinline__ void seq_bounds(const int32_t* cu, int b, int64_t L, int64_t total, int64_t& s, int64_t& e) {
    if (cu) {
        s = min(max((int64_t)cu[b], (int64_t)0), total);
        e = min(max((int64_t)cu[b + 1], s), total);
    } else {
        s = (int64_t)b * L;
        e = s + L;
    }
}

// 64 rows x 64 dims of one head into a [64][LDS] tile: 512 16-byte chunks, 4 per thread; rows >= n are zero-filled
template <typename T>
__device__ __forceinline__ void load_tile(T* dst, const T* base, int64_t row0, int64_t n, int64_t rstride, int tid) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int e = tid + NT * j, r = e >> 3, c = (e & 7) * 8;
        const bool on = r < n;
        cp_async16(dst + r * LDS + c, on ? base + (row0 + r) * rstride + c : base, on ? 16 : 0);
    }
}

template <typename T>
__global__ void __launch_bounds__(NT) k_attn(Attn a) {
    __shared__ __align__(128) T sQ[BM * LDS];
    __shared__ __align__(128) T sK[2][BN * LDS];
    __shared__ __align__(128) T sV[2][BN * LDS];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int b = blockIdx.x / a.nqb, h = blockIdx.y;
    int64_t qs, qe, ks, ke;
    seq_bounds(a.cu_q, b, a.Lq, a.total_q, qs, qe);
    seq_bounds(a.cu_k, b, a.Lk, a.total_k, ks, ke);
    const int64_t lq = qe - qs, lk = ke - ks;
    const int ntiles = (int)((lk + BN - 1) / BN);
    const T* Q = (const T*)a.q + h * a.q_head;
    const T* K = (const T*)a.k + h * a.k_head;
    const T* V = (const T*)a.v + h * a.v_head;
    T* O = (T*)a.out;

    for (int64_t q0 = (int64_t)(blockIdx.x % a.nqb) * BM; q0 < lq; q0 += (int64_t)a.nqb * BM) {
        load_tile(sQ, Q, qs + q0, lq - q0, a.q_row, tid);
        if (ntiles > 0) {
            load_tile(sK[0], K, ks, lk, a.k_row, tid);
            load_tile(sV[0], V, ks, lk, a.v_row, tid);
        }
        cp_async_commit();

        float o[8][4], m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
        for (int i = 0; i < 8; i++)
#pragma unroll
            for (int j = 0; j < 4; j++) o[i][j] = 0.f;
        uint32_t qf[4][4];

        for (int kt = 0; kt < ntiles; kt++) {
            if (kt + 1 < ntiles) {
                const int64_t k0 = (int64_t)(kt + 1) * BN;
                load_tile(sK[(kt + 1) & 1], K, ks + k0, lk - k0, a.k_row, tid);
                load_tile(sV[(kt + 1) & 1], V, ks + k0, lk - k0, a.v_row, tid);
            }
            cp_async_commit();
            cp_async_wait<1>();
            __syncthreads();
            if (kt == 0) {
#pragma unroll
                for (int kk = 0; kk < 4; kk++)
                    ldmatrix_x4(qf[kk], sQ + (warp * 16 + (lane & 15)) * LDS + kk * 16 + (lane >> 4) * 8);
            }
            const T* Ks = sK[kt & 1];
            const T* Vs = sV[kt & 1];

            // S = Q.K^T: 16 rows x 64 keys per warp, as 8 n-tiles of 8 keys
            float s[8][4];
#pragma unroll
            for (int i = 0; i < 8; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) s[i][j] = 0.f;
#pragma unroll
            for (int kk = 0; kk < 4; kk++)
#pragma unroll
                for (int nj = 0; nj < 4; nj++) {
                    uint32_t bf[4];
                    ldmatrix_x4(bf, Ks + (nj * 16 + (lane & 7) + ((lane >> 4) << 3)) * LDS + kk * 16 + ((lane >> 3) & 1) * 8);
                    mma<T>(s[2 * nj], qf[kk], bf[0], bf[1]);
                    mma<T>(s[2 * nj + 1], qf[kk], bf[2], bf[3]);
                }

            // online softmax; thread holds rows g (s[.][0..1]) and g + 8 (s[.][2..3]) at keys ni*8 + 2t + {0, 1}
            const int64_t kleft = lk - (int64_t)kt * BN;
#pragma unroll
            for (int ni = 0; ni < 8; ni++)
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const float x = s[ni][j] * a.sl2;
                    s[ni][j] = ni * 8 + 2 * t + (j & 1) < kleft ? x : -INFINITY;
                }
            float alpha[2];
#pragma unroll
            for (int r = 0; r < 2; r++) {
                float mx = m[r];
#pragma unroll
                for (int ni = 0; ni < 8; ni++) mx = fmaxf(mx, fmaxf(s[ni][2 * r], s[ni][2 * r + 1]));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                alpha[r] = exp2f(m[r] - mx);   // m = -inf on the first tile: alpha = 0
                m[r] = mx;
                float sum = 0.f;
#pragma unroll
                for (int ni = 0; ni < 8; ni++) {
                    s[ni][2 * r] = exp2f(s[ni][2 * r] - mx);
                    s[ni][2 * r + 1] = exp2f(s[ni][2 * r + 1] - mx);
                    sum += s[ni][2 * r] + s[ni][2 * r + 1];
                }
                l[r] = l[r] * alpha[r] + sum;
            }
#pragma unroll
            for (int ni = 0; ni < 8; ni++) {
                o[ni][0] *= alpha[0]; o[ni][1] *= alpha[0];
                o[ni][2] *= alpha[1]; o[ni][3] *= alpha[1];
            }

            // O += P.V: P (rounded to T) is the A fragment of each 16-key step; V [key][dim] read transposed
#pragma unroll
            for (int kk = 0; kk < 4; kk++) {
                uint32_t pf[4];
                pf[0] = pack2<T>(s[2 * kk][0], s[2 * kk][1]);
                pf[1] = pack2<T>(s[2 * kk][2], s[2 * kk][3]);
                pf[2] = pack2<T>(s[2 * kk + 1][0], s[2 * kk + 1][1]);
                pf[3] = pack2<T>(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
                for (int nj = 0; nj < 4; nj++) {
                    uint32_t bf[4];
                    ldmatrix_x4_trans(bf, Vs + (kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS + nj * 16 + (lane >> 4) * 8);
                    mma<T>(o[2 * nj], pf, bf[0], bf[1]);
                    mma<T>(o[2 * nj + 1], pf, bf[2], bf[3]);
                }
            }
            __syncthreads();   // the next iteration's loads overwrite this tile's stage
        }
        cp_async_wait<0>();

        // O / l, rounded once, staged through this warp's own rows of sQ for 16-byte stores
        T* st = sQ + warp * 16 * LDS;
        __syncthreads();       // no warp still reads sQ (kt == 0 fragments, or the ring when ntiles == 0)
#pragma unroll
        for (int r = 0; r < 2; r++) {
            float lr = l[r];
            lr += __shfl_xor_sync(0xffffffffu, lr, 1);
            lr += __shfl_xor_sync(0xffffffffu, lr, 2);
#pragma unroll
            for (int ni = 0; ni < 8; ni++) {
                const float v0 = lr > 0.f ? __fdiv_rn(o[ni][2 * r], lr) : 0.f;
                const float v1 = lr > 0.f ? __fdiv_rn(o[ni][2 * r + 1], lr) : 0.f;
                *reinterpret_cast<uint32_t*>(st + (g + 8 * r) * LDS + ni * 8 + 2 * t) = pack2<T>(v0, v1);
            }
        }
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int e = lane + 32 * j, r = e >> 3, c = (e & 7) * 8;
            const int64_t row = q0 + warp * 16 + r;
            if (row < lq)
                *reinterpret_cast<uint4*>(O + ((qs + row) * a.H + h) * D + c) =
                    *reinterpret_cast<const uint4*>(st + r * LDS + c);
        }
        __syncthreads();       // sQ is reloaded by the next query block
    }
}

bool bad_view(const char* fn, const char* nm, const void* p, int64_t rs, int64_t hs) {
    if (!p) { gs_set_error("%s: %s is NULL", fn, nm); return true; }
    if (((uintptr_t)p & 15) || rs % 8 || hs % 8 || rs < 0 || hs < 0) {
        gs_set_error("%s: %s must be 16-byte aligned with row / head strides multiples of 8 elements (got %lld, %lld)",
                     fn, nm, (long long)rs, (long long)hs);
        return true;
    }
    return false;
}

}  // namespace

int32_t gs_b200_attn_forward(int32_t dtype, int32_t B, int32_t H, int32_t d, const void* q, int64_t q_row_stride,
                             int64_t q_head_stride, const void* k, int64_t k_row_stride, int64_t k_head_stride,
                             const void* v, int64_t v_row_stride, int64_t v_head_stride, const int32_t* cu_seqlens_q,
                             const int32_t* cu_seqlens_k, int64_t max_seqlen_q, int64_t max_seqlen_k, int64_t total_q,
                             int64_t total_k, float softmax_scale, void* out, void* stream) {
    static const char* fn = "attn_forward";
    if (dtype != GS_B200_ATTN_F16 && dtype != GS_B200_ATTN_BF16) { gs_set_error("%s: dtype %d", fn, dtype); return 1; }
    if (d != GS_B200_ATTN_HEAD_DIM) { gs_set_error("%s: head dim %d (only %d)", fn, d, GS_B200_ATTN_HEAD_DIM); return 1; }
    if (B < 0 || H < 1 || H > 65535 || max_seqlen_q < 0 || max_seqlen_k < 0 || total_q < 0 || total_k < 0) {
        gs_set_error("%s: B %d, H %d, max_seqlen %lld / %lld, total %lld / %lld", fn, B, H, (long long)max_seqlen_q,
                     (long long)max_seqlen_k, (long long)total_q, (long long)total_k);
        return 1;
    }
    if ((!cu_seqlens_q && (int64_t)B * max_seqlen_q != total_q) || (!cu_seqlens_k && (int64_t)B * max_seqlen_k != total_k)) {
        gs_set_error("%s: without cu_seqlens the total must be B * max_seqlen (%lld / %lld rows for B %d, L %lld / %lld)",
                     fn, (long long)total_q, (long long)total_k, B, (long long)max_seqlen_q, (long long)max_seqlen_k);
        return 1;
    }
    if (B == 0 || total_q == 0) return 0;
    if (!out || ((uintptr_t)out & 15)) { gs_set_error("%s: out must be non-NULL and 16-byte aligned", fn); return 1; }
    if (bad_view(fn, "q", q, q_row_stride, q_head_stride)) return 1;
    if (total_k > 0 && (bad_view(fn, "k", k, k_row_stride, k_head_stride) || bad_view(fn, "v", v, v_row_stride, v_head_stride)))
        return 1;
    Attn a{};
    a.q = q; a.k = k; a.v = v; a.out = out;
    a.q_row = q_row_stride; a.q_head = q_head_stride;
    a.k_row = k_row_stride; a.k_head = k_head_stride;
    a.v_row = v_row_stride; a.v_head = v_head_stride;
    a.cu_q = cu_seqlens_q; a.cu_k = cu_seqlens_k;
    a.total_q = total_q; a.total_k = total_k; a.Lq = max_seqlen_q; a.Lk = max_seqlen_k;
    a.B = B; a.H = H;
    a.sl2 = (float)((double)softmax_scale * 1.4426950408889634);
    // max_seqlen_q only sizes the grid: each CTA walks its sequence's query blocks with a stride of nqb
    const int64_t want = std::max<int64_t>(1, (max_seqlen_q + BM - 1) / BM);
    a.nqb = (int)std::min<int64_t>(want, INT_MAX / B);
    cudaStream_t s = (cudaStream_t)stream;
    const dim3 grid((unsigned)((int64_t)B * a.nqb), (unsigned)H);
    if (dtype == GS_B200_ATTN_F16) k_attn<__half><<<grid, NT, 0, s>>>(a);
    else k_attn<__nv_bfloat16><<<grid, NT, 0, s>>>(a);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
