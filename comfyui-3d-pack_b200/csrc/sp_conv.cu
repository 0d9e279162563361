// spconv's submanifold 3D convolution (SubMConv3d, k = 1 or 3, stride 1, dilation 1) on the GPU (include/gs_b200.h,
// "spconv" section): the neighbour map, the forward implicit GEMM (fp16 on tensor cores, fp32 on FFMA), dgrad,
// wgrad and dbias.
//
// Neighbour map (k = 3): each row's 32-bit key ((b*X + x)*Y + y)*Z + z is sorted with its row index as value by the
// stable onesweep radix sort (gs_sort_pairs_u32), so equal keys sit in ascending row order and the first valid one is
// the smallest row.  A row then finds its 27 neighbours with 9 binary searches, one per (dx, dy), each followed by a
// forward walk over dz; every coordinate is bounds-checked before a key is formed.
//
// GEMM: a CTA owns 64 output rows x 64 output channels and loops over the offsets present in its rows (the OR of
// their bitmasks) and over Cin in chunks.  Each step gathers the 64 input rows of one offset and the weight slab of
// that offset into shared memory; every output is one fixed-order sum, so results have the same bits on every run.
#include "../../include/gs_b200.h"
#include "gs_common.cuh"
#include "mma_sm90.cuh"

#include <cuda_fp16.h>
#include <algorithm>

namespace {

constexpr int TPB = 256;
constexpr uint32_t ROW_INVALID = 0x80000000u;      // sorted-row flag: the row lies outside the grid
constexpr uint32_t MASK_OFFSETS = 0x07ffffffu;     // bits 0..26 of a row's mask: offsets whose neighbour is present
constexpr uint32_t MASK_DUP = 0x80000000u;         // the row repeats the coordinate of a smaller row
constexpr int K3MAP = 27;

inline unsigned nblocks(int64_t n, int per = TPB) { return (unsigned)((n + per - 1) / per); }
inline size_t al(size_t b) { return (b + 255) & ~(size_t)255; }

// ---- neighbour map -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(TPB) k_keys(int N, int B, int X, int Y, int Z, const int32_t* __restrict__ idx,
                                              uint32_t* __restrict__ keys, uint32_t* __restrict__ rows) {
    const int i = blockIdx.x * TPB + threadIdx.x;
    if (i >= N) return;
    const int4 c = reinterpret_cast<const int4*>(idx)[i];
    const bool ok = (unsigned)c.x < (unsigned)B && (unsigned)c.y < (unsigned)X && (unsigned)c.z < (unsigned)Y &&
                    (unsigned)c.w < (unsigned)Z;
    keys[i] = ok ? (uint32_t)((((uint64_t)c.x * X + c.y) * Y + c.z) * Z + c.w) : 0xffffffffu;
    rows[i] = ok ? (uint32_t)i : ROW_INVALID | (uint32_t)i;
}

__device__ __forceinline__ int lower_bound(const uint32_t* __restrict__ k, int n, uint32_t t) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (k[mid] < t) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(TPB) k_search(int N, int B, int X, int Y, int Z, const int32_t* __restrict__ idx,
                                                const uint32_t* __restrict__ sk, const uint32_t* __restrict__ sr,
                                                int32_t* __restrict__ nbr, uint32_t* __restrict__ mask) {
    const int i = blockIdx.x * TPB + threadIdx.x;
    if (i >= N) return;
    const int4 c = reinterpret_cast<const int4*>(idx)[i];
    int32_t* o = nbr + (size_t)i * K3MAP;
    const bool ok = (unsigned)c.x < (unsigned)B && (unsigned)c.y < (unsigned)X && (unsigned)c.z < (unsigned)Y &&
                    (unsigned)c.w < (unsigned)Z;
    uint32_t m = 0;
    const int zlo = max(c.w - 1, 0), zhi = min(c.w + 1, Z - 1);
    for (int a = 0; a < 3; a++) {
        for (int b = 0; b < 3; b++) {
            const int xx = c.y + a - 1, yy = c.z + b - 1;
            const bool inside = ok && (unsigned)xx < (unsigned)X && (unsigned)yy < (unsigned)Y;
            int p = 0;
            uint32_t base = 0;
            if (inside) {
                base = (uint32_t)((((uint64_t)c.x * X + xx) * Y + yy) * Z);
                p = lower_bound(sk, N, base + (uint32_t)zlo);
            }
            for (int d = 0; d < 3; d++) {
                const int zz = c.w + d - 1, off = (a * 3 + b) * 3 + d;
                int32_t j = -1;
                if (inside && zz >= zlo && zz <= zhi) {
                    const uint32_t t = base + (uint32_t)zz;
                    while (p < N && sk[p] < t) p++;
                    int q = p;
                    while (q < N && sk[q] == t && (sr[q] & ROW_INVALID)) q++;
                    if (q < N && sk[q] == t) j = (int32_t)sr[q];
                }
                o[off] = j;
                if (j >= 0) m |= 1u << off;
            }
        }
    }
    if (m && o[13] != i) m |= MASK_DUP;
    mask[i] = m;
}

// upstream gradient for dgrad: each coordinate's smallest valid row receives the sum of its valid rows' gradients
// (ascending row, fp32, one rounding); only those rows are ever a neighbour, so the other rows are not written.  One
// warp per sorted position: the position holding the first valid row of a run of equal keys does the sum.
template <typename T>
__global__ void __launch_bounds__(TPB) k_fold_dups(int N, int C, const uint32_t* __restrict__ sk,
                                                   const uint32_t* __restrict__ sr, const T* __restrict__ g,
                                                   T* __restrict__ out) {
    const int p = (int)((blockIdx.x * (unsigned)TPB + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (p >= N || (sr[p] & ROW_INVALID)) return;
    const uint32_t t = sk[p];
    for (int q = p - 1; q >= 0 && sk[q] == t; q--)
        if (!(sr[q] & ROW_INVALID)) return;
    int end = p + 1;
    while (end < N && sk[end] == t) end++;
    T* o = out + (size_t)sr[p] * C;
    for (int c = lane; c < C; c += 32) {
        float acc = 0.f;
        for (int q = p; q < end; q++)
            if (!(sr[q] & ROW_INVALID)) acc += (float)g[(size_t)sr[q] * C + c];
        o[c] = T(acc);
    }
}

// ---- implicit GEMM -------------------------------------------------------------------------------------------------
// out[r, n] = bias[n] + sum over present offsets o (ascending) and input channels c (ascending) of
// in[nbr[r, o], c] * w[n, slab(o), c], with w laid out [Nout][K3][Kin].  nbr == NULL: k = 1, every row reads itself.
// dgrad runs the same loop with w = W^T ([Cin][K3][Cout]) and slab(o) = K3 - 1 - o: a submanifold map with odd k is
// symmetric, so row j's neighbour at -o is the row that reads j at +o.  Rows flagged MASK_DUP then get 0.
struct Gemm {
    int N, Kin, Nout, K3, dgrad;
    const void* in; const int32_t* nbr; const uint32_t* mask; const void* w; const void* bias; void* out;
};

__device__ __forceinline__ uint32_t tile_offsets(const Gemm& a, int row0, int tid, uint32_t* s_mask) {
    if (tid == 0) *s_mask = 0;
    __syncthreads();
    if (tid < 64 && row0 + tid < a.N) atomicOr(s_mask, a.nbr ? a.mask[row0 + tid] & MASK_OFFSETS : 1u);
    __syncthreads();
    return *s_mask;
}

__device__ __forceinline__ int src_row(const Gemm& a, int r, int o) {
    if (r >= a.N) return -1;
    return a.nbr ? a.nbr[(size_t)r * a.K3 + o] : r;
}

// fp16: mma.sync.m16n8k16 (fp16 x fp16 -> fp32).  64 x 64 CTA tile, 4 warps of 32 x 32, Kin chunks of 32, a 3-stage
// cp.async ring (16 B copies with zero-fill for absent rows and tails) padded to 40 halves per row so that ldmatrix
// reads are free of bank conflicts.  VEC = false (Kin not a multiple of 8 or an unaligned base) loads element-wise.
constexpr int HBM = 64, HBN = 64, HBK = 32, HST = 3, HLD = HBK + 8, HT = 128;

template <bool VEC>
__device__ __forceinline__ void load_chunk16(__half* dst, const __half* base, int rowsrc, int c, int lim) {
    if (VEC) {
        const bool on = rowsrc >= 0 && c < lim;
        cp_async16(dst, on ? base + (size_t)rowsrc * lim + c : base, on ? 16 : 0);
    } else {
        __align__(16) __half v[8];
#pragma unroll
        for (int e = 0; e < 8; e++)
            v[e] = (rowsrc >= 0 && c + e < lim) ? base[(size_t)rowsrc * lim + c + e] : __float2half_rn(0.f);
        *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(v);
    }
}

template <bool VEC>
__global__ void __launch_bounds__(HT) k_gemm_f16(Gemm a) {
    __shared__ __align__(128) __half sA[HST][HBM * HLD];
    __shared__ __align__(128) __half sB[HST][HBN * HLD];
    __shared__ uint32_t s_mask;
    __shared__ int s_off[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int row0 = blockIdx.x * HBM, col0 = blockIdx.y * HBN;
    const uint32_t m = tile_offsets(a, row0, tid, &s_mask);
    if (tid == 0)
        for (uint32_t r = m, k = 0; r; r &= r - 1) s_off[k++] = __ffs(r) - 1;
    __syncthreads();
    const int noff = __popc(m);
    const int nck = (a.Kin + HBK - 1) / HBK, steps = noff * nck;
    const __half* in = (const __half*)a.in;
    const __half* w = (const __half*)a.w;

    // each thread copies 2 of the 256 16-byte chunks of A (64 rows x 4) and 2 of B per step
    auto load = [&](int step, int st) {
        const int o = s_off[step / nck], c0 = (step % nck) * HBK, slab = a.dgrad ? a.K3 - 1 - o : o;
#pragma unroll
        for (int j = 0; j < 2; j++) {
            const int e = tid + HT * j, r = e >> 2, cc = (e & 3) * 8;
            load_chunk16<VEC>(&sA[st][r * HLD + cc], in, src_row(a, row0 + r, o), c0 + cc, a.Kin);
            const int n = col0 + r;
            load_chunk16<VEC>(&sB[st][r * HLD + cc], w + (size_t)slab * a.Kin, n < a.Nout ? n * a.K3 : -1, c0 + cc,
                              a.Kin);
        }
    };

    float acc[2][4][4];
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int k = 0; k < 4; k++) acc[i][j][k] = 0.f;

#pragma unroll
    for (int s = 0; s < HST - 1; s++) {
        if (s < steps) load(s, s);
        cp_async_commit();
    }
    const int wm = warp >> 1, wn = warp & 1;
    for (int step = 0; step < steps; step++) {
        cp_async_wait<HST - 2>();
        __syncthreads();
        const int nxt = step + HST - 1;
        if (nxt < steps) load(nxt, nxt % HST);
        cp_async_commit();
        const __half* A = sA[step % HST];
        const __half* Bm = sB[step % HST];
#pragma unroll
        for (int kk = 0; kk < HBK / 16; kk++) {
            uint32_t af[2][4], bf[2][4];
#pragma unroll
            for (int mi = 0; mi < 2; mi++)
                ldmatrix_x4(af[mi], A + (wm * 32 + mi * 16 + (lane & 15)) * HLD + kk * 16 + (lane >> 4) * 8);
#pragma unroll
            for (int nj = 0; nj < 2; nj++)
                ldmatrix_x4(bf[nj], Bm + (wn * 32 + nj * 16 + (lane & 7) + ((lane >> 4) << 3)) * HLD + kk * 16 +
                                        ((lane >> 3) & 1) * 8);
#pragma unroll
            for (int mi = 0; mi < 2; mi++)
#pragma unroll
                for (int ni = 0; ni < 4; ni++)
                    mma16816(acc[mi][ni], af[mi], bf[ni >> 1][(ni & 1) * 2], bf[ni >> 1][(ni & 1) * 2 + 1]);
        }
    }
    cp_async_wait<0>();

    const int g = lane >> 2, t = lane & 3;
    const __half* bias = (const __half*)a.bias;
    __half* out = (__half*)a.out;
#pragma unroll
    for (int mi = 0; mi < 2; mi++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int r = row0 + wm * 32 + mi * 16 + g + h * 8;
            if (r >= a.N) continue;
            const bool zero = a.dgrad && a.nbr && (a.mask[r] & MASK_DUP);
#pragma unroll
            for (int ni = 0; ni < 4; ni++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int n = col0 + wn * 32 + ni * 8 + 2 * t + e;
                    if (n >= a.Nout) continue;
                    const float v = zero ? 0.f : acc[mi][ni][h * 2 + e] + (bias ? __half2float(bias[n]) : 0.f);
                    out[(size_t)r * a.Nout + n] = __float2half_rn(v);
                }
        }
}

// fp32: true fp32 FFMA.  64 x 64 CTA tile, 256 threads of 4 x 4 outputs, Kin chunks of 16; each output is one fmaf
// chain in (offset, channel) order.
constexpr int FBM = 64, FBN = 64, FBK = 16;

__global__ void __launch_bounds__(TPB) k_gemm_f32(Gemm a) {
    __shared__ float sA[FBK][FBM + 4];
    __shared__ float sB[FBK][FBN + 4];
    __shared__ uint32_t s_mask;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int row0 = blockIdx.x * FBM, col0 = blockIdx.y * FBN;
    uint32_t m = tile_offsets(a, row0, tid, &s_mask);
    const float* in = (const float*)a.in;
    const float* w = (const float*)a.w;
    float acc[4][4] = {};
    const int lr = tid >> 2, lc = (tid & 3) * 4;       // loader: row (or output channel) lr, channels lc..lc+3
    while (m) {
        const int o = __ffs(m) - 1;
        m &= m - 1;
        const int slab = a.dgrad ? a.K3 - 1 - o : o;
        const int src = src_row(a, row0 + lr, o);
        const int n = col0 + lr;
        const float* wrow = n < a.Nout ? w + ((size_t)n * a.K3 + slab) * a.Kin : nullptr;
        for (int c0 = 0; c0 < a.Kin; c0 += FBK) {
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int c = c0 + lc + e;
                sA[lc + e][lr] = (src >= 0 && c < a.Kin) ? in[(size_t)src * a.Kin + c] : 0.f;
                sB[lc + e][lr] = (wrow && c < a.Kin) ? wrow[c] : 0.f;
            }
            __syncthreads();
#pragma unroll
            for (int k = 0; k < FBK; k++) {
                float av[4], bv[4];
#pragma unroll
                for (int i = 0; i < 4; i++) { av[i] = sA[k][ty * 4 + i]; bv[i] = sB[k][tx * 4 + i]; }
#pragma unroll
                for (int i = 0; i < 4; i++)
#pragma unroll
                    for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
            }
            __syncthreads();
        }
    }
    const float* bias = (const float*)a.bias;
    float* out = (float*)a.out;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int r = row0 + ty * 4 + i;
        if (r >= a.N) continue;
        const bool zero = a.dgrad && a.nbr && (a.mask[r] & MASK_DUP);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int n = col0 + tx * 4 + j;
            if (n < a.Nout) out[(size_t)r * a.Nout + n] = zero ? 0.f : acc[i][j] + (bias ? bias[n] : 0.f);
        }
    }
}

// ---- wgrad / dbias ----------------------------------------------------------------------------------------------------
// partial[chunk][co][o][ci] = sum over the chunk's rows r (ascending) of dout[r, co] * in[nbr[r, o], ci], one fmaf
// chain in fp32; the chunks are then added in ascending order (k_sum_chunks).  Tile 64 co x 64 ci, rows in steps of 16.
template <typename T>
__global__ void __launch_bounds__(TPB) k_wgrad(int N, int Cin, int Cout, int K3, int chunk, const T* __restrict__ x,
                                               const T* __restrict__ dout, const int32_t* __restrict__ nbr,
                                               float* __restrict__ partial) {
    __shared__ float sD[16][64 + 4];
    __shared__ float sX[16][64 + 4];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int ci0 = blockIdx.x * 64, co0 = blockIdx.y * 64, o = blockIdx.z % K3, ch = blockIdx.z / K3;
    const int r0 = ch * chunk, r1 = min(N, r0 + chunk);
    float acc[4][4] = {};
    const int lr = tid >> 4, lc = (tid & 15) * 4;      // loader: row lr of the step, channels lc..lc+3
    for (int rb = r0; rb < r1; rb += 16) {
        const int r = rb + lr;
        const int src = r < r1 ? (nbr ? nbr[(size_t)r * K3 + o] : r) : -1;
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const int co = co0 + lc + e, ci = ci0 + lc + e;
            sD[lr][lc + e] = (r < r1 && co < Cout) ? (float)dout[(size_t)r * Cout + co] : 0.f;
            sX[lr][lc + e] = (src >= 0 && ci < Cin) ? (float)x[(size_t)src * Cin + ci] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 16; k++) {
            float dv[4], xv[4];
#pragma unroll
            for (int i = 0; i < 4; i++) { dv[i] = sD[k][ty * 4 + i]; xv[i] = sX[k][tx * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = fmaf(dv[i], xv[j], acc[i][j]);
        }
        __syncthreads();
    }
    float* p = partial + (size_t)ch * Cout * K3 * Cin;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int co = co0 + ty * 4 + i;
        if (co >= Cout) continue;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int ci = ci0 + tx * 4 + j;
            if (ci < Cin) p[((size_t)co * K3 + o) * Cin + ci] = acc[i][j];
        }
    }
}

// partial[chunk][c] = sum of dout[r, c] over the chunk's rows, ascending
template <typename T>
__global__ void __launch_bounds__(TPB) k_dbias(int N, int Cout, int chunk, const T* __restrict__ dout,
                                               float* __restrict__ partial) {
    const int c = blockIdx.x * TPB + threadIdx.x, ch = blockIdx.y;
    if (c >= Cout) return;
    const int r1 = min(N, (ch + 1) * chunk);
    float acc = 0.f;
    for (int r = ch * chunk; r < r1; r++) acc += (float)dout[(size_t)r * Cout + c];
    partial[(size_t)ch * Cout + c] = acc;
}

template <typename T>
__global__ void __launch_bounds__(TPB) k_sum_chunks(int64_t M, int nch, const float* __restrict__ partial,
                                                    T* __restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * TPB + threadIdx.x;
    if (e >= M) return;
    float acc = 0.f;
    for (int ch = 0; ch < nch; ch++) acc += partial[(size_t)ch * M + e];
    out[e] = T(acc);
}

// W [Cout][K3][Cin] -> W^T [Cin][K3][Cout]
template <typename T>
__global__ void __launch_bounds__(TPB) k_transpose_w(int Cin, int Cout, int K3, const T* __restrict__ w, T* __restrict__ wt) {
    const int64_t e = (int64_t)blockIdx.x * TPB + threadIdx.x;
    if (e >= (int64_t)Cin * Cout * K3) return;
    const int co = (int)(e % Cout);
    const int64_t r = e / Cout;
    const int o = (int)(r % K3), ci = (int)(r / K3);
    wt[e] = w[((size_t)co * K3 + o) * Cin + ci];
}

// ---- host side -------------------------------------------------------------------------------------------------------
bool bad_dims(const char* fn, int dtype, int64_t N, int Cin, int Cout, int k) {
    if (dtype != GS_B200_SPCONV_F32 && dtype != GS_B200_SPCONV_F16) { gs_set_error("%s: dtype %d", fn, dtype); return true; }
    if (N < 0 || Cin < 1 || Cout < 1 || (k != 1 && k != 3)) {
        gs_set_error("%s: N %lld, Cin %d, Cout %d, k %d (need N >= 0, channels >= 1, k 1 or 3)", fn, (long long)N, Cin, Cout, k);
        return true;
    }
    if (N > GS_B200_SPCONV_MAX_ROWS || (double)N * std::max(Cin, Cout) >= 2147483648.0 ||
        (double)Cin * Cout * k * k * k >= 2147483648.0) {
        gs_set_error("%s: N %lld x %d / %d channels is too large", fn, (long long)N, Cin, Cout);
        return true;
    }
    return false;
}

// wgrad row chunks: a function of the shape alone, so the partial sums, and the bits, never depend on the device
void wgrad_chunks(int64_t N, int Cin, int Cout, int K3, int& chunk, int& nch) {
    const int64_t per = (int64_t)Cin * Cout * K3 + Cout;
    const int64_t cap = std::max<int64_t>(1, std::min<int64_t>(256, ((int64_t)1 << 25) / per));
    int64_t c = std::max<int64_t>(1024, (N + cap - 1) / cap);
    c = (c + 15) / 16 * 16;
    chunk = (int)c;
    nch = (int)std::max<int64_t>(1, (N + c - 1) / c);
}

int gemm(int dtype, const Gemm& a, cudaStream_t s) {
    if (a.N == 0) return 0;
    if (dtype == GS_B200_SPCONV_F16) {
        const dim3 grid(nblocks(a.N, HBM), nblocks(a.Nout, HBN));
        const bool vec = a.Kin % 8 == 0 && ((uintptr_t)a.in & 15) == 0 && ((uintptr_t)a.w & 15) == 0;
        if (vec) k_gemm_f16<true><<<grid, HT, 0, s>>>(a);
        else k_gemm_f16<false><<<grid, HT, 0, s>>>(a);
    } else {
        k_gemm_f32<<<dim3(nblocks(a.N, FBM), nblocks(a.Nout, FBN)), TPB, 0, s>>>(a);
    }
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

}  // namespace

size_t gs_b200_spconv_map_scratch_bytes(int64_t N) {
    if (N < 0 || N > GS_B200_SPCONV_MAX_ROWS) { gs_set_error("spconv_map_scratch_bytes: N %lld", (long long)N); return 0; }
    return al((size_t)N * 4) * 2 + al(gs_sort_scratch_bytes(N)) + 256;
}

int32_t gs_b200_spconv_build_map(int64_t N, int32_t B, int32_t X, int32_t Y, int32_t Z, const int32_t* indices,
                                 int32_t* nbr, uint32_t* mask, uint32_t* sorted_keys, uint32_t* sorted_rows,
                                 void* scratch, void* stream) {
    static const char* fn = "spconv_build_map";
    if (N < 0 || N > GS_B200_SPCONV_MAX_ROWS || B < 1 || X < 1 || Y < 1 || Z < 1) {
        gs_set_error("%s: N %lld, batch %d, spatial shape [%d, %d, %d]", fn, (long long)N, B, X, Y, Z);
        return 1;
    }
    if ((double)B * X * Y * Z > 4294967296.0) { gs_set_error("%s: B*X*Y*Z exceeds 2^32", fn); return 1; }
    if (N == 0) return 0;
    if (!indices || !nbr || !mask || !sorted_keys || !sorted_rows || !scratch) { gs_set_error("%s: NULL pointer", fn); return 1; }
    if (((uintptr_t)indices & 15) != 0) { gs_set_error("%s: indices must be 16-byte aligned", fn); return 1; }
    cudaStream_t s = (cudaStream_t)stream;
    char* scr = (char*)(((uintptr_t)scratch + 255) & ~(uintptr_t)255);
    uint32_t* keys_alt = (uint32_t*)scr;
    uint32_t* rows_alt = (uint32_t*)(scr + al((size_t)N * 4));
    void* sort_scratch = scr + 2 * al((size_t)N * 4);
    const int n = (int)N;
    k_keys<<<nblocks(n), TPB, 0, s>>>(n, B, X, Y, Z, indices, sorted_keys, sorted_rows);
    gs_count_launches(1);
    int alt = 0;
    if (gs_sort_pairs_u32(sorted_keys, keys_alt, sorted_rows, rows_alt, N, 0, 32, sort_scratch, &alt, s)) return 1;
    if (alt) {
        GS_CUDA_CHECK(cudaMemcpyAsync(sorted_keys, keys_alt, (size_t)N * 4, cudaMemcpyDeviceToDevice, s));
        GS_CUDA_CHECK(cudaMemcpyAsync(sorted_rows, rows_alt, (size_t)N * 4, cudaMemcpyDeviceToDevice, s));
    }
    k_search<<<nblocks(n), TPB, 0, s>>>(n, B, X, Y, Z, indices, sorted_keys, sorted_rows, nbr, mask);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int32_t gs_b200_spconv_forward(int32_t dtype, int64_t N, int32_t Cin, int32_t Cout, int32_t k, const void* features,
                               const int32_t* nbr, const uint32_t* mask, const void* weight, const void* bias,
                               void* out, void* stream) {
    static const char* fn = "spconv_forward";
    if (bad_dims(fn, dtype, N, Cin, Cout, k)) return 1;
    if (N == 0) return 0;
    if (!features || !weight || !out || (k == 3 && (!nbr || !mask))) { gs_set_error("%s: NULL pointer", fn); return 1; }
    const Gemm a{(int)N, Cin, Cout, k * k * k, 0, features, k == 3 ? nbr : nullptr, mask, weight, bias, out};
    return gemm(dtype, a, (cudaStream_t)stream);
}

size_t gs_b200_spconv_backward_scratch_bytes(int32_t dtype, int64_t N, int32_t Cin, int32_t Cout, int32_t k) {
    if (bad_dims("spconv_backward_scratch_bytes", dtype, N, Cin, Cout, k)) return 0;
    const size_t elt = dtype == GS_B200_SPCONV_F16 ? 2 : 4;
    const int K3 = k * k * k;
    int chunk, nch;
    wgrad_chunks(N, Cin, Cout, K3, chunk, nch);
    const size_t wgrad = al((size_t)nch * ((size_t)Cin * Cout * K3 + Cout) * 4);
    const size_t dgrad = al((size_t)Cin * Cout * K3 * elt) + al((size_t)N * Cout * elt);
    return std::max(wgrad, dgrad) + 256;
}

int32_t gs_b200_spconv_dgrad(int32_t dtype, int64_t N, int32_t Cin, int32_t Cout, int32_t k, const void* grad_out,
                             const int32_t* nbr, const uint32_t* mask, const uint32_t* sorted_keys,
                             const uint32_t* sorted_rows, const void* weight, void* grad_features, void* scratch,
                             void* stream) {
    static const char* fn = "spconv_dgrad";
    if (bad_dims(fn, dtype, N, Cin, Cout, k)) return 1;
    if (N == 0) return 0;
    if (!grad_out || !weight || !grad_features || !scratch || (k == 3 && (!nbr || !mask || !sorted_keys || !sorted_rows))) {
        gs_set_error("%s: NULL pointer", fn);
        return 1;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const int K3 = k * k * k;
    const size_t elt = dtype == GS_B200_SPCONV_F16 ? 2 : 4;
    char* scr = (char*)(((uintptr_t)scratch + 255) & ~(uintptr_t)255);
    void* wt = scr;
    void* gfold = scr + al((size_t)Cin * Cout * K3 * elt);
    const int64_t nw = (int64_t)Cin * Cout * K3;
    const int n = (int)N;
    if (dtype == GS_B200_SPCONV_F16) {
        k_transpose_w<__half><<<nblocks(nw), TPB, 0, s>>>(Cin, Cout, K3, (const __half*)weight, (__half*)wt);
        if (k == 3)
            k_fold_dups<__half><<<nblocks((int64_t)n * 32), TPB, 0, s>>>(n, Cout, sorted_keys, sorted_rows,
                                                                       (const __half*)grad_out, (__half*)gfold);
    } else {
        k_transpose_w<float><<<nblocks(nw), TPB, 0, s>>>(Cin, Cout, K3, (const float*)weight, (float*)wt);
        if (k == 3)
            k_fold_dups<float><<<nblocks((int64_t)n * 32), TPB, 0, s>>>(n, Cout, sorted_keys, sorted_rows,
                                                                      (const float*)grad_out, (float*)gfold);
    }
    gs_count_launches(k == 3 ? 2 : 1);
    const Gemm a{n, Cout, Cin, K3, 1, k == 3 ? gfold : grad_out, k == 3 ? nbr : nullptr, mask, wt, nullptr, grad_features};
    return gemm(dtype, a, s);
}

int32_t gs_b200_spconv_wgrad(int32_t dtype, int64_t N, int32_t Cin, int32_t Cout, int32_t k, const void* features,
                             const void* grad_out, const int32_t* nbr, void* grad_weight, void* grad_bias,
                             void* scratch, void* stream) {
    static const char* fn = "spconv_wgrad";
    if (bad_dims(fn, dtype, N, Cin, Cout, k)) return 1;
    if (!grad_weight && !grad_bias) return 0;
    const int K3 = k * k * k;
    const size_t elt = dtype == GS_B200_SPCONV_F16 ? 2 : 4;
    cudaStream_t s = (cudaStream_t)stream;
    if (N == 0) {
        if (grad_weight) GS_CUDA_CHECK(cudaMemsetAsync(grad_weight, 0, (size_t)Cout * K3 * Cin * elt, s));
        if (grad_bias) GS_CUDA_CHECK(cudaMemsetAsync(grad_bias, 0, (size_t)Cout * elt, s));
        return 0;
    }
    if (!features || !grad_out || !scratch || (k == 3 && !nbr)) { gs_set_error("%s: NULL pointer", fn); return 1; }
    int chunk, nch;
    wgrad_chunks(N, Cin, Cout, K3, chunk, nch);
    float* part = (float*)(((uintptr_t)scratch + 255) & ~(uintptr_t)255);
    const int64_t M = (int64_t)Cout * K3 * Cin;
    float* part_b = part + (size_t)nch * M;
    const int n = (int)N;
    const int32_t* map = k == 3 ? nbr : nullptr;
    const dim3 wg(nblocks(Cin, 64), nblocks(Cout, 64), (unsigned)(K3 * nch));
    if (dtype == GS_B200_SPCONV_F16) {
        if (grad_weight) {
            k_wgrad<__half><<<wg, TPB, 0, s>>>(n, Cin, Cout, K3, chunk, (const __half*)features, (const __half*)grad_out, map, part);
            k_sum_chunks<__half><<<nblocks(M), TPB, 0, s>>>(M, nch, part, (__half*)grad_weight);
        }
        if (grad_bias) {
            k_dbias<__half><<<dim3(nblocks(Cout), nch), TPB, 0, s>>>(n, Cout, chunk, (const __half*)grad_out, part_b);
            k_sum_chunks<__half><<<nblocks(Cout), TPB, 0, s>>>(Cout, nch, part_b, (__half*)grad_bias);
        }
    } else {
        if (grad_weight) {
            k_wgrad<float><<<wg, TPB, 0, s>>>(n, Cin, Cout, K3, chunk, (const float*)features, (const float*)grad_out, map, part);
            k_sum_chunks<float><<<nblocks(M), TPB, 0, s>>>(M, nch, part, (float*)grad_weight);
        }
        if (grad_bias) {
            k_dbias<float><<<dim3(nblocks(Cout), nch), TPB, 0, s>>>(n, Cout, chunk, (const float*)grad_out, part_b);
            k_sum_chunks<float><<<nblocks(Cout), TPB, 0, s>>>(Cout, nch, part_b, (float*)grad_bias);
        }
    }
    gs_count_launches((grad_weight ? 2 : 0) + (grad_bias ? 2 : 0));
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
