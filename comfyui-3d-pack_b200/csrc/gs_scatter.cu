// torch_scatter's scatter_sum / scatter_mean / scatter_max on the GPU (include/gs_b200.h, "scatter" section).
//
// Every kernel walks one of four element orders, described by a Geo: a list of dimensions (innermost last) with,
// per dimension, its size and its element stride in each tensor the kernel touches.  A linear thread id is decoded
// into per-tensor offsets and the coordinate along the scatter dimension.  A tensor that broadcasts has stride 0.
//
// "Index rows" are the combinations of the non-scatter coordinates along which the index varies (size > 1 and a
// non-zero index stride); "columns" are those along which it is broadcast.  The fp32 sum and mean sort
// (row * dim_size + index, position) pairs once per index row with the stable onesweep sort, so each output slot's
// list is in ascending position, and then fold each list in that order, one thread per (slot, column).  That is the
// left fold torch's CPU scatter_add_ makes, so the bits do not depend on the schedule.  Integer sums use integer
// atomics (exact).  Max is an atomicMax over an order-preserving key, then an atomicMin over the positions that hold
// the maximum: both results are independent of the order in which the atomics land.
#include "../../include/gs_b200.h"
#include "gs_common.cuh"

#include <float.h>
#include <stdlib.h>
#include <algorithm>

namespace {

constexpr int GMAX = GS_B200_SCATTER_MAX_DIMS;
enum { S_SRC = 0, S_IDX, S_OUT, S_AUX, S_GS, S_ROW, NS };    // src, index, out, contiguous out (argmax), grad_src, row id

struct Geo {
    int nd;                   // dimensions in the list
    int pd;                   // list position of the scatter dimension (-1: absent)
    uint32_t size[GMAX];
    int64_t st[GMAX][NS];
    int64_t dst[NS];          // strides along the scatter dimension, for offsets the index value selects
};

__device__ __forceinline__ uint32_t geo_decode(const Geo& g, uint32_t t, int64_t (&off)[NS]) {
    uint32_t p = 0;
#pragma unroll
    for (int s = 0; s < NS; s++) off[s] = 0;
#pragma unroll
    for (int k = GMAX - 1; k >= 0; k--) {
        if (k >= g.nd) continue;
        const uint32_t c = t % g.size[k];
        t /= g.size[k];
        if (k == g.pd) p = c;
#pragma unroll
        for (int s = 0; s < NS; s++) off[s] += (int64_t)c * g.st[k][s];
    }
    return p;
}

constexpr int TPB = 256;
inline unsigned nblocks(int64_t n) { return (unsigned)((n + TPB - 1) / TPB); }

// ---- index range: min and max over the distinct index elements (one thread per (row, position)) ----------------
__global__ void k_range_init(int64_t* range) { range[0] = INT64_MAX; range[1] = INT64_MIN; }

__global__ void __launch_bounds__(TPB) k_range(Geo g, uint32_t n, const int64_t* __restrict__ index, int64_t* range) {
    long long lo = INT64_MAX, hi = INT64_MIN;
    for (uint32_t t = blockIdx.x * TPB + threadIdx.x; t < n; t += gridDim.x * TPB) {
        int64_t off[NS];
        geo_decode(g, t, off);
        const long long v = index[off[S_IDX]];
        lo = min(lo, v); hi = max(hi, v);
    }
    __shared__ long long s_lo[TPB / 32], s_hi[TPB / 32];
    for (int o = 16; o; o >>= 1) {
        lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    if ((threadIdx.x & 31) == 0) { s_lo[threadIdx.x >> 5] = lo; s_hi[threadIdx.x >> 5] = hi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < TPB / 32; w++) { lo = min(lo, s_lo[w]); hi = max(hi, s_hi[w]); }
        atomicMin((long long*)range, lo);
        atomicMax((long long*)range + 1, hi);
    }
}

// ---- fp32 sum / mean -----------------------------------------------------------------------------------------------
// keys in (row, position) order, so the stable sort keeps each slot's positions ascending
__global__ void __launch_bounds__(TPB) k_keys(Geo g, uint32_t n, const int64_t* __restrict__ index, int64_t dim_size,
                                              uint32_t* keys, uint32_t* vals, uint32_t* counts) {
    const uint32_t t = blockIdx.x * TPB + threadIdx.x;
    if (t >= n) return;
    int64_t off[NS];
    const uint32_t p = geo_decode(g, t, off);
    int64_t j = index[off[S_IDX]];
    j = min(max(j, (int64_t)0), dim_size - 1);          // validated by the caller; never address outside counts
    const uint32_t key = (uint32_t)(off[S_ROW] * dim_size + j);
    keys[t] = key;
    vals[t] = p;
    atomicAdd(counts + key, 1u);
}

// one thread per (row, slot, column): out = (out0 or +0) + src[p0] + src[p1] + ... in ascending position
template <bool MEAN>
__global__ void __launch_bounds__(TPB) k_fold(Geo g, uint32_t n, int64_t dim_size, const float* __restrict__ src,
                                              float* out, int has_out, const uint32_t* __restrict__ pos,
                                              const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ counts) {
    const uint32_t t = blockIdx.x * TPB + threadIdx.x;
    if (t >= n) return;
    int64_t off[NS];
    const uint32_t j = geo_decode(g, t, off);
    const uint32_t key = (uint32_t)(off[S_ROW] * dim_size + j);
    const uint32_t beg = offsets[key], cnt = counts[key];
    const float* s = src + off[S_SRC];
    const int64_t ss = g.dst[S_SRC];
    float acc = has_out ? out[off[S_OUT]] : 0.f;
    uint32_t i = 0;
    for (; i + 8 <= cnt; i += 8) {                       // loads first, then the adds in order
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; u++) v[u] = s[(int64_t)pos[beg + i + u] * ss];
#pragma unroll
        for (int u = 0; u < 8; u++) acc += v[u];
    }
    for (; i < cnt; i++) acc += s[(int64_t)pos[beg + i] * ss];
    if (MEAN) acc = acc / (float)max(cnt, 1u);
    out[off[S_OUT]] = acc;
}

// ---- integer sum ---------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(TPB) k_fill_zero(Geo g, uint32_t n, T* out) {
    const uint32_t t = blockIdx.x * TPB + threadIdx.x;
    if (t >= n) return;
    int64_t off[NS];
    geo_decode(g, t, off);
    out[off[S_OUT]] = 0;
}

__device__ __forceinline__ void int_add(int32_t* a, int32_t v) { atomicAdd((int*)a, (int)v); }
__device__ __forceinline__ void int_add(int64_t* a, int64_t v) {
    atomicAdd((unsigned long long*)a, (unsigned long long)v);    // two's complement: the same bits as a signed add
}

template <typename T>
__global__ void __launch_bounds__(TPB) k_isum(Geo g, uint32_t n, const T* __restrict__ src,
                                              const int64_t* __restrict__ index, int64_t dim_size, T* out) {
    const uint32_t t = blockIdx.x * TPB + threadIdx.x;
    if (t >= n) return;
    int64_t off[NS];
    geo_decode(g, t, off);
    const int64_t j = index[off[S_IDX]];
    if (j < 0 || j >= dim_size) return;
    int_add(out + off[S_OUT] + j * g.dst[S_OUT], src[off[S_SRC]]);
}

// ---- max -----------------------------------------------------------------------------------------------------------
template <typename T> struct MaxKey;
template <> struct MaxKey<float> {
    using K = unsigned int;
    static __device__ float lowest() { return -FLT_MAX; }
    // order-preserving u32; -0 is keyed as +0 so the two tie as they compare
    static __device__ K enc(float v) {
        const uint32_t b = __float_as_uint(v == 0.f ? 0.f : v);
        return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    }
    static __device__ float dec(K k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }
    static __device__ void amax(K* a, K k) { atomicMax(a, k); }
};
template <> struct MaxKey<int32_t> {
    using K = int;
    static __device__ int32_t lowest() { return INT32_MIN; }
    static __device__ K enc(int32_t v) { return v; }
    static __device__ int32_t dec(K k) { return k; }
    static __device__ void amax(K* a, K k) { atomicMax(a, k); }
};
template <> struct MaxKey<int64_t> {
    using K = long long;
    static __device__ int64_t lowest() { return INT64_MIN; }
    static __device__ K enc(int64_t v) { return v; }
    static __device__ int64_t dec(K k) { return k; }
    static __device__ void amax(K* a, K k) { atomicMax(a, k); }
};

template <typename T>
__global__ void __launch_bounds__(TPB) k_max_init(Geo g, uint32_t n, const T* out, int has_out, int64_t L,
                                                  typename MaxKey<T>::K* keys, int64_t* arg) {
    const uint32_t t = blockIdx.x * TPB + threadIdx.x;
    if (t >= n) return;
    int64_t off[NS];
    geo_decode(g, t, off);
    keys[off[S_AUX]] = MaxKey<T>::enc(has_out ? out[off[S_OUT]] : MaxKey<T>::lowest());
    arg[off[S_AUX]] = L;
}

// ARG = false: value pass (atomicMax of the keys); ARG = true: argmax pass (smallest position holding the maximum)
template <typename T, bool ARG>
__global__ void __launch_bounds__(TPB) k_max_pass(Geo g, uint32_t n, const T* __restrict__ src,
                                                  const int64_t* __restrict__ index, int64_t dim_size, const T* out,
                                                  int has_out, typename MaxKey<T>::K* keys, int64_t* arg) {
    const uint32_t t = blockIdx.x * TPB + threadIdx.x;
    if (t >= n) return;
    int64_t off[NS];
    const uint32_t p = geo_decode(g, t, off);
    const int64_t j = index[off[S_IDX]];
    if (j < 0 || j >= dim_size) return;
    const T v = src[off[S_SRC]];
    const T init = has_out ? out[off[S_OUT] + j * g.dst[S_OUT]] : MaxKey<T>::lowest();
    if (!(v > init)) return;                             // strictly greater: NaN and ties with the initial value lose
    const int64_t a = off[S_AUX] + j * g.dst[S_AUX];
    if (!ARG) MaxKey<T>::amax(keys + a, MaxKey<T>::enc(v));
    else if (v == MaxKey<T>::dec(keys[a])) atomicMin((long long*)arg + a, (long long)p);
}

template <typename T>
__global__ void __launch_bounds__(TPB) k_max_final(Geo g, uint32_t n, const T* __restrict__ src, T* out, int has_out,
                                                   int64_t L, const int64_t* __restrict__ arg) {
    const uint32_t t = blockIdx.x * TPB + threadIdx.x;
    if (t >= n) return;
    int64_t off[NS];
    geo_decode(g, t, off);
    const int64_t a = arg[off[S_AUX]];
    if (a < L) out[off[S_OUT]] = src[off[S_SRC] + a * g.dst[S_SRC]];     // the winner's own bits (-0 stays -0)
    else if (!has_out) out[off[S_OUT]] = 0;
}

// ---- backward: gathers, no atomics --------------------------------------------------------------------------------
template <int OP>
__global__ void __launch_bounds__(TPB) k_bwd(Geo g, uint32_t n, const int64_t* __restrict__ index, int64_t dim_size,
                                             const float* __restrict__ go, const int64_t* __restrict__ arg,
                                             const uint32_t* __restrict__ counts, float* __restrict__ gs) {
    const uint32_t t = blockIdx.x * TPB + threadIdx.x;
    if (t >= n) return;
    int64_t off[NS];
    const uint32_t p = geo_decode(g, t, off);
    int64_t j = index[off[S_IDX]];
    j = min(max(j, (int64_t)0), dim_size - 1);
    const float v = go[off[S_OUT] + j * g.dst[S_OUT]];
    float r;
    if (OP == GS_B200_SCATTER_SUM) r = v;
    else if (OP == GS_B200_SCATTER_MEAN) r = v / (float)max(counts[off[S_ROW] * dim_size + j], 1u);
    else r = arg[off[S_AUX] + j * g.dst[S_AUX]] == (int64_t)p ? v : 0.f;
    gs[off[S_GS]] = r;
}

__global__ void __launch_bounds__(TPB) k_bwd_out_mean(Geo g, uint32_t n, int64_t dim_size, const float* __restrict__ go,
                                                      const uint32_t* __restrict__ counts, float* __restrict__ gout) {
    const uint32_t t = blockIdx.x * TPB + threadIdx.x;
    if (t >= n) return;
    int64_t off[NS];
    const uint32_t j = geo_decode(g, t, off);
    gout[off[S_AUX]] = go[off[S_OUT]] / (float)max(counts[off[S_ROW] * dim_size + j], 1u);
}

// ---- host side -----------------------------------------------------------------------------------------------------
struct Shape {
    int nd, dim;
    int64_t size[GMAX];
    int64_t L, dim_size;
    int64_t rows, cols;          // index rows, broadcast columns
    bool isrow[GMAX];
    int64_t rowst[GMAX];         // row-major stride of a row dimension among the row dimensions
    int64_t src_numel, out_numel, idx_numel;
};

inline bool trivial(const Shape& sh, int d) { return d != sh.dim && sh.size[d] <= 1; }

int make_shape(const char* fn, int ndim, const int64_t* shape, int dim, const int64_t* istr, int64_t dim_size, Shape& sh) {
    if (ndim < 1 || ndim > GMAX) { gs_set_error("%s: %d dimensions (1..%d supported)", fn, ndim, GMAX); return 1; }
    if (!shape || !istr) { gs_set_error("%s: NULL shape / index strides", fn); return 1; }
    if (dim < 0 || dim >= ndim) { gs_set_error("%s: dim %d out of range for %d dimensions", fn, dim, ndim); return 1; }
    if (dim_size < 0) { gs_set_error("%s: negative dim_size %lld", fn, (long long)dim_size); return 1; }
    sh.nd = ndim; sh.dim = dim; sh.dim_size = dim_size;
    sh.rows = 1; sh.cols = 1;
    double src_n = 1, out_n = 1;
    for (int d = 0; d < ndim; d++) {
        if (shape[d] < 0) { gs_set_error("%s: negative size %lld", fn, (long long)shape[d]); return 1; }
        sh.size[d] = shape[d];
        src_n *= (double)shape[d];
        out_n *= (double)(d == dim ? dim_size : shape[d]);
    }
    // every kernel decodes 32-bit element ids; the sort holds fewer than 2^30 pairs
    if (src_n >= 2147483648.0 || out_n >= 2147483648.0) {
        gs_set_error("%s: %.0f source / %.0f output elements: fewer than 2^31 of each are supported", fn, src_n, out_n);
        return 1;
    }
    sh.src_numel = (int64_t)src_n; sh.out_numel = (int64_t)out_n;
    sh.L = shape[dim];
    for (int d = ndim - 1; d >= 0; d--) {
        sh.isrow[d] = !trivial(sh, d) && d != dim && istr[d] != 0;
        sh.rowst[d] = 0;
        if (sh.isrow[d]) { sh.rowst[d] = sh.rows; sh.rows *= sh.size[d]; }
        else if (d != dim && !trivial(sh, d)) sh.cols *= sh.size[d];
    }
    sh.idx_numel = sh.src_numel ? sh.rows * sh.L : 0;       // a size-0 dimension empties the index
    return 0;
}

inline void geo_add(Geo& g, int64_t size, const int64_t (&st)[NS]) {
    g.size[g.nd] = (uint32_t)size;
    for (int s = 0; s < NS; s++) g.st[g.nd][s] = st[s];
    g.nd++;
}

// index elements: row dimensions, then the scatter dimension (innermost), so thread id = row * L + position
Geo geo_index(const Shape& sh, const int64_t* istr) {
    Geo g = {}; g.pd = -1;
    for (int d = 0; d < sh.nd; d++)
        if (sh.isrow[d]) { int64_t st[NS] = {0, istr[d], 0, 0, 0, sh.rowst[d]}; geo_add(g, sh.size[d], st); }
    g.pd = g.nd;
    int64_t st[NS] = {0, istr[sh.dim], 0, 0, 0, 0};
    geo_add(g, sh.L, st);
    return g;
}

inline void contiguous(const Shape& sh, bool out_shape, int64_t* c) {
    int64_t run = 1;
    for (int d = sh.nd - 1; d >= 0; d--) { c[d] = run; run *= (d == sh.dim && out_shape) ? sh.dim_size : sh.size[d]; }
}

// source elements; src_order: dimensions by descending src stride (coalesced src reads), else logical order
Geo geo_src(const Shape& sh, const int64_t* sstr, const int64_t* istr, const int64_t* ostr, bool src_order) {
    int64_t aux[GMAX], gsc[GMAX];
    contiguous(sh, true, aux);
    contiguous(sh, false, gsc);
    int order[GMAX];
    for (int d = 0; d < sh.nd; d++) order[d] = d;
    if (src_order)
        std::stable_sort(order, order + sh.nd, [&](int a, int b) { return std::llabs(sstr[a]) > std::llabs(sstr[b]); });
    Geo g = {}; g.pd = -1;
    for (int k = 0; k < sh.nd; k++) {
        const int d = order[k];
        if (trivial(sh, d)) continue;
        const bool sd = d == sh.dim;
        if (sd) g.pd = g.nd;
        int64_t st[NS] = {sstr ? sstr[d] : 0, istr[d], sd ? 0 : ostr[d], sd ? 0 : aux[d], gsc[d], sh.rowst[d]};
        geo_add(g, sh.size[d], st);
    }
    g.dst[S_SRC] = sstr ? sstr[sh.dim] : 0; g.dst[S_OUT] = ostr[sh.dim]; g.dst[S_AUX] = aux[sh.dim];
    return g;
}

// output elements in logical order; the scatter dimension (size dim_size) is the slot
Geo geo_out(const Shape& sh, const int64_t* sstr, const int64_t* ostr) {
    int64_t aux[GMAX];
    contiguous(sh, true, aux);
    Geo g = {}; g.pd = -1;
    for (int d = 0; d < sh.nd; d++) {
        if (trivial(sh, d)) continue;
        const bool sd = d == sh.dim;
        if (sd) g.pd = g.nd;
        int64_t st[NS] = {sd || !sstr ? 0 : sstr[d], 0, ostr[d], aux[d], 0, sh.rowst[d]};
        geo_add(g, sd ? sh.dim_size : sh.size[d], st);
    }
    g.dst[S_SRC] = sstr ? sstr[sh.dim] : 0;
    return g;
}

// the fold: row dimensions, the slot, then the broadcast columns (innermost, so a warp reads along them)
Geo geo_fold(const Shape& sh, const int64_t* sstr, const int64_t* ostr) {
    Geo g = {}; g.pd = -1;
    for (int d = 0; d < sh.nd; d++)
        if (sh.isrow[d]) { int64_t st[NS] = {sstr[d], 0, ostr[d], 0, 0, sh.rowst[d]}; geo_add(g, sh.size[d], st); }
    g.pd = g.nd;
    { int64_t st[NS] = {0, 0, ostr[sh.dim], 0, 0, 0}; geo_add(g, sh.dim_size, st); }
    for (int d = 0; d < sh.nd; d++)
        if (!sh.isrow[d] && d != sh.dim && !trivial(sh, d)) { int64_t st[NS] = {sstr[d], 0, ostr[d], 0, 0, 0}; geo_add(g, sh.size[d], st); }
    g.dst[S_SRC] = sstr[sh.dim];
    return g;
}

inline size_t al(size_t b) { return (b + 255) & ~(size_t)255; }

struct FoldScratch { uint32_t *counts, *offsets, *keys, *keys_alt, *vals, *vals_alt; unsigned long long* total; void *scan, *sort; size_t bytes; };

FoldScratch fold_scratch(const Shape& sh, char* base) {
    const int64_t K = sh.rows * sh.dim_size, n = sh.idx_numel;
    FoldScratch f;
    size_t o = 0;
    auto take = [&](size_t b) { char* p = base ? base + o : nullptr; o += al(b); return p; };
    f.counts = (uint32_t*)take(K * 4);
    f.offsets = (uint32_t*)take(K * 4);
    f.total = (unsigned long long*)take(8);
    f.keys = (uint32_t*)take(n * 4); f.keys_alt = (uint32_t*)take(n * 4);
    f.vals = (uint32_t*)take(n * 4); f.vals_alt = (uint32_t*)take(n * 4);
    f.scan = take(gs_scan_scratch_bytes(K));
    f.sort = take(gs_sort_scratch_bytes(n));
    f.bytes = o;
    return f;
}

size_t max_key_bytes(int dtype) { return dtype == GS_B200_SCATTER_I64 ? 8 : 4; }

bool op_ok(const char* fn, int op, int dtype) {
    if (op < GS_B200_SCATTER_SUM || op > GS_B200_SCATTER_MAX || dtype < GS_B200_SCATTER_F32 || dtype > GS_B200_SCATTER_I64) {
        gs_set_error("%s: unknown op %d / dtype %d", fn, op, dtype); return false;
    }
    if (op == GS_B200_SCATTER_MEAN && dtype != GS_B200_SCATTER_F32) { gs_set_error("%s: mean is fp32 only", fn); return false; }
    return true;
}

template <typename T>
void launch_max(const Shape& sh, const Geo& gs, const Geo& go, const T* src, const int64_t* index, T* out, int has_out,
                int64_t* arg, void* scratch, cudaStream_t s) {
    using K = typename MaxKey<T>::K;
    K* keys = (K*)scratch;
    const uint32_t no = (uint32_t)sh.out_numel, ns = (uint32_t)sh.src_numel;
    k_max_init<T><<<nblocks(no), TPB, 0, s>>>(go, no, out, has_out, sh.L, keys, arg);
    if (ns) {
        k_max_pass<T, false><<<nblocks(ns), TPB, 0, s>>>(gs, ns, src, index, sh.dim_size, out, has_out, keys, arg);
        k_max_pass<T, true><<<nblocks(ns), TPB, 0, s>>>(gs, ns, src, index, sh.dim_size, out, has_out, keys, arg);
    }
    k_max_final<T><<<nblocks(no), TPB, 0, s>>>(go, no, src, out, has_out, sh.L, arg);
    gs_count_launches(ns ? 4 : 2);
}

template <typename T>
void launch_isum(const Shape& sh, const Geo& gs, const Geo& go, const T* src, const int64_t* index, T* out, int has_out,
                 cudaStream_t s) {
    const uint32_t no = (uint32_t)sh.out_numel, ns = (uint32_t)sh.src_numel;
    if (!has_out) { k_fill_zero<T><<<nblocks(no), TPB, 0, s>>>(go, no, out); gs_count_launches(1); }
    if (ns) { k_isum<T><<<nblocks(ns), TPB, 0, s>>>(gs, ns, src, index, sh.dim_size, out); gs_count_launches(1); }
}

}  // namespace

int32_t gs_b200_scatter_index_range(int32_t ndim, const int64_t* shape_host, int32_t dim, const int64_t* index,
                                    const int64_t* index_strides_host, int64_t* range_out, void* stream) {
    Shape sh;
    if (make_shape("scatter_index_range", ndim, shape_host, dim, index_strides_host, 0, sh)) return 1;
    if (!range_out || (sh.idx_numel && !index)) { gs_set_error("scatter_index_range: NULL pointer"); return 1; }
    cudaStream_t s = (cudaStream_t)stream;
    k_range_init<<<1, 1, 0, s>>>(range_out);
    const uint32_t n = (uint32_t)sh.idx_numel;
    if (n) {
        const Geo g = geo_index(sh, index_strides_host);
        k_range<<<std::min(nblocks(n), (unsigned)GS_NUM_SMS * 8), TPB, 0, s>>>(g, n, index, range_out);
    }
    gs_count_launches(n ? 2 : 1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

size_t gs_b200_scatter_scratch_bytes(int32_t op, int32_t dtype, int32_t ndim, const int64_t* shape_host, int32_t dim,
                                     const int64_t* index_strides_host, int64_t dim_size) {
    Shape sh;
    if (!op_ok("scatter_scratch_bytes", op, dtype)) return 0;
    if (make_shape("scatter_scratch_bytes", ndim, shape_host, dim, index_strides_host, dim_size, sh)) return 0;
    if (op == GS_B200_SCATTER_MAX) return al(max_key_bytes(dtype) * (size_t)sh.out_numel) + 256;
    if (dtype != GS_B200_SCATTER_F32) return 256;
    return fold_scratch(sh, nullptr).bytes + 256;
}

int32_t gs_b200_scatter_forward(int32_t op, int32_t dtype, int32_t ndim, const int64_t* shape_host, int32_t dim,
                                int64_t dim_size, const void* src, const int64_t* src_strides_host, const int64_t* index,
                                const int64_t* index_strides_host, void* out, const int64_t* out_strides_host,
                                int32_t has_out, int64_t* argmax, void* scratch, void* stream) {
    static const char* fn = "scatter_forward";
    Shape sh;
    if (!op_ok(fn, op, dtype)) return 1;
    if (make_shape(fn, ndim, shape_host, dim, index_strides_host, dim_size, sh)) return 1;
    if (!src_strides_host || !out_strides_host) { gs_set_error("%s: NULL strides", fn); return 1; }
    if (sh.L > 0 && sh.dim_size == 0 && sh.src_numel > 0) { gs_set_error("%s: dim_size 0 with a non-empty index", fn); return 1; }
    if ((sh.src_numel && (!src || !index)) || (sh.out_numel && (!out || !scratch)) ||
        (op == GS_B200_SCATTER_MAX && sh.out_numel && !argmax)) {
        gs_set_error("%s: NULL pointer", fn); return 1;
    }
    if (sh.out_numel == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    char* scr = (char*)(((uintptr_t)scratch + 255) & ~(uintptr_t)255);
    const Geo gs = geo_src(sh, src_strides_host, index_strides_host, out_strides_host, true);
    const Geo go = geo_out(sh, src_strides_host, out_strides_host);
    if (op == GS_B200_SCATTER_MAX) {
        if (dtype == GS_B200_SCATTER_F32) launch_max<float>(sh, gs, go, (const float*)src, index, (float*)out, has_out, argmax, scr, s);
        else if (dtype == GS_B200_SCATTER_I32) launch_max<int32_t>(sh, gs, go, (const int32_t*)src, index, (int32_t*)out, has_out, argmax, scr, s);
        else launch_max<int64_t>(sh, gs, go, (const int64_t*)src, index, (int64_t*)out, has_out, argmax, scr, s);
    } else if (dtype == GS_B200_SCATTER_I32) {
        launch_isum<int32_t>(sh, gs, go, (const int32_t*)src, index, (int32_t*)out, has_out, s);
    } else if (dtype == GS_B200_SCATTER_I64) {
        launch_isum<int64_t>(sh, gs, go, (const int64_t*)src, index, (int64_t*)out, has_out, s);
    } else {
        const int64_t K = sh.rows * sh.dim_size, n = sh.idx_numel;
        if (n >= (1ll << 30)) { gs_set_error("%s: %lld index elements: fewer than 2^30 are supported", fn, (long long)n); return 1; }
        const FoldScratch f = fold_scratch(sh, scr);
        GS_CUDA_CHECK(cudaMemsetAsync(f.counts, 0, (size_t)K * 4, s));
        if (n) {
            k_keys<<<nblocks(n), TPB, 0, s>>>(geo_index(sh, index_strides_host), (uint32_t)n, index, sh.dim_size, f.keys,
                                              f.vals, f.counts);
            gs_count_launches(1);
        }
        if (gs_scan_gather_u32(f.counts, nullptr, f.offsets, f.total, K, f.scan, s)) return 1;
        int bits = 0;
        while (bits < 32 && (1ll << bits) < K) bits++;
        int in_alt = 0;
        if (n && gs_sort_pairs_u32(f.keys, f.keys_alt, f.vals, f.vals_alt, n, 0, bits, f.sort, &in_alt, s)) return 1;
        const Geo gf = geo_fold(sh, src_strides_host, out_strides_host);
        const uint32_t no = (uint32_t)sh.out_numel;
        const uint32_t* pos = in_alt ? f.vals_alt : f.vals;
        if (op == GS_B200_SCATTER_MEAN)
            k_fold<true><<<nblocks(no), TPB, 0, s>>>(gf, no, sh.dim_size, (const float*)src, (float*)out, has_out, pos, f.offsets, f.counts);
        else
            k_fold<false><<<nblocks(no), TPB, 0, s>>>(gf, no, sh.dim_size, (const float*)src, (float*)out, has_out, pos, f.offsets, f.counts);
        gs_count_launches(1);
    }
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int32_t gs_b200_scatter_backward(int32_t op, int32_t ndim, const int64_t* shape_host, int32_t dim, int64_t dim_size,
                                 const int64_t* index, const int64_t* index_strides_host, const float* grad_out,
                                 const int64_t* grad_out_strides_host, const int64_t* argmax, const void* fwd_scratch,
                                 float* grad_src, float* grad_out_mean, void* stream) {
    static const char* fn = "scatter_backward";
    Shape sh;
    if (!op_ok(fn, op, GS_B200_SCATTER_F32)) return 1;
    if (make_shape(fn, ndim, shape_host, dim, index_strides_host, dim_size, sh)) return 1;
    if (!grad_out_strides_host) { gs_set_error("%s: NULL strides", fn); return 1; }
    const uint32_t* counts = (const uint32_t*)(((uintptr_t)fwd_scratch + 255) & ~(uintptr_t)255);
    if ((sh.out_numel && !grad_out) || (sh.src_numel && (!index || !grad_src)) ||
        (op == GS_B200_SCATTER_MAX && sh.out_numel && !argmax) ||
        (op == GS_B200_SCATTER_MEAN && sh.out_numel && !fwd_scratch)) {
        gs_set_error("%s: NULL pointer", fn); return 1;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t ns = (uint32_t)sh.src_numel, no = (uint32_t)sh.out_numel;
    if (ns && no) {
        const Geo g = geo_src(sh, nullptr, index_strides_host, grad_out_strides_host, false);
        if (op == GS_B200_SCATTER_SUM) k_bwd<GS_B200_SCATTER_SUM><<<nblocks(ns), TPB, 0, s>>>(g, ns, index, sh.dim_size, grad_out, argmax, counts, grad_src);
        else if (op == GS_B200_SCATTER_MEAN) k_bwd<GS_B200_SCATTER_MEAN><<<nblocks(ns), TPB, 0, s>>>(g, ns, index, sh.dim_size, grad_out, argmax, counts, grad_src);
        else k_bwd<GS_B200_SCATTER_MAX><<<nblocks(ns), TPB, 0, s>>>(g, ns, index, sh.dim_size, grad_out, argmax, counts, grad_src);
        gs_count_launches(1);
    } else if (ns) {
        GS_CUDA_CHECK(cudaMemsetAsync(grad_src, 0, (size_t)ns * 4, s));
    }
    if (op == GS_B200_SCATTER_MEAN && grad_out_mean && no) {
        k_bwd_out_mean<<<nblocks(no), TPB, 0, s>>>(geo_out(sh, nullptr, grad_out_strides_host), no, sh.dim_size, grad_out,
                                                     counts, grad_out_mean);
        gs_count_launches(1);
    }
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
