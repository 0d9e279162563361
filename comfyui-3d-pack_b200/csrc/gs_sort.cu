// CUB-free onesweep LSD radix sort (u32 key, u32 value) + gather-scan.
//
// Replaces cub::DeviceRadixSort::SortPairs and cub::DeviceScan::InclusiveSum in
// the binning stage of diff_gaussian_rasterization (SURVEY.md §2.4, App. A.1.5).
//
// Onesweep (Adinets & Merrill 2022): ONE upfront histogram kernel for all digit
// positions, then one kernel per 8-bit digit in which every CTA takes a
// partition by atomic ticket, ranks its keys, publishes its per-digit counts and
// resolves its global offsets with a decoupled look-back over earlier
// partitions — so each pass reads and writes every pair exactly once
// (16 B/pair/pass + 4 B/pair for the histogram).
//
// The sort is STABLE (ties keep input order), which the tile/depth/index
// ordering contract of the rasterizer relies on.
#include "../../include/gs_b200.h"
#include "gs_common.cuh"

#include <algorithm>

namespace {

constexpr int RS_THREADS = 512;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr int RS_ITEMS = 8;
constexpr int RS_PART = RS_THREADS * RS_ITEMS;   // 4096 pairs per partition
constexpr int RS_RADIX = 256;
constexpr int RS_MAX_PASSES = 4;
constexpr uint32_t FLAG_AGG = 1u << 30, FLAG_PFX = 2u << 30, VAL_MASK = (1u << 30) - 1;
static_assert(GS_MAX_SEG_KEYS <= (int64_t)VAL_MASK, "a segment's digit counts must fit the status word");

// ---- segments -----------------------------------------------------------------
// The keys are sorted as nseg independent segments [off[i], off[i+1]) of one array (the multi-view step sorts
// every view of a chunk in one launch per digit pass).  Each segment has its own digit histograms, trivial flags
// and look-back chain; partitions never straddle two segments.  part0[i] = index of segment i's first partition.
struct SegParts {
    int n;
    int64_t off[GS_MAX_SEGS + 1];
    uint32_t part0[GS_MAX_SEGS + 1];
};

// ---- upfront histogram of every digit position -------------------------------
// key_bias (may be NULL): per-segment device words (segment i at key_bias[i * bias_stride]) subtracted from every
// key before digits are taken.  The depth sort passes each view's minimum visible depth key, so that the high
// digit(s) of (key - min) are all zero whenever the depth range spans < 2^24 float steps; such a pass is detected
// from the histogram (one bin holds all of the segment's keys) and degenerates to a straight copy instead of the
// rank/look-back/scatter chain.  grid = (blocks per segment, segments); ghist is [segment][RS_MAX_PASSES][256].
__global__ void __launch_bounds__(RS_THREADS)
rs_histogram(const uint32_t* __restrict__ keys, const __grid_constant__ SegParts sp, uint32_t* __restrict__ ghist,
             int begin_bit, int npasses, const uint32_t* __restrict__ key_bias, int bias_stride) {
    __shared__ uint32_t sh[RS_MAX_PASSES][RS_RADIX];
    for (int i = threadIdx.x; i < RS_MAX_PASSES * RS_RADIX; i += RS_THREADS) (&sh[0][0])[i] = 0;
    __syncthreads();
    const int seg = blockIdx.y;
    const int64_t n = sp.off[seg + 1] - sp.off[seg];
    keys += sp.off[seg];
    const int64_t stride = (int64_t)gridDim.x * RS_THREADS;
    const uint32_t bias = key_bias ? __ldg(key_bias + (size_t)seg * bias_stride) : 0u;
    for (int64_t i0 = (int64_t)blockIdx.x * RS_THREADS; i0 < n; i0 += stride) {   // block-uniform trip count
        const int64_t i = i0 + threadIdx.x;
        const bool ok = i < n;
        const uint32_t k = ok ? (__ldg(keys + i) - bias) : 0u;
        const uint32_t okmask = __ballot_sync(0xFFFFFFFFu, ok);
        for (int p = 0; p < npasses; p++) {
            // clustered digits (high bits of depths / of tile ids) would serialise 32-way on one shared-memory
            // bin: when the whole warp agrees, one lane adds the count; otherwise plain shared atomics.
            const uint32_t d = (k >> (begin_bit + 8 * p)) & 0xFF;
            const uint32_t d0 = __shfl_sync(0xFFFFFFFFu, d, __ffs(okmask) - 1);
            if (__all_sync(0xFFFFFFFFu, !ok || d == d0)) {
                if ((threadIdx.x & 31) == 0 && okmask) atomicAdd(&sh[p][d0], __popc(okmask));
            } else if (ok) {
                atomicAdd(&sh[p][d], 1u);
            }
        }
    }
    __syncthreads();
    uint32_t* gh = ghist + (size_t)seg * RS_MAX_PASSES * RS_RADIX;
    for (int i = threadIdx.x; i < npasses * RS_RADIX; i += RS_THREADS) {
        const uint32_t c = (&sh[0][0])[i];
        if (c) atomicAdd(gh + i, c);
    }
}

// exclusive scan of each (segment, pass)'s 256 bins, in place; grid = (passes, segments).
// trivial[segment][pass] = 1 when one bin holds all of the segment's keys.
__global__ void __launch_bounds__(RS_RADIX) rs_scan_hist(uint32_t* __restrict__ ghist, uint32_t* __restrict__ trivial,
                                                         const __grid_constant__ SegParts sp) {
    __shared__ uint32_t s[RS_RADIX];
    const int seg = blockIdx.y, p = blockIdx.x;
    const uint32_t n = (uint32_t)(sp.off[seg + 1] - sp.off[seg]);
    uint32_t* h = ghist + ((size_t)seg * RS_MAX_PASSES + p) * RS_RADIX;
    uint32_t* triv = trivial + seg * RS_MAX_PASSES + p;
    const int t = threadIdx.x;
    const uint32_t v = h[t];
    if (t == 0) *triv = 0;
    __syncthreads();
    if (v == n) *triv = 1;
    s[t] = v;
    __syncthreads();
    for (int off = 1; off < RS_RADIX; off <<= 1) {
        uint32_t a = (t >= off) ? s[t - off] : 0;
        __syncthreads();
        s[t] += a;
        __syncthreads();
    }
    h[t] = s[t] - v;
}

__device__ __forceinline__ uint32_t ld_relaxed(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ---- one digit pass -------------------------------------------------------------
// 512 threads x 8 items: the stable in-warp ranking is a dependent chain of (match, LDS, STS) rounds, so the
// chain is kept short (8) and the CTA wide (16 warps) to have enough warps in flight to hide its latency.
template <bool HAS_VALS>
__global__ void __launch_bounds__(RS_THREADS, 3)
rs_onesweep(const uint32_t* __restrict__ keys_in, uint32_t* __restrict__ keys_out,
            const uint32_t* __restrict__ vals_in, uint32_t* __restrict__ vals_out, const __grid_constant__ SegParts sp,
            int pass, int shift, const uint32_t* __restrict__ ghist_excl, uint32_t* __restrict__ status,
            uint32_t* __restrict__ ticket, const uint32_t* __restrict__ key_bias, int bias_stride,
            const uint32_t* __restrict__ trivial) {
    __shared__ uint32_t s_keys[RS_PART];
    __shared__ uint32_t s_vals[HAS_VALS ? RS_PART : 1];
    __shared__ uint16_t s_whist[RS_WARPS][RS_RADIX];   // counts <= 256 per (warp,digit), offsets <= 4096
    __shared__ uint32_t s_start[RS_RADIX];     // block-local exclusive start of each digit
    __shared__ int64_t s_gbase[RS_RADIX];      // global position of block-sorted slot 0 of each digit, minus s_start
    __shared__ uint32_t s_wtot[RS_RADIX / 32];
    // this CTA's (segment, partition, valid keys, key bias), re-read from shared memory where they are needed so
    // that they hold no registers across the ranking (the pass runs at 40 registers)
    __shared__ uint32_t s_seg, s_part, s_valid, s_bias;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        // the ticket orders the partitions of every segment: a partition's predecessors were all handed out before it
        const uint32_t gpart = atomicAdd(ticket, 1u);
        int seg = 0;
        while (seg + 1 < sp.n && gpart >= sp.part0[seg + 1]) seg++;     // (segments without keys have no partitions)
        const uint32_t part = gpart - sp.part0[seg];
        s_seg = seg; s_part = part;
        s_valid = (uint32_t)min((int64_t)RS_PART, sp.off[seg + 1] - sp.off[seg] - (int64_t)part * RS_PART);
        s_bias = key_bias ? __ldg(key_bias + (size_t)seg * bias_stride) : 0u;
    }
    for (int i = tid; i < RS_WARPS * RS_RADIX / 2; i += RS_THREADS) reinterpret_cast<uint32_t*>(&s_whist[0][0])[i] = 0;
    __syncthreads();
    const int64_t base = sp.off[s_seg] + (int64_t)s_part * RS_PART;
    if (__ldg(trivial + s_seg * RS_MAX_PASSES + pass)) {
        // every key of the segment has the same digit here: the stable pass is the identity permutation
        const int valid = (int)s_valid;
#pragma unroll 4
        for (int i = tid; i < RS_PART; i += RS_THREADS) {
            if (i < valid) { keys_out[base + i] = __ldg(keys_in + base + i); if (HAS_VALS) vals_out[base + i] = __ldg(vals_in + base + i); }
        }
        return;
    }

    // warp-striped load: warp w owns [w*256, (w+1)*256) of the partition, item i lane l -> +i*32+l
    // The values wait in s_keys at their input slots until the scatter: in registers they would not fit the pass's
    // 40 registers (the ranks are kept two per register for the same reason).
    uint32_t k[RS_ITEMS];
    uint32_t rank2[RS_ITEMS / 2];     // in-warp ranks (< 4096)
    const int wbase = warp * (RS_ITEMS * 32) + lane;
#pragma unroll
    for (int i = 0; i < RS_ITEMS; i++) {
        const int loc = wbase + i * 32;
        if (loc < (int)s_valid) {
            k[i] = __ldg(keys_in + base + loc) - s_bias;
            if (HAS_VALS) s_keys[loc] = __ldg(vals_in + base + loc);
        } else {
            k[i] = 0xFFFFFFFFu;   // padding: highest digit, highest index -> lands past `valid`
            if (HAS_VALS) s_keys[loc] = 0;
        }
    }
    // stable rank inside the warp, digit by digit
    const uint32_t lt_mask = (1u << lane) - 1;
#pragma unroll
    for (int i = 0; i < RS_ITEMS; i++) {
        const uint32_t d = (k[i] >> shift) & 0xFF;
        // lanes holding the same digit.  NOT match.any: MATCH is a slow, shared-unit warp instruction, while
        // 8 VOTE + 8 LOP3 issue at full rate.
        uint32_t peers = 0xFFFFFFFFu;
#pragma unroll
        for (int b = 0; b < 8; b++) {
            const bool bit = (d >> b) & 1u;
            const uint32_t bal = __ballot_sync(0xFFFFFFFFu, bit);
            peers &= bit ? bal : ~bal;
        }
        const uint32_t prev = s_whist[warp][d];
        __syncwarp();
        const uint32_t r = __popc(peers & lt_mask);
        if (r == 0) s_whist[warp][d] = (uint16_t)(prev + __popc(peers));
        __syncwarp();
        const uint32_t rk = prev + r;
        if (i & 1) rank2[i >> 1] |= rk << 16; else rank2[i >> 1] = rk;
    }
    __syncthreads();

    // threads 0..255 own one digit each: exclusive scan over warps, publish, scan over digits, look-back
    uint32_t count = 0, pub = 0;
    const uint32_t part = s_part;
    status += (size_t)sp.part0[s_seg] * RS_RADIX;      // this segment's look-back chain
    uint32_t* my_status = status + (size_t)part * RS_RADIX + tid;
    if (tid < RS_RADIX) {
        uint32_t sum = 0;
#pragma unroll
        for (int w = 0; w < RS_WARPS; w++) {
            const uint32_t c = s_whist[w][tid];
            s_whist[w][tid] = (uint16_t)sum;
            sum += c;
        }
        count = sum;
        const uint32_t pad = (uint32_t)RS_PART - s_valid;
        pub = (tid == RS_RADIX - 1) ? count - pad : count;      // padding is all digit 255
        st_relaxed(my_status, (part == 0 ? FLAG_PFX : FLAG_AGG) | pub);
        // exclusive scan over the 256 digits: shuffle scan per warp + 8 warp totals
        uint32_t inc = count;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) s_wtot[warp] = inc;
        count = inc - count;                                     // warp-local exclusive
    }
    __syncthreads();
    if (tid < RS_RADIX) {
        uint32_t woff = 0;
#pragma unroll
        for (int w = 0; w < RS_RADIX / 32; w++) woff += (w < warp) ? s_wtot[w] : 0u;
        const uint32_t start = woff + count;
        s_start[tid] = start;
        // decoupled look-back over earlier partitions, 4 status words in flight per step (the walk is a chain
        // of dependent L2 round trips; prefetching the next predecessors cuts its latency ~4x)
        uint32_t excl = 0;
        if (part > 0) {
            int64_t p = (int64_t)part - 1;
            bool done = false;
            while (!done) {
                uint32_t sv[4];
#pragma unroll
                for (int i = 0; i < 4; i++)
                    sv[i] = (p - i >= 0) ? ld_relaxed(status + (size_t)(p - i) * RS_RADIX + tid) : FLAG_PFX;
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    if (done) break;
                    uint32_t x = sv[i];
                    while ((x & ~VAL_MASK) == 0) x = ld_relaxed(status + (size_t)(p - i) * RS_RADIX + tid);
                    excl += x & VAL_MASK;
                    if ((x & ~VAL_MASK) == FLAG_PFX) done = true;
                }
                p -= 4;
            }
            st_relaxed(my_status, FLAG_PFX | ((excl + pub) & VAL_MASK));
        }
        const uint32_t g0 = ghist_excl[((size_t)s_seg * RS_MAX_PASSES + pass) * RS_RADIX + tid];
        s_gbase[tid] = sp.off[s_seg] + (int64_t)g0 + (int64_t)excl - (int64_t)start;
    }
    __syncthreads();

    // scatter into block-sorted order in shared memory
    uint32_t v[RS_ITEMS];
    if (HAS_VALS) {
#pragma unroll
        for (int i = 0; i < RS_ITEMS; i++) v[i] = s_keys[wbase + i * 32];
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < RS_ITEMS; i++) {
        const uint32_t d = (k[i] >> shift) & 0xFF;
        const uint32_t pos = s_start[d] + s_whist[warp][d] + ((rank2[i >> 1] >> (16 * (i & 1))) & 0xFFFFu);
        s_keys[pos] = k[i];
        if (HAS_VALS) s_vals[pos] = v[i];
    }
    __syncthreads();
    // coalesced write-out: consecutive slots of one digit are consecutive in global memory
    const int valid = (int)s_valid;
    const uint32_t bias = s_bias;
#pragma unroll
    for (int j = 0; j < RS_ITEMS; j++) {
        const int pos = j * RS_THREADS + tid;
        if (pos < valid) {
            const uint32_t key = s_keys[pos];
            const int64_t g = s_gbase[(key >> shift) & 0xFF] + pos;
            keys_out[g] = key + bias;
            if (HAS_VALS) vals_out[g] = s_vals[pos];
        }
    }
}

// ---- gather + exclusive scan ------------------------------------------------
constexpr int SC_THREADS = 256;
constexpr int SC_ITEMS = 8;
constexpr int SC_TILE = SC_THREADS * SC_ITEMS;

__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* s_warp, uint32_t& block_total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xFFFFFFFFu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = (lane < SC_THREADS / 32) ? s_warp[lane] : 0;
        uint32_t winc = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t t = __shfl_up_sync(0xFFFFFFFFu, winc, o);
            if (lane >= o) winc += t;
        }
        if (lane < SC_THREADS / 32) s_warp[lane] = winc - w;
        if (lane == SC_THREADS / 32 - 1) s_warp[SC_THREADS / 32] = winc;
    }
    __syncthreads();
    block_total = s_warp[SC_THREADS / 32];
    const uint32_t r = s_warp[warp] + inc - v;
    __syncthreads();
    return r;
}

// Gather-scan of nseg segments of n elements each, back to back (grid.y = segment; ids are indices inside the
// segment).  block_sums is [segment][gridDim.x], total [segment].
__global__ void __launch_bounds__(SC_THREADS)
scan_reduce(const uint32_t* __restrict__ tiles, const uint32_t* __restrict__ ids, int64_t n,
            unsigned long long* __restrict__ block_sums) {
    __shared__ unsigned long long s_red[SC_THREADS / 32];
    tiles += (int64_t)blockIdx.y * n;
    if (ids) ids += (int64_t)blockIdx.y * n;
    block_sums += (size_t)blockIdx.y * gridDim.x;
    const int64_t base = (int64_t)blockIdx.x * SC_TILE;
    unsigned long long sum = 0;
#pragma unroll
    for (int i = 0; i < SC_ITEMS; i++) {
        const int64_t j = base + i * SC_THREADS + threadIdx.x;
        if (j < n) sum += tiles[ids ? ids[j] : j];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, o);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int w = 0; w < SC_THREADS / 32; w++) t += s_red[w];
        block_sums[blockIdx.x] = t;
    }
}

// one CTA per segment: exclusive scan of the block sums (sequential over chunks), writes the total
__global__ void __launch_bounds__(1024)
scan_block_sums(unsigned long long* __restrict__ block_sums, int nblocks, unsigned long long* __restrict__ total) {
    __shared__ unsigned long long s[1024];
    __shared__ unsigned long long carry;
    block_sums += (size_t)blockIdx.x * nblocks;
    total += blockIdx.x;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < nblocks; base += 1024) {
        const int i = base + threadIdx.x;
        const unsigned long long v = (i < nblocks) ? block_sums[i] : 0;
        s[threadIdx.x] = v;
        __syncthreads();
        for (int off = 1; off < 1024; off <<= 1) {
            unsigned long long a = (threadIdx.x >= off) ? s[threadIdx.x - off] : 0;
            __syncthreads();
            s[threadIdx.x] += a;
            __syncthreads();
        }
        if (i < nblocks) block_sums[i] = carry + s[threadIdx.x] - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry += s[1023];
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}

__global__ void __launch_bounds__(SC_THREADS)
scan_apply(const uint32_t* __restrict__ tiles, const uint32_t* __restrict__ ids, int64_t n,
           const unsigned long long* __restrict__ block_sums, uint32_t* __restrict__ offsets) {
    __shared__ uint32_t s_warp[SC_THREADS / 32 + 1];
    tiles += (int64_t)blockIdx.y * n;
    if (ids) ids += (int64_t)blockIdx.y * n;
    offsets += (int64_t)blockIdx.y * n;
    block_sums += (size_t)blockIdx.y * gridDim.x;
    const int64_t base = (int64_t)blockIdx.x * SC_TILE + (int64_t)threadIdx.x * SC_ITEMS;   // blocked
    uint32_t v[SC_ITEMS];
    uint32_t tsum = 0;
#pragma unroll
    for (int i = 0; i < SC_ITEMS; i++) {
        const int64_t j = base + i;
        v[i] = (j < n) ? tiles[ids ? ids[j] : j] : 0;
        tsum += v[i];
    }
    uint32_t btotal;
    uint32_t run = block_exclusive_scan(tsum, s_warp, btotal) + (uint32_t)block_sums[blockIdx.x];
#pragma unroll
    for (int i = 0; i < SC_ITEMS; i++) {
        const int64_t j = base + i;
        if (j < n) offsets[j] = run;
        run += v[i];
    }
}

}  // namespace

// scratch layout for the sort: [ghist nseg*4*256 u32][tickets 8 u32][trivial nseg*4 u32 (+pad)][status passes*parts*256 u32]
static size_t sort_head_words(int nseg) { return (size_t)nseg * RS_MAX_PASSES * RS_RADIX + 8 + GS_MAX_SEGS * RS_MAX_PASSES + 56; }

size_t gs_sort_seg_scratch_bytes(int nseg, int64_t total_n) {
    const int64_t parts = (total_n + RS_PART - 1) / RS_PART + nseg;      // a partial partition per segment at most
    return sort_head_words(nseg) * 4 + (size_t)RS_MAX_PASSES * (size_t)parts * RS_RADIX * 4;
}
size_t gs_sort_hist_bytes(int nseg) { return (size_t)nseg * RS_MAX_PASSES * RS_RADIX * 4; }
size_t gs_sort_scratch_bytes(int64_t n) { return gs_sort_seg_scratch_bytes(1, n); }

int gs_sort_pairs_u32(uint32_t* keys, uint32_t* keys_alt, uint32_t* vals, uint32_t* vals_alt, int64_t n,
                      int begin_bit, int end_bit, void* scratch, int* result_in_alt, cudaStream_t s) {
    SortSegs sg; sg.n = 1; sg.off[0] = 0; sg.off[1] = n < 0 ? 0 : n;
    return gs_sort_pairs_segmented(keys, keys_alt, vals, vals_alt, sg, begin_bit, end_bit, scratch, result_in_alt,
                                   nullptr, 0, false, s);
}

extern "C" size_t gs_b200_sort_scratch_bytes(int64_t n) { return gs_sort_scratch_bytes(n); }

extern "C" int32_t gs_b200_sort_pairs_u32(uint32_t* keys, uint32_t* keys_alt, uint32_t* vals, uint32_t* vals_alt, int64_t n,
                                          int32_t begin_bit, int32_t end_bit, void* scratch, int32_t* result_in_alt,
                                          void* stream) {
    int r = 0;
    int rc = gs_sort_pairs_u32(keys, keys_alt, vals, vals_alt, n, begin_bit, end_bit, scratch, &r, (cudaStream_t)stream);
    if (result_in_alt) *result_in_alt = r;
    return rc;
}

int gs_sort_pairs_segmented(uint32_t* keys, uint32_t* keys_alt, uint32_t* vals, uint32_t* vals_alt, const SortSegs& segs,
                            int begin_bit, int end_bit, void* scratch, int* result_in_alt, const uint32_t* key_bias,
                            int bias_stride, bool hist_ready, cudaStream_t s) {
    *result_in_alt = 0;
    if (segs.n < 1 || segs.n > GS_MAX_SEGS) { gs_set_error("sort: %d segments (1..%d)", segs.n, GS_MAX_SEGS); return 1; }
    SegParts sp;
    sp.n = segs.n;
    int64_t parts = 0, maxlen = 0;
    for (int i = 0; i <= segs.n; i++) {
        sp.off[i] = segs.off[i];
        sp.part0[i] = (uint32_t)parts;
        if (i == segs.n) break;
        const int64_t len = segs.off[i + 1] - segs.off[i];
        if (len < 0) { gs_set_error("sort: segment %d has negative length", i); return 1; }
        if (len > GS_MAX_SEG_KEYS) { gs_set_error("sort: segment %d has %lld keys (at most %lld)", i, (long long)len, (long long)GS_MAX_SEG_KEYS); return 1; }
        maxlen = std::max(maxlen, len);
        parts += (len + RS_PART - 1) / RS_PART;
    }
    if (parts == 0 || end_bit <= begin_bit) return 0;
    if (parts >= (int64_t)UINT32_MAX) { gs_set_error("sort: too many partitions"); return 1; }
    const int npasses = (end_bit - begin_bit + 7) / 8;
    if (npasses > RS_MAX_PASSES) { gs_set_error("sort: more than 32 key bits"); return 1; }
    uint32_t* ghist = (uint32_t*)scratch;
    uint32_t* tickets = ghist + (size_t)segs.n * RS_MAX_PASSES * RS_RADIX;
    uint32_t* trivial = tickets + 8;
    uint32_t* status = (uint32_t*)scratch + sort_head_words(segs.n);
    // hist_ready: the caller has already counted the digit histograms into ghist (the emit of the tile sort does)
    char* zero_from = hist_ready ? (char*)tickets : (char*)scratch;
    GS_CUDA_CHECK(cudaMemsetAsync(zero_from, 0, (char*)(status + (size_t)npasses * parts * RS_RADIX) - zero_from, s));
    if (!hist_ready) {
        const int64_t hb = (maxlen + RS_THREADS * 8 - 1) / (RS_THREADS * 8);
        const int64_t cap = std::max(1, GS_NUM_SMS * 8 / segs.n);
        rs_histogram<<<dim3((unsigned)std::min(hb, cap), segs.n), RS_THREADS, 0, s>>>(keys, sp, ghist, begin_bit, npasses,
                                                                                     key_bias, bias_stride);
    }
    rs_scan_hist<<<dim3(npasses, segs.n), RS_RADIX, 0, s>>>(ghist, trivial, sp);
    uint32_t *kin = keys, *kout = keys_alt, *vin = vals, *vout = vals_alt;
    for (int p = 0; p < npasses; p++) {
        const int shift = begin_bit + 8 * p;
        uint32_t* st = status + (size_t)p * parts * RS_RADIX;
        if (vals)
            rs_onesweep<true><<<(unsigned)parts, RS_THREADS, 0, s>>>(kin, kout, vin, vout, sp, p, shift, ghist, st, tickets + p, key_bias, bias_stride, trivial);
        else
            rs_onesweep<false><<<(unsigned)parts, RS_THREADS, 0, s>>>(kin, kout, nullptr, nullptr, sp, p, shift, ghist, st, tickets + p, key_bias, bias_stride, trivial);
        uint32_t* t = kin; kin = kout; kout = t;
        t = vin; vin = vout; vout = t;
        *result_in_alt ^= 1;
    }
    gs_count_launches((hist_ready ? 1 : 2) + npasses);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

size_t gs_scan_seg_scratch_bytes(int64_t n, int nseg) {
    const int64_t blocks = (n + SC_TILE - 1) / SC_TILE;
    return (size_t)nseg * (blocks + 1) * sizeof(unsigned long long);
}
size_t gs_scan_scratch_bytes(int64_t n) { return gs_scan_seg_scratch_bytes(n, 1); }

int gs_scan_gather_u32(const uint32_t* tiles, const uint32_t* ids, uint32_t* offsets, unsigned long long* total,
                       int64_t n, void* scratch, cudaStream_t s) {
    return gs_scan_gather_seg_u32(tiles, ids, offsets, total, n, 1, scratch, s);
}

int gs_scan_gather_seg_u32(const uint32_t* tiles, const uint32_t* ids, uint32_t* offsets, unsigned long long* totals,
                           int64_t n, int nseg, void* scratch, cudaStream_t s) {
    if (nseg <= 0) return 0;
    if (n <= 0) { GS_CUDA_CHECK(cudaMemsetAsync(totals, 0, (size_t)nseg * sizeof(unsigned long long), s)); return 0; }
    if (nseg > 65535) { gs_set_error("scan: %d segments", nseg); return 1; }
    const int blocks = (int)((n + SC_TILE - 1) / SC_TILE);
    unsigned long long* bs = (unsigned long long*)scratch;
    scan_reduce<<<dim3(blocks, nseg), SC_THREADS, 0, s>>>(tiles, ids, n, bs);
    scan_block_sums<<<nseg, 1024, 0, s>>>(bs, blocks, totals);
    scan_apply<<<dim3(blocks, nseg), SC_THREADS, 0, s>>>(tiles, ids, n, bs, offsets);
    gs_count_launches(3);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
