// Binning stage: tile-key duplication (in depth order), per-tile ranges, and the
// debug reconstruction of the package's 64-bit keys.
//
// Replaces duplicateWithKeys / identifyTileRanges of diff_gaussian_rasterization
// (SURVEY.md App. A.1.5).  GPU-first restructuring: the package sorts K*N
// 64-bit (tile|depth) keys in one go; here the N Gaussians are depth-sorted
// FIRST (N 32-bit keys), pairs are emitted in that order, and only the tile id
// (ceil(log2(tiles)) bits) is sorted over the K*N pairs.  Both sorts are stable,
// so the resulting per-tile order (depth, then Gaussian index) and therefore
// point_list / ranges are bit-identical to the single 64-bit sort, at ~1/3 of
// its memory traffic.
#include "gs_common.cuh"

#include <algorithm>

namespace {

// Each warp takes 32 consecutive depth-sorted Gaussians.  Their output runs are back to back
// ([offsets[s0], offsets[s0+32]) is one contiguous span), so the lanes sweep that span with fully
// coalesced stores and find the owning Gaussian of each slot by binary search over the 32 offsets.
// TIGHT: the per-row tile spans written by the preprocess (tile culling) replace the full square.
// grid = (blocks per view, views): the warps of a view's blocks stride over its Gaussians, and each block counts
// the digits of the keys it writes (the histograms of the following tile sort) in shared memory, then adds them
// to the view's global histograms once.
constexpr int EMIT_WARPS = 8;
constexpr int EMIT_HIST_PASSES = 4;
template <bool TIGHT>
__global__ void __launch_bounds__(EMIT_WARPS * 32)
emit_kernel(const SplatRec* __restrict__ recs, const uint4* __restrict__ spans, const uint32_t* __restrict__ sorted_ids,
            const uint32_t* __restrict__ offsets, int N, int tiles_x, int tiles_y, const __grid_constant__ ViewSpans vs,
            uint32_t* __restrict__ tile_keys, uint32_t* __restrict__ vals, uint32_t* __restrict__ hist, int hist_passes) {
    __shared__ uint32_t s_off[EMIT_WARPS][33];
    __shared__ int s_x0[EMIT_WARPS][32], s_y0[EMIT_WARPS][32], s_w[EMIT_WARPS][32];
    __shared__ uint32_t s_idx[EMIT_WARPS][32];
    __shared__ uint4 s_span[TIGHT ? EMIT_WARPS : 1][32];
    __shared__ uint32_t s_hist[EMIT_HIST_PASSES][256];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int v = blockIdx.y;
    const size_t vo = (size_t)v * N;
    recs += vo; sorted_ids += vo; offsets += vo;
    if (TIGHT) spans += vo;
    tile_keys += vs.base[v]; vals += vs.base[v];
    for (int i = threadIdx.x; i < hist_passes * 256; i += EMIT_WARPS * 32) (&s_hist[0][0])[i] = 0;
    __syncthreads();
    for (int s0 = (blockIdx.x * EMIT_WARPS + warp) * 32; s0 < N; s0 += gridDim.x * EMIT_WARPS * 32) {
        const int s = s0 + lane;
        uint32_t idx = 0, off = 0, cnt = 0;
        int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
        uint4 sp = make_uint4(0xFFFFFFFFu, 0u, 0u, 0u);
        if (s < N) {
            idx = sorted_ids[s];
            off = offsets[s];
            const float4 g = __ldg(&recs[idx].g);
            const int radius = __float_as_int(g.w);
            if (radius > 0) {
                get_rect(g.x, g.y, radius, tiles_x, tiles_y, x0, y0, x1, y1);
                cnt = (uint32_t)((x1 - x0) * (y1 - y0));
                if (TIGHT) {
                    sp = __ldg(&spans[idx]);
                    if (sp.x != 0xFFFFFFFFu)
                        cnt = ((sp.x >> 8) & 255u) + (sp.x >> 24) + ((sp.y >> 8) & 255u) + (sp.y >> 24) +
                              ((sp.z >> 8) & 255u) + (sp.z >> 24) + ((sp.w >> 8) & 255u) + (sp.w >> 24);
                }
            }
        }
        if (TIGHT) s_span[warp][lane] = sp;
        // lanes past N inherit the end of the span so the offsets stay non-decreasing
        const uint32_t endv = off + cnt;
        const int last = min(31, N - 1 - s0);
        const uint32_t span_end = __shfl_sync(0xFFFFFFFFu, endv, last);
        if (s >= N) off = span_end;
        s_off[warp][lane] = off; s_x0[warp][lane] = x0; s_y0[warp][lane] = y0; s_w[warp][lane] = x1 - x0; s_idx[warp][lane] = idx;
        if (lane == 0) s_off[warp][32] = span_end;
        __syncwarp();
        const uint32_t base = s_off[warp][0];
        for (uint32_t t0 = base; t0 < span_end; t0 += 32) {          // warp-uniform trip count (the digit votes)
            const uint32_t t = t0 + lane;
            const bool ok = t < span_end;
            uint32_t key = 0;
            if (ok) {
                // largest L with s_off[L] <= t  (zero-count entries share an offset with their successor: skipped naturally)
                int lo = 0;
#pragma unroll
                for (int step = 16; step > 0; step >>= 1)
                    if (s_off[warp][lo + step] <= t) lo += step;
                uint32_t local = t - s_off[warp][lo];
                const int w = s_w[warp][lo];
                int ry, rx;
                bool full = true;
                if (TIGHT) {
                    const uint4 q = s_span[warp][lo];
                    if (q.x != 0xFFFFFFFFu) {
                        full = false;
                        const uint32_t rows[4] = {q.x, q.y, q.z, q.w};
                        ry = 0; rx = 0;
                        bool found = false;
#pragma unroll
                        for (int r = 0; r < 8; r++) {
                            const uint32_t e = (rows[r >> 1] >> (16 * (r & 1))) & 0xFFFFu;
                            const uint32_t c = e >> 8;
                            if (!found) {
                                if (local < c) { found = true; ry = r; rx = (int)((e & 255u) + local); }
                                else local -= c;
                            }
                        }
                    }
                }
                if (full) { ry = (int)local / w; rx = (int)local - ry * w; }
                key = (uint32_t)((s_y0[warp][lo] + ry) * tiles_x + s_x0[warp][lo] + rx);
                tile_keys[t] = key;
                vals[t] = s_idx[warp][lo];
            }
            // digit histograms of the tile sort: neighbouring slots mostly share their high digits, so a warp that
            // agrees adds its count from one lane (as rs_histogram)
            const uint32_t okmask = __ballot_sync(0xFFFFFFFFu, ok);
            for (int p = 0; p < hist_passes; p++) {
                const uint32_t d = (key >> (8 * p)) & 0xFF;
                const uint32_t d0 = __shfl_sync(0xFFFFFFFFu, d, 0);
                if (__all_sync(0xFFFFFFFFu, !ok || d == d0)) {
                    if (lane == 0) atomicAdd(&s_hist[p][d0], __popc(okmask));
                } else if (ok) {
                    atomicAdd(&s_hist[p][d], 1u);
                }
            }
        }
        __syncwarp();      // the warp's staging arrays are rewritten by its next group of Gaussians
    }
    __syncthreads();
    uint32_t* gh = hist + (size_t)v * EMIT_HIST_PASSES * 256;
    for (int i = threadIdx.x; i < hist_passes * 256; i += EMIT_WARPS * 32) {
        const uint32_t c = (&s_hist[0][0])[i];
        if (c) atomicAdd(gh + i, c);
    }
}

// one thread per pair of the chunk buffer; view v's pairs are [base[v], base[v+1]) and its ranges [v][tiles][2]
__global__ void __launch_bounds__(256)
ranges_kernel(const uint32_t* __restrict__ keys, const __grid_constant__ ViewSpans vs, int ntiles,
              uint32_t* __restrict__ ranges) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= vs.base[vs.n]) return;
    int v = 0;
    while (v + 1 < vs.n && g >= vs.base[v + 1]) v++;
    const int64_t b = vs.base[v], i = g - b, P = vs.base[v + 1] - b;
    keys += b;
    ranges += (size_t)v * ntiles * 2;
    const uint32_t t = keys[i];
    if (i == 0) ranges[2 * t] = 0;
    else {
        const uint32_t prev = keys[i - 1];
        if (prev != t) { ranges[2 * prev + 1] = (uint32_t)i; ranges[2 * t] = (uint32_t)i; }
    }
    if (i == P - 1) ranges[2 * t + 1] = (uint32_t)P;
}

__global__ void __launch_bounds__(256)
sorted_keys_kernel(const SplatRec* __restrict__ recs, const uint32_t* __restrict__ point_list,
                   const uint32_t* __restrict__ tile_keys, int64_t P, uint64_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float depth = recs[point_list[i]].g.z;
    out[i] = ((uint64_t)tile_keys[i] << 32) | (uint64_t)__float_as_uint(depth);
}

}  // namespace

int gs_launch_emit_multi(const SplatRec* recs, const uint4* spans, const uint32_t* sorted_ids, const uint32_t* offsets,
                         int N, int tiles_x, int tiles_y, const ViewSpans& vs, uint32_t* tile_keys, uint32_t* vals,
                         uint32_t* hist, int hist_passes, cudaStream_t s) {
    if (N <= 0 || vs.n <= 0) return 0;
    if (vs.n > GS_MAX_SEGS || hist_passes < 0 || hist_passes > EMIT_HIST_PASSES || !hist) { gs_set_error("emit: bad argument"); return 1; }
    // about two waves of 256-thread blocks over the whole card, split between the views: enough warps in flight,
    // few enough blocks that the per-block histogram flush stays small next to the pairs
    const int per_view = (N + EMIT_WARPS * 32 - 1) / (EMIT_WARPS * 32);
    const int bpv = std::max(1, std::min(per_view, GS_NUM_SMS * 16 / vs.n));
    const dim3 grid(bpv, vs.n);
    if (spans) emit_kernel<true><<<grid, EMIT_WARPS * 32, 0, s>>>(recs, spans, sorted_ids, offsets, N, tiles_x, tiles_y, vs, tile_keys, vals, hist, hist_passes);
    else emit_kernel<false><<<grid, EMIT_WARPS * 32, 0, s>>>(recs, nullptr, sorted_ids, offsets, N, tiles_x, tiles_y, vs, tile_keys, vals, hist, hist_passes);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int gs_launch_ranges_multi(const uint32_t* sorted_tile_keys, const ViewSpans& vs, int ntiles, uint32_t* ranges,
                           cudaStream_t s) {
    const int64_t P = vs.n > 0 ? vs.base[vs.n] : 0;
    if (P <= 0) return 0;
    ranges_kernel<<<(unsigned)((P + 255) / 256), 256, 0, s>>>(sorted_tile_keys, vs, ntiles, ranges);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int gs_launch_sorted_keys(const SplatRec* recs, const uint32_t* point_list, const uint32_t* tile_keys, int64_t P,
                          uint64_t* keys_out, cudaStream_t s) {
    if (P <= 0) return 0;
    sorted_keys_kernel<<<(unsigned)((P + 255) / 256), 256, 0, s>>>(recs, point_list, tile_keys, P, keys_out);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
