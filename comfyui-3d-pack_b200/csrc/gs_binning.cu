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

namespace {

// Each warp takes 32 consecutive depth-sorted Gaussians.  Their output runs are back to back
// ([offsets[s0], offsets[s0+32]) is one contiguous span), so the lanes sweep that span with fully
// coalesced stores and find the owning Gaussian of each slot by binary search over the 32 offsets.
// TIGHT: the per-row tile spans written by the preprocess (tile culling) replace the full square.
constexpr int EMIT_WARPS = 8;
template <bool TIGHT>
__global__ void __launch_bounds__(EMIT_WARPS * 32)
emit_kernel(const SplatRec* __restrict__ recs, const uint4* __restrict__ spans, const uint32_t* __restrict__ sorted_ids,
            const uint32_t* __restrict__ offsets, int N, int tiles_x, int tiles_y,
            uint32_t* __restrict__ tile_keys, uint32_t* __restrict__ vals) {
    __shared__ uint32_t s_off[EMIT_WARPS][33];
    __shared__ int s_x0[EMIT_WARPS][32], s_y0[EMIT_WARPS][32], s_w[EMIT_WARPS][32];
    __shared__ uint32_t s_idx[EMIT_WARPS][32];
    __shared__ uint4 s_span[TIGHT ? EMIT_WARPS : 1][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int s0 = (blockIdx.x * EMIT_WARPS + warp) * 32;
    if (s0 >= N) return;
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
    for (uint32_t t = base + lane; t < span_end; t += 32) {
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
        tile_keys[t] = (uint32_t)((s_y0[warp][lo] + ry) * tiles_x + s_x0[warp][lo] + rx);
        vals[t] = s_idx[warp][lo];
    }
}

__global__ void __launch_bounds__(256)
ranges_kernel(const uint32_t* __restrict__ keys, int64_t P, uint32_t* __restrict__ ranges) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
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

int gs_launch_emit(const SplatRec* recs, const uint4* spans, const uint32_t* sorted_ids, const uint32_t* offsets, int N,
                   int tiles_x, int tiles_y, uint32_t* tile_keys, uint32_t* vals, cudaStream_t s) {
    if (N <= 0) return 0;
    const int blocks = (N + EMIT_WARPS * 32 - 1) / (EMIT_WARPS * 32);
    if (spans) emit_kernel<true><<<blocks, EMIT_WARPS * 32, 0, s>>>(recs, spans, sorted_ids, offsets, N, tiles_x, tiles_y, tile_keys, vals);
    else emit_kernel<false><<<blocks, EMIT_WARPS * 32, 0, s>>>(recs, nullptr, sorted_ids, offsets, N, tiles_x, tiles_y, tile_keys, vals);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int gs_launch_ranges(const uint32_t* sorted_tile_keys, int64_t P, uint32_t* ranges, cudaStream_t s) {
    if (P <= 0) return 0;
    ranges_kernel<<<(unsigned)((P + 255) / 256), 256, 0, s>>>(sorted_tile_keys, P, ranges);
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
