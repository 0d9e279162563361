// distCUDA2 replacement: mean squared distance to the 3 nearest neighbours.
// Replaces simple_knn._C.distCUDA2 (called once per run from
// main_3DGS_renderer.py:408,419; SURVEY.md App. A.5).
//
// Two exact algorithms, same result (the three smallest squared distances per point):
//  * knn3_kernel      tiled all-pairs search, O(N^2): every thread keeps its 3 smallest squared distances while
//                     tiles of 1024 points stream through shared memory.  Used for small N and as the fallback
//                     for non-finite input.  0.66 s at N = 1e6.
//  * grid search      uniform grid over the bounding box (~3 points per cell), points counting-sorted by cell
//                     with the library's radix sort, then per point ring-by-ring search of the surrounding cells
//                     until the third-best distance is inside the searched block ((ring * cell)^2 bound) — exact,
//                     O(N) for non-degenerate clouds.
#include "../../include/gs_b200.h"
#include "gs_common.cuh"
#include <algorithm>
#include <cmath>

namespace {
constexpr int KT = 256;
constexpr int KTILE = 1024;

__global__ void __launch_bounds__(KT) knn3_kernel(const float* __restrict__ pts, int N, float* __restrict__ out) {
    __shared__ float sx[KTILE], sy[KTILE], sz[KTILE];
    const int i = blockIdx.x * KT + threadIdx.x;
    float x = 0.f, y = 0.f, z = 0.f;
    if (i < N) { x = pts[3 * i]; y = pts[3 * i + 1]; z = pts[3 * i + 2]; }
    float b0 = 3.0e38f, b1 = 3.0e38f, b2 = 3.0e38f;   // b0 <= b1 <= b2
    for (int base = 0; base < N; base += KTILE) {
        __syncthreads();
        for (int j = threadIdx.x; j < KTILE; j += KT) {
            const int g = base + j;
            if (g < N) { sx[j] = pts[3 * g]; sy[j] = pts[3 * g + 1]; sz[j] = pts[3 * g + 2]; }
            else { sx[j] = 1.0e18f; sy[j] = 1.0e18f; sz[j] = 1.0e18f; }
        }
        __syncthreads();
        const int self = i - base;
#pragma unroll 8
        for (int j = 0; j < KTILE; j++) {
            const float dx = sx[j] - x, dy = sy[j] - y, dz = sz[j] - z;
            float d = dx * dx + dy * dy + dz * dz;
            if (j == self) d = 3.0e38f;
            if (d < b2) {
                if (d < b1) { b2 = b1; if (d < b0) { b1 = b0; b0 = d; } else b1 = d; }
                else b2 = d;
            }
        }
    }
    if (i < N) {
        // fewer than 3 other points: average what exists (matches an all-pairs definition)
        float s = 0.f; int c = 0;
        if (b0 < 1.0e37f) { s += b0; c++; }
        if (b1 < 1.0e37f) { s += b1; c++; }
        if (b2 < 1.0e37f) { s += b2; c++; }
        out[i] = c ? s / 3.0f : 0.f;
    }
}
// ---- grid search ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ int ordered_int(float f) { const int i = __float_as_int(f); return i ^ ((i >> 31) & 0x7fffffff); }
__device__ __forceinline__ float ordered_float(int i) { return __int_as_float(i ^ ((i >> 31) & 0x7fffffff)); }

// box[0..2] = min, box[3..5] = max (ordered ints), box[6] = 1 if a non-finite coordinate was seen
__global__ void __launch_bounds__(256) knn_bbox_kernel(const float* __restrict__ pts, int N, int* __restrict__ box) {
    __shared__ int s_box[7];
    if (threadIdx.x < 3) s_box[threadIdx.x] = 0x7fffffff;
    else if (threadIdx.x < 6) s_box[threadIdx.x] = (int)0x80000000;
    else if (threadIdx.x == 6) s_box[6] = 0;
    __syncthreads();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
#pragma unroll
        for (int d = 0; d < 3; d++) {
            const float v = pts[3 * (size_t)i + d];
            if (!isfinite(v)) { s_box[6] = 1; continue; }
            const int o = ordered_int(v);
            atomicMin(&s_box[d], o); atomicMax(&s_box[3 + d], o);
        }
    }
    __syncthreads();
    if (threadIdx.x < 3) atomicMin(&box[threadIdx.x], s_box[threadIdx.x]);
    else if (threadIdx.x < 6) atomicMax(&box[threadIdx.x], s_box[threadIdx.x]);
    else if (threadIdx.x == 6 && s_box[6]) atomicOr(&box[6], 1);
}

struct KnnGrid { float mn[3]; float inv_cs, cs; int G; };

__device__ __forceinline__ KnnGrid knn_grid_of(const int* __restrict__ box, int G) {
    KnnGrid g; g.G = G;
    float ext = 0.f;
#pragma unroll
    for (int d = 0; d < 3; d++) { g.mn[d] = ordered_float(box[d]); ext = fmaxf(ext, ordered_float(box[3 + d]) - g.mn[d]); }
    g.cs = fmaxf(ext, 1e-30f) / (float)G * 1.0001f;      // cubic cells; the slack keeps the max coordinate inside cell G-1
    g.inv_cs = 1.0f / g.cs;
    return g;
}
__device__ __forceinline__ int knn_cell1(const KnnGrid& g, float v, int d) { return min(g.G - 1, max(0, (int)((v - g.mn[d]) * g.inv_cs))); }

__global__ void __launch_bounds__(256) knn_cells_kernel(const float* __restrict__ pts, int N, const int* __restrict__ box, int G,
                                                        uint32_t* __restrict__ keys, uint32_t* __restrict__ ids) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const KnnGrid g = knn_grid_of(box, G);
    const int cx = knn_cell1(g, pts[3 * (size_t)i], 0), cy = knn_cell1(g, pts[3 * (size_t)i + 1], 1), cz = knn_cell1(g, pts[3 * (size_t)i + 2], 2);
    keys[i] = (uint32_t)((cz * G + cy) * G + cx);
    ids[i] = (uint32_t)i;
}

// sorted point records + first index of every cell (cell_start has G^3 + 1 entries, pre-filled with N)
__global__ void __launch_bounds__(256) knn_gather_kernel(const float* __restrict__ pts, int N, const uint32_t* __restrict__ keys,
                                                         const uint32_t* __restrict__ ids, float4* __restrict__ sorted,
                                                         uint32_t* __restrict__ cell_start) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const uint32_t id = ids[i], k = keys[i];
    sorted[i] = make_float4(pts[3 * (size_t)id], pts[3 * (size_t)id + 1], pts[3 * (size_t)id + 2], __uint_as_float(id));
    if (i == 0 || keys[i - 1] != k) cell_start[k] = (uint32_t)i;
}

// cell_start[c] = first point of the next non-empty cell for empty cells (suffix minimum), one block-strided backward pass
__global__ void knn_fill_empty_kernel(uint32_t* __restrict__ cell_start, int ncells, int N) {
    // single thread block walks backwards in chunks; ncells <= 2^24, cheap next to the search
    __shared__ uint32_t carry;
    if (threadIdx.x == 0) carry = (uint32_t)N;
    __syncthreads();
    for (int hi = ncells; hi > 0; hi -= blockDim.x) {
        const int c = hi - 1 - (int)threadIdx.x;
        uint32_t v = (c >= 0) ? cell_start[c] : 0xFFFFFFFFu;
        // inclusive suffix-min inside the chunk (thread 0 holds the highest cell)
        for (int o = 1; o < (int)blockDim.x; o <<= 1) {
            __shared__ uint32_t buf[1024];
            buf[threadIdx.x] = v; __syncthreads();
            if ((int)threadIdx.x >= o) v = min(v, buf[threadIdx.x - o]);
            __syncthreads();
        }
        v = min(v, carry);
        if (c >= 0) cell_start[c] = v;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1 || c == 0) carry = v;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(128) knn_search_kernel(const float4* __restrict__ sorted, int N, const int* __restrict__ box, int G,
                                                         const uint32_t* __restrict__ cell_start, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const KnnGrid g = knn_grid_of(box, G);
    const float4 p = sorted[i];
    const int cx = knn_cell1(g, p.x, 0), cy = knn_cell1(g, p.y, 1), cz = knn_cell1(g, p.z, 2);
    float b0 = 3.0e38f, b1 = 3.0e38f, b2 = 3.0e38f;   // b0 <= b1 <= b2
    for (int r = 0; r < G; r++) {
        const int z0 = max(cz - r, 0), z1 = min(cz + r, G - 1), y0 = max(cy - r, 0), y1 = min(cy + r, G - 1);
        for (int z = z0; z <= z1; z++) {
            for (int y = y0; y <= y1; y++) {
                const bool shell = (abs(z - cz) == r) || (abs(y - cy) == r);
                // on the shell's z / y faces the whole x run belongs to ring r, elsewhere only its two end cells
                for (int part = 0; part < (shell ? 1 : 2); part++) {
                    int xa, xb;
                    if (shell) { xa = max(cx - r, 0); xb = min(cx + r, G - 1); }
                    else { xa = xb = (part == 0) ? cx - r : cx + r; if (xa < 0 || xa >= G) continue; }
                    const size_t row = ((size_t)z * G + y) * G;
                    const uint32_t j0 = cell_start[row + xa], j1 = cell_start[row + xb + 1];
                    for (uint32_t j = j0; j < j1; j++) {
                        if ((int)j == i) continue;
                        const float4 q = sorted[j];
                        const float dx = q.x - p.x, dy = q.y - p.y, dz = q.z - p.z;
                        const float d = dx * dx + dy * dy + dz * dz;
                        if (d < b2) {
                            if (d < b1) { b2 = b1; if (d < b0) { b1 = b0; b0 = d; } else b1 = d; }
                            else b2 = d;
                        }
                    }
                }
            }
        }
        const float reach = (float)r * g.cs;                       // every unsearched point is farther than this
        if (b2 <= reach * reach) break;
        if (cx - r <= 0 && cy - r <= 0 && cz - r <= 0 && cx + r >= G - 1 && cy + r >= G - 1 && cz + r >= G - 1) break;
    }
    float sum = 0.f; int c = 0;
    if (b0 < 1.0e37f) { sum += b0; c++; }
    if (b1 < 1.0e37f) { sum += b1; c++; }
    if (b2 < 1.0e37f) { sum += b2; c++; }
    out[__float_as_uint(p.w)] = c ? sum / 3.0f : 0.f;
}
}  // namespace

extern "C" int32_t gs_b200_knn_mean_dist2(const float* points, int32_t N, float* out, void* stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    if (N <= 0) return 0;
    if (!points || !out) { gs_set_error("knn: NULL"); return 1; }
    if (N < 8192) {
        knn3_kernel<<<(N + KT - 1) / KT, KT, 0, s>>>(points, N, out);
        gs_count_launches(1);
        GS_CUDA_CHECK(cudaGetLastError());
        return 0;
    }
    int G = (int)ceil(cbrt((double)N / 3.0));
    G = std::max(1, std::min(G, 256));
    const int ncells = G * G * G;
    int bits = 0; while ((1 << bits) < ncells) bits++;
    const size_t sort_b = gs_sort_scratch_bytes(N);
    const size_t need = 256 + (size_t)N * 4 * 4 + (size_t)N * 16 + ((size_t)ncells + 1) * 4 + sort_b + 1024;
    char* buf = nullptr;
    GS_CUDA_CHECK(cudaMallocAsync((void**)&buf, need, s));
    int* box = (int*)buf;
    uint32_t* keys = (uint32_t*)(buf + 256); uint32_t* keys_alt = keys + N; uint32_t* ids = keys_alt + N; uint32_t* ids_alt = ids + N;
    float4* sorted = (float4*)(ids_alt + N);
    uint32_t* cell_start = (uint32_t*)(sorted + N);
    void* sort_scratch = (void*)(((uintptr_t)(cell_start + ncells + 1) + 255) & ~(uintptr_t)255);
    const int init[7] = {0x7fffffff, 0x7fffffff, 0x7fffffff, (int)0x80000000, (int)0x80000000, (int)0x80000000, 0};
    GS_CUDA_CHECK(cudaMemcpyAsync(box, init, sizeof(init), cudaMemcpyHostToDevice, s));
    knn_bbox_kernel<<<std::min((N + 255) / 256, GS_NUM_SMS * 8), 256, 0, s>>>(points, N, box);
    int hbox[7];
    GS_CUDA_CHECK(cudaMemcpyAsync(hbox, box, sizeof(hbox), cudaMemcpyDeviceToHost, s));
    GS_CUDA_CHECK(cudaStreamSynchronize(s));
    int rc = 0;
    if (hbox[6]) {                      // non-finite coordinates: the all-pairs kernel defines the result
        knn3_kernel<<<(N + KT - 1) / KT, KT, 0, s>>>(points, N, out);
        gs_count_launches(2);
    } else {
        knn_cells_kernel<<<(N + 255) / 256, 256, 0, s>>>(points, N, box, G, keys, ids);
        int in_alt = 0;
        rc = gs_sort_pairs_u32(keys, keys_alt, ids, ids_alt, N, 0, std::max(bits, 1), sort_scratch, &in_alt, s);
        if (!rc) {
            GS_CUDA_CHECK(cudaMemsetAsync(cell_start, 0xFF, ((size_t)ncells + 1) * 4, s));
            knn_gather_kernel<<<(N + 255) / 256, 256, 0, s>>>(points, N, in_alt ? keys_alt : keys, in_alt ? ids_alt : ids, sorted, cell_start);
            knn_fill_empty_kernel<<<1, 1024, 0, s>>>(cell_start, ncells + 1, N);
            knn_search_kernel<<<(N + 127) / 128, 128, 0, s>>>(sorted, N, box, G, cell_start, out);
            gs_count_launches(5);
        }
    }
    cudaError_t e = cudaGetLastError();
    cudaFreeAsync(buf, s);
    if (e != cudaSuccess) { gs_set_error("knn: %s", cudaGetErrorString(e)); return 1; }
    return rc;
}
