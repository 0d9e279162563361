// Marching cubes over a dense [X,Y,Z] fp32 volume (the PyMCubes `marching_cubes(volume, iso)` contract), sm_90a.
//
// Count pass -> two scans -> (host reads the totals: the one sync) -> write pass.  Vertices are ordered by
// (owner point, axis x<y<z), every crossing edge being owned by its lower end; triangles by (cell, table order),
// a cell being named by its min corner.  Both passes read the volume through a shared-memory brick of
// BX*BY*BZ points with a +2 halo, so each sample comes from HBM once per pass (halo re-reads hit L2).
//
// Algorithmic bytes (N grid points, V vertices, F triangles):
//   count  4 (volume) + 4 + 4 (vertex and triangle counts)                                  = 12 B/point
//   scans  2 x (count read twice: 8, offset written: 4)                                      = 24 B/point
//   write  4 (volume) + 4 + 4 (vertex and triangle offsets) + 12 B/vertex + 12 B/triangle  = 12 B/point
//   total  48 B/point + 12 B/vertex + 12 B/triangle: a 256^3 grid moves ~0.8 GB, ~0.24 ms at 3.35 TB/s (a model).
#include "../../include/ngp_b200.h"
#include "gs_common.cuh"
#include "mc_table.cuh"

namespace {

constexpr int BZ = 32, BY = 8, BX = 4;                 // points per brick; z is the contiguous axis
constexpr int HZ = BZ + 2, HY = BY + 2, HX = BX + 2;   // +2: the write pass reads crossings of owner points at +1
constexpr int MC_THREADS = BZ * BY;                    // one thread per (y, z) column of the brick, BX points each

struct Grid {
    int X, Y, Z;
    long long YZ;
};

// s[i][j][k] = vol[x0+i, y0+j, z0+k] (0 outside the volume: such samples are never read as corners or edge ends)
__device__ __forceinline__ void load_brick(const float* __restrict__ vol, const Grid g, int x0, int y0, int z0,
                                           float (*s)[HY][HZ]) {
    for (int t = threadIdx.x; t < HX * HY * HZ; t += MC_THREADS) {
        const int k = t % HZ, j = (t / HZ) % HY, i = t / (HZ * HY);
        const int x = x0 + i, y = y0 + j, z = z0 + k;
        s[i][j][k] = (x < g.X && y < g.Y && z < g.Z) ? __ldg(vol + (long long)x * g.YZ + (long long)y * g.Z + z) : 0.f;
    }
    __syncthreads();
}

// bit a set iff the edge from brick point (i,j,k) along axis a exists and crosses
__device__ __forceinline__ uint32_t edge_mask(float (*s)[HY][HZ], int i, int j, int k, int x, int y, int z,
                                              const Grid g, float iso) {
    const bool up = s[i][j][k] > iso;
    uint32_t m = 0;
    if (x + 1 < g.X && (s[i + 1][j][k] > iso) != up) m |= 1u;
    if (y + 1 < g.Y && (s[i][j + 1][k] > iso) != up) m |= 2u;
    if (z + 1 < g.Z && (s[i][j][k + 1] > iso) != up) m |= 4u;
    return m;
}

__device__ __forceinline__ uint32_t cube_index(float (*s)[HY][HZ], int i, int j, int k, float iso) {
    uint32_t c = 0;
#pragma unroll
    for (int q = 0; q < 8; q++) c |= (uint32_t)(s[i + (q & 1)][j + ((q >> 1) & 1)][k + (q >> 2)] > iso) << q;
    return c;
}

__global__ void __launch_bounds__(MC_THREADS) mc_count_kernel(const float* __restrict__ vol, const Grid g, float iso,
                                                             uint32_t* __restrict__ vcount, uint32_t* __restrict__ tcount,
                                                             unsigned long long* __restrict__ nonfinite) {
    __shared__ float s[HX][HY][HZ];
    const int z0 = blockIdx.x * BZ, y0 = blockIdx.y * BY, x0 = blockIdx.z * BX;
    load_brick(vol, g, x0, y0, z0, s);
    const int k = threadIdx.x % BZ, j = threadIdx.x / BZ;
    const int y = y0 + j, z = z0 + k;
    bool bad = false;
    if (y < g.Y && z < g.Z) {
        for (int i = 0; i < BX && x0 + i < g.X; i++) {
            const int x = x0 + i;
            const long long p = (long long)x * g.YZ + (long long)y * g.Z + z;
            bad |= !isfinite(s[i][j][k]);
            vcount[p] = __popc(edge_mask(s, i, j, k, x, y, z, g, iso));
            const bool cell = x + 1 < g.X && y + 1 < g.Y && z + 1 < g.Z;
            tcount[p] = cell ? mc_tri_count[cube_index(s, i, j, k, iso)] : 0u;
        }
    }
    if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(nonfinite, 1ull);
}

__global__ void __launch_bounds__(MC_THREADS) mc_write_kernel(const float* __restrict__ vol, const Grid g, float iso,
                                                             const uint32_t* __restrict__ voff,
                                                             const uint32_t* __restrict__ toff, float* __restrict__ verts,
                                                             int32_t* __restrict__ tris) {
    __shared__ float s[HX][HY][HZ];
    const int z0 = blockIdx.x * BZ, y0 = blockIdx.y * BY, x0 = blockIdx.z * BX;
    load_brick(vol, g, x0, y0, z0, s);
    const int k = threadIdx.x % BZ, j = threadIdx.x / BZ;
    const int y = y0 + j, z = z0 + k;
    if (y >= g.Y || z >= g.Z) return;
    for (int i = 0; i < BX && x0 + i < g.X; i++) {
        const int x = x0 + i;
        const long long p = (long long)x * g.YZ + (long long)y * g.Z + z;
        const uint32_t m = edge_mask(s, i, j, k, x, y, z, g, iso);
        if (m) {
            const float va = s[i][j][k];
            const float vb[3] = {s[i + 1][j][k], s[i][j + 1][k], s[i][j][k + 1]};
            const int idx[3] = {x, y, z};
            uint32_t v = __ldg(voff + p);
#pragma unroll
            for (int a = 0; a < 3; a++) {
                if (!((m >> a) & 1u)) continue;
                // fp32, no contraction possible: t = (iso - va) / (vb - va); coord = float(index) + t
                const float t = __fdiv_rn(__fsub_rn(iso, va), __fsub_rn(vb[a], va));
                float* o = verts + 3ull * v++;
                o[0] = (float)x; o[1] = (float)y; o[2] = (float)z;
                o[a] = __fadd_rn((float)idx[a], t);
            }
        }
        if (x + 1 >= g.X || y + 1 >= g.Y || z + 1 >= g.Z) continue;
        const uint32_t cube = cube_index(s, i, j, k, iso);
        const int nt = mc_tri_count[cube];
        if (!nt) continue;
        int32_t* o = tris + 3ll * __ldg(toff + p);
        for (int q = 0; q < 3 * nt; q++) {
            const int e = mc_tri_edges[cube][q], a = e >> 2, lo = e & 1, hi = (e >> 1) & 1;
            // owner corner offset: along a 0; along the other two axes b < c, (lo, hi)
            const int ox = a == 0 ? 0 : lo, oy = a == 0 ? lo : (a == 1 ? 0 : hi), oz = a == 2 ? 0 : hi;
            const int qi = i + ox, qj = j + oy, qk = k + oz;
            uint32_t vid = __ldg(voff + p + (long long)ox * g.YZ + (long long)oy * g.Z + oz);
            const bool up = s[qi][qj][qk] > iso;
            if (a >= 1 && x + ox + 1 < g.X && (s[qi + 1][qj][qk] > iso) != up) vid++;
            if (a == 2 && y + oy + 1 < g.Y && (s[qi][qj + 1][qk] > iso) != up) vid++;
            o[q] = (int32_t)vid;
        }
    }
}

inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace

// scratch: vertex counts, triangle counts, vertex offsets, triangle offsets (u32 per point each), scan scratch
static size_t mc_scratch_bytes(long long n) { return 4 * align256((size_t)n * 4) + gs_scan_scratch_bytes(n); }

static bool mc_dims_ok(int X, int Y, int Z) {
    return X >= 0 && Y >= 0 && Z >= 0 && (X + BX - 1LL) / BX <= 65535 && (Y + BY - 1LL) / BY <= 65535;
}

extern "C" {

size_t ngp_b200_mcubes_scratch_bytes(int32_t X, int32_t Y, int32_t Z) {
    if (X < 2 || Y < 2 || Z < 2) return 0;
    return mc_scratch_bytes((long long)X * Y * Z);
}

int32_t ngp_b200_mcubes_count(const float* volume, int32_t X, int32_t Y, int32_t Z, float iso,
                              unsigned long long* totals_dev3, void* scratch, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!totals_dev3) { gs_set_error("mcubes_count: NULL totals"); return 1; }
    if (!mc_dims_ok(X, Y, Z)) { gs_set_error("mcubes_count: unsupported volume shape %dx%dx%d", X, Y, Z); return 1; }
    GS_CUDA_CHECK(cudaMemsetAsync(totals_dev3, 0, 3 * sizeof(unsigned long long), s));
    if (X < 2 || Y < 2 || Z < 2) return 0;
    if (!volume || !scratch) { gs_set_error("mcubes_count: NULL volume / scratch"); return 1; }
    const long long n = (long long)X * Y * Z;
    const size_t arr = align256((size_t)n * 4);
    uint32_t* vcount = (uint32_t*)scratch;
    uint32_t* tcount = (uint32_t*)((char*)scratch + arr);
    uint32_t* voff = (uint32_t*)((char*)scratch + 2 * arr);
    uint32_t* toff = (uint32_t*)((char*)scratch + 3 * arr);
    void* scan_scratch = (char*)scratch + 4 * arr;
    const Grid g{X, Y, Z, (long long)Y * Z};
    const dim3 grid((Z + BZ - 1) / BZ, (Y + BY - 1) / BY, (X + BX - 1) / BX);
    mc_count_kernel<<<grid, MC_THREADS, 0, s>>>(volume, g, iso, vcount, tcount, totals_dev3 + 2);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    if (gs_scan_gather_u32(vcount, nullptr, voff, totals_dev3, n, scan_scratch, s)) return 1;
    if (gs_scan_gather_u32(tcount, nullptr, toff, totals_dev3 + 1, n, scan_scratch, s)) return 1;
    return 0;
}

int32_t ngp_b200_mcubes_write(const float* volume, int32_t X, int32_t Y, int32_t Z, float iso,
                              const unsigned long long* totals_host3, float* verts, int32_t* tris, void* scratch,
                              void* stream) {
    if (!totals_host3) { gs_set_error("mcubes_write: NULL totals"); return 1; }
    if (!mc_dims_ok(X, Y, Z)) { gs_set_error("mcubes_write: unsupported volume shape %dx%dx%d", X, Y, Z); return 1; }
    if (totals_host3[2]) { gs_set_error("mcubes: the volume holds a non-finite sample (NaN or inf)"); return 1; }
    if (totals_host3[0] >= (1ull << 31) || totals_host3[1] >= (1ull << 31)) {
        gs_set_error("mcubes: %llu vertices / %llu triangles: int32 indices need fewer than 2^31 of each",
                     totals_host3[0], totals_host3[1]);
        return 1;
    }
    if (X < 2 || Y < 2 || Z < 2 || (totals_host3[0] == 0 && totals_host3[1] == 0)) return 0;
    if (!volume || !scratch || !verts || !tris) { gs_set_error("mcubes_write: NULL pointer"); return 1; }
    const size_t arr = align256((size_t)X * Y * Z * 4);
    const uint32_t* voff = (const uint32_t*)((char*)scratch + 2 * arr);
    const uint32_t* toff = (const uint32_t*)((char*)scratch + 3 * arr);
    const Grid g{X, Y, Z, (long long)Y * Z};
    const dim3 grid((Z + BZ - 1) / BZ, (Y + BY - 1) / BY, (X + BX - 1) / BX);
    mc_write_kernel<<<grid, MC_THREADS, 0, (cudaStream_t)stream>>>(volume, g, iso, voff, toff, verts, tris);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

}  // extern "C"
