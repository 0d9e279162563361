// Differentiable dual marching cubes over a dense [X,Y,Z] fp32 grid (the `diso.DiffDMC` contract of include/ngp_b200.h,
// called by TripoSG and Hunyuan3D's mesh extraction), sm_90a.
//
// The grid is read as if padded by a virtual ring of samples iso + 1 (deform 0), so it has PX x PY x PZ = (X+2) x
// (Y+2) x (Z+2) points and (X+1)(Y+1)(Z+1) cubes.  Work is split into padded z-rows: CTA (I, J) owns point row (I, J),
// the cube row (I, J) and the quads of the edges whose lower end lies on point row (I, J).  It stages the 3 x 3 point
// rows (I-1..I+1, J-1..J+1) in shared memory, from which it derives the cases of the 4 cube rows (I-1..I, J-1..J);
// those are all the cubes that touch point row (I, J).  Row offsets (vertices, quads) are the only per-row state kept
// between passes; every in-row rank is recomputed from the staged samples.  So:
//   count    -> per-row vertex and quad counts + below / above / NaN flags of the real samples
//   scan     -> per-row offsets and totals; a 1-thread pass applies the empty-grid rule
//   (host reads the totals: the one sync)
//   write    -> dual vertices of cube row (I, J), then the quads (or triangles, split here) of point row (I, J); a quad
//               corner's index is its row offset + its in-row rank, and its position (for the split) is recomputed
//   backward -> per real point, a gather over its up to 6 crossed edges of sum(dL/dv / n_group) over each edge's
//               live cubes, in fixed order (no atomics, no host read, no workspace)
//
// Memory at 513^3 (R = 515^2 = 265,225 rows): scratch = counts 2 x 4R + offsets 2 x 4R + scan partials ~4 KB
// = 4.25 MB, independent of the number of cubes; the backward workspace is 0 B.  Shared memory per CTA is
// 9 x 4 PZ (samples) + 4 x 2 PZ (cube cases) + 4 x 4 PZ (in-row ranks, write and backward) = 60 PZ B (31 KB at
// PZ = 515), which caps Z at DMC_MAX_Z.
//
// Algorithmic bytes per point (count and write each): 4 (grid, from HBM once; the other 8 reads of each sample hit
// L2) + 8 x 4 / PZ (row counts / offsets); write adds 12 B/vertex (+12 with deform) and 16 B/quad or 24 B/triangle
// pair.  At 513^3 that is ~0.54 GB per pass, ~0.16 ms at 3.35 TB/s (a model, not a measurement).
#include "../../include/ngp_b200.h"
#include "gs_common.cuh"
#include "fc_table.cuh"

namespace {

constexpr int DMC_MAX_THREADS = 256;
constexpr int DMC_MAX_Z = 3000;

struct Dims {
    int X, Y, Z;          // unpadded
    int PX, PY, PZ;       // padded (+2)
    float iso, ring;      // ring = iso + 1 (fp32)
    int normalize;
};

// local edge (fc_cube_edges numbering) of the cube edge along `axis` whose lower corner is corner c; -1: none
__device__ const signed char dmc_edge_at[3][8] = {
    {0, -1, 4, -1, 2, -1, 6, -1}, {8, 9, -1, -1, 11, 10, -1, -1}, {3, 1, 7, 5, -1, -1, -1, -1}};
// the 4 cubes around an edge along a are P - db e_b - dc e_c, (a, b, c) cyclic; listed (db, dc) from the lowest
// cube, so that the quad's right-hand normal points from the above end to the below end
__device__ const unsigned char dmc_cycle[2][4][2] = {
    {{1, 1}, {0, 1}, {0, 0}, {1, 0}},     // lower end above: normal +e_a
    {{1, 1}, {1, 0}, {0, 0}, {0, 1}}};    // lower end below: normal -e_a

struct Smem {
    float* v;             // [9][PZ]: v[(di*3 + dj)*PZ + k] = padded point (I-1+di, J-1+dj, k)
    uint16_t* cube;       // [4][PZ]: cube (I-1+ci, J-1+cj, k), q = ci*2 + cj: bits 0-7 case, bit 8 live
    uint32_t* rank;       // [4][PZ]: exclusive in-row vertex rank
};

__device__ __forceinline__ Smem smem_layout(char* base, int PZ, bool ranks) {
    Smem s;
    s.v = (float*)base;
    s.cube = (uint16_t*)(base + 36 * (size_t)PZ);
    s.rank = ranks ? (uint32_t*)(base + 44 * (size_t)PZ) : nullptr;
    return s;
}

__device__ __forceinline__ bool real_point(const Dims& d, int pi, int pj, int pk) {
    return pi >= 1 && pi <= d.X && pj >= 1 && pj <= d.Y && pk >= 1 && pk <= d.Z;
}

__device__ void load_rows(const float* __restrict__ grid, const Dims& d, int I, int J, float* v) {
    for (int t = threadIdx.x; t < 9 * d.PZ; t += blockDim.x) {
        const int row = t / d.PZ, k = t - row * d.PZ;
        const int pi = I - 1 + row / 3, pj = J - 1 + row % 3;
        v[t] = real_point(d, pi, pj, k) ? __ldg(grid + ((long long)(pi - 1) * d.Y + (pj - 1)) * d.Z + (k - 1)) : d.ring;
    }
}

__device__ __forceinline__ uint16_t cube_info(const float* v, const Dims& d, int I, int J, int q, int k) {
    const int ci = q >> 1, cj = q & 1;
    const int cI = I - 1 + ci, cJ = J - 1 + cj;
    if (cI < 0 || cI > d.PX - 2 || cJ < 0 || cJ > d.PY - 2 || k < 0 || k > d.PZ - 2) return 0;
    uint32_t c = 0;
    bool live = true;
#pragma unroll
    for (int n = 0; n < 8; n++) {
        const float s = v[((ci + (n & 1)) * 3 + cj + ((n >> 1) & 1)) * d.PZ + k + (n >> 2)];
        live &= isfinite(s);
        c |= (uint32_t)(s < d.iso) << n;
    }
    return live ? (uint16_t)(0x100u | c) : (uint16_t)0;
}

__device__ __forceinline__ uint32_t nvd_of(uint16_t info) { return (info & 0x100u) ? fc_num_vd[info & 0xff] : 0u; }

// exclusive scan across the block of N values per thread (blockDim a multiple of 32, <= DMC_MAX_THREADS)
template <int N>
__device__ void block_exclusive_scan(uint32_t (&x)[N], uint32_t (&total)[N]) {
    __shared__ uint32_t wsum[DMC_MAX_THREADS / 32][N];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    uint32_t incl[N];
#pragma unroll
    for (int n = 0; n < N; n++) {
        incl[n] = x[n];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, incl[n], o);
            if (lane >= o) incl[n] += y;
        }
        if (lane == 31) wsum[warp][n] = incl[n];
    }
    __syncthreads();
#pragma unroll
    for (int n = 0; n < N; n++) {
        uint32_t before = 0, all = 0;
        for (int w = 0; w < nw; w++) {
            if (w < warp) before += wsum[w][n];
            all += wsum[w][n];
        }
        x[n] = before + incl[n] - x[n];
        total[n] = all;
    }
    __syncthreads();
}

// each thread owns the contiguous k range [k0, k1) of the row
__device__ __forceinline__ void seg(const Dims& d, int& k0, int& k1) {
    const int per = (d.PZ + blockDim.x - 1) / blockDim.x;
    k0 = min(d.PZ, (int)threadIdx.x * per);
    k1 = min(d.PZ, k0 + per);
}

// cases of the 4 cube rows over [k0, k1); returns the thread's vertex counts per cube row
__device__ __forceinline__ void cube_rows(const Smem& s, const Dims& d, int I, int J, int k0, int k1,
                                          uint32_t (&nv)[4]) {
    for (int q = 0; q < 4; q++) nv[q] = 0;
    for (int k = k0; k < k1; k++) {
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const uint16_t c = cube_info(s.v, d, I, J, q, k);
            s.cube[q * d.PZ + k] = c;
            nv[q] += nvd_of(c);
        }
    }
}

// cube rows and in-row ranks (write and backward); ends with the block synchronised
__device__ void cube_rows_ranked(const Smem& s, const Dims& d, int I, int J, int k0, int k1) {
    uint32_t nv[4], tot[4];
    cube_rows(s, d, I, J, k0, k1, nv);
    block_exclusive_scan<4>(nv, tot);
    for (int k = k0; k < k1; k++) {
#pragma unroll
        for (int q = 0; q < 4; q++) {
            s.rank[q * d.PZ + k] = nv[q];
            nv[q] += nvd_of(s.cube[q * d.PZ + k]);
        }
    }
    __syncthreads();
}

// the cube (as cube row q, k) and local edge of corner t of the quad around the edge from point (I, J, k) along a;
// false if that cube is not live
__device__ __forceinline__ bool quad_cube(const Smem& s, const Dims& d, int a, int k, int side, int t, int lo_a,
                                          int& q, int& kk, int& e, uint16_t& info) {
    const int b = (a + 1) % 3, c = (a + 2) % 3;
    int off[3];
    off[a] = -lo_a;                             // 0: the edge's lower end is the centre point; 1: it is one below
    off[b] = -dmc_cycle[side][t][0];
    off[c] = -dmc_cycle[side][t][1];
    q = (off[0] + 1) * 2 + (off[1] + 1);
    kk = k + off[2];
    if (kk < 0) return false;
    info = s.cube[q * d.PZ + kk];
    if (!(info & 0x100u)) return false;
    // corner of the edge's lower end inside the cube: the centre point offset by -lo_a along a, minus the cube offset
    int co[3] = {-off[0], -off[1], -off[2]};
    co[a] -= lo_a;
    e = dmc_edge_at[a][co[0] | (co[1] << 1) | (co[2] << 2)];
    return true;
}

// sample value of a point at offset (oi, oj) in {-1,0,1} from the centre row
__device__ __forceinline__ float sample(const Smem& s, const Dims& d, int oi, int oj, int k) {
    return s.v[((oi + 1) * 3 + oj + 1) * d.PZ + k];
}

// the edge from centre point (I, J, k) along a is crossed and its 4 cubes are live
__device__ __forceinline__ bool quad_at(const Smem& s, const Dims& d, int a, int k, int& side) {
    if (a == 2 && k + 1 >= d.PZ) return false;
    const float lo = sample(s, d, 0, 0, k);
    const float up = sample(s, d, a == 0, a == 1, k + (a == 2));
    const bool bl = lo < d.iso;
    if (bl == (up < d.iso)) return false;
    side = bl;
    for (int t = 0; t < 4; t++) {
        int q, kk, e;
        uint16_t info;
        if (!quad_cube(s, d, a, k, side, t, 0, q, kk, e, info)) return false;
    }
    return true;
}

__device__ __forceinline__ float3 point_pos(const float* __restrict__ deform, const Dims& d, int pi, int pj, int pk) {
    float3 p = make_float3((float)(pi - 1), (float)(pj - 1), (float)(pk - 1));
    if (deform && real_point(d, pi, pj, pk)) {
        const float* q = deform + 3 * (((long long)(pi - 1) * d.Y + (pj - 1)) * d.Z + (pk - 1));
        p.x = __fadd_rn(p.x, __ldg(q));
        p.y = __fadd_rn(p.y, __ldg(q + 1));
        p.z = __fadd_rn(p.z, __ldg(q + 2));
    }
    return p;
}

// dual vertex of group g of cube (I-1+ci, J-1+cj, kk): mean of the group's crossings in ascending edge order
__device__ float3 dual_vertex(const Smem& s, const Dims& d, const float* __restrict__ deform, int I, int J, int q,
                              int kk, uint32_t cs, int g) {
    const int ci = q >> 1, cj = q & 1;
    float3 sum = make_float3(0.f, 0.f, 0.f);
    int n = 0;
    for (int e = 0; e < 12; e++) {
        if (fc_group_of[cs][e] != g) continue;
        const int c0 = min(fc_cube_edges[e][0], fc_cube_edges[e][1]), c1 = max(fc_cube_edges[e][0], fc_cube_edges[e][1]);
        const int ai = ci + (c0 & 1), aj = cj + ((c0 >> 1) & 1), ak = kk + (c0 >> 2);
        const int bi = ci + (c1 & 1), bj = cj + ((c1 >> 1) & 1), bk = kk + (c1 >> 2);
        const float sa = s.v[(ai * 3 + aj) * d.PZ + ak], sb = s.v[(bi * 3 + bj) * d.PZ + bk];
        const float3 pa = point_pos(deform, d, I - 1 + ai, J - 1 + aj, ak);
        const float3 pb = point_pos(deform, d, I - 1 + bi, J - 1 + bj, bk);
        const float t = __fdiv_rn(__fsub_rn(d.iso, sa), __fsub_rn(sb, sa));
        sum.x = __fadd_rn(sum.x, __fadd_rn(pa.x, __fmul_rn(t, __fsub_rn(pb.x, pa.x))));
        sum.y = __fadd_rn(sum.y, __fadd_rn(pa.y, __fmul_rn(t, __fsub_rn(pb.y, pa.y))));
        sum.z = __fadd_rn(sum.z, __fadd_rn(pa.z, __fmul_rn(t, __fsub_rn(pb.z, pa.z))));
        n++;
    }
    float3 v = make_float3(__fdiv_rn(sum.x, (float)n), __fdiv_rn(sum.y, (float)n), __fdiv_rn(sum.z, (float)n));
    if (d.normalize) {
        v.x = __fdiv_rn(v.x, (float)(d.X - 1));
        v.y = __fdiv_rn(v.y, (float)(d.Y - 1));
        v.z = __fdiv_rn(v.z, (float)(d.Z - 1));
    }
    return v;
}

__device__ __forceinline__ int group_size(uint32_t cs, int g) {
    int n = 0;
    for (int i = 0; i < FC_MAX_GROUP_EDGES; i++) n += fc_groups[cs][g][i] >= 0;
    return n;
}

__device__ __forceinline__ float3 unit(float3 v) {
    const float l = fmaxf(sqrtf(v.x * v.x + v.y * v.y + v.z * v.z), 1e-12f);
    return make_float3(v.x / l, v.y / l, v.z / l);
}

__device__ __forceinline__ float cos_at(float3 a, float3 b, float3 c) {
    const float3 u = unit(make_float3(b.x - a.x, b.y - a.y, b.z - a.z));
    const float3 w = unit(make_float3(c.x - a.x, c.y - a.y, c.z - a.z));
    return u.x * w.x + u.y * w.y + u.z * w.z;
}

__device__ __forceinline__ float max_cos(float3 a, float3 b, float3 c) {
    return fmaxf(cos_at(a, b, c), fmaxf(cos_at(b, c, a), cos_at(c, a, b)));
}

__device__ __forceinline__ long long row_id(const Dims& d, int I, int J) { return (long long)I * d.PY + J; }

__global__ void __launch_bounds__(DMC_MAX_THREADS) dmc_count_kernel(const float* __restrict__ grid, const Dims d,
                                                                    uint32_t* __restrict__ counts,
                                                                    unsigned long long* __restrict__ flags) {
    extern __shared__ __align__(16) char dmc_smem[];
    const Smem s = smem_layout(dmc_smem, d.PZ, false);
    const int J = blockIdx.x, I = blockIdx.y;
    load_rows(grid, d, I, J, s.v);
    __syncthreads();
    int k0, k1;
    seg(d, k0, k1);
    uint32_t nv[4];
    cube_rows(s, d, I, J, k0, k1, nv);
    bool below = false, above = false, nan = false;
    if (I >= 1 && I <= d.X && J >= 1 && J <= d.Y) {
        for (int k = max(k0, 1); k < min(k1, d.Z + 1); k++) {
            const float v = sample(s, d, 0, 0, k);
            below |= v < d.iso;
            above |= v > d.iso;
            nan |= isnan(v);
        }
    }
    __syncthreads();
    uint32_t c[2] = {nv[3], 0}, tot[2];
    for (int k = k0; k < k1; k++) {
        int side;
        for (int a = 0; a < 3; a++) c[1] += quad_at(s, d, a, k, side);
    }
    block_exclusive_scan<2>(c, tot);
    const unsigned long long f = (__syncthreads_or(below) ? 1ull : 0ull) | (__syncthreads_or(above) ? 2ull : 0ull) |
                                 (__syncthreads_or(nan) ? 4ull : 0ull);
    if (threadIdx.x == 0) {
        const long long r = row_id(d, I, J), R = (long long)d.PX * d.PY;
        counts[r] = tot[0];
        counts[R + r] = tot[1];
        if (f) atomicOr(flags, f);
    }
}

// the grid is empty (diso's min >= iso or max <= iso, NaN propagating): no vertex, no quad
__global__ void dmc_empty_rule_kernel(unsigned long long* totals) {
    const unsigned long long f = totals[2];
    if (!(f & 4ull) && (!(f & 1ull) || !(f & 2ull))) totals[0] = totals[1] = 0;
}

template <bool QUADS>
__global__ void __launch_bounds__(DMC_MAX_THREADS) dmc_write_kernel(const float* __restrict__ grid,
                                                                    const float* __restrict__ deform, const Dims d,
                                                                    const uint32_t* __restrict__ offsets,
                                                                    float* __restrict__ verts,
                                                                    int32_t* __restrict__ faces) {
    extern __shared__ __align__(16) char dmc_smem[];
    const Smem s = smem_layout(dmc_smem, d.PZ, true);
    const int J = blockIdx.x, I = blockIdx.y;
    const long long R = (long long)d.PX * d.PY;
    load_rows(grid, d, I, J, s.v);
    __syncthreads();
    int k0, k1;
    seg(d, k0, k1);
    cube_rows_ranked(s, d, I, J, k0, k1);
    uint32_t voff[4];
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const int cI = I - 1 + (q >> 1), cJ = J - 1 + (q & 1);
        voff[q] = (cI >= 0 && cJ >= 0) ? __ldg(offsets + row_id(d, cI, cJ)) : 0u;
    }
    // dual vertices of cube row (I, J)
    for (int k = k0; k < k1; k++) {
        const uint16_t info = s.cube[3 * d.PZ + k];
        const uint32_t n = nvd_of(info);
        for (uint32_t g = 0; g < n; g++) {
            const float3 v = dual_vertex(s, d, deform, I, J, 3, k, info & 0xff, g);
            float* o = verts + 3ull * (voff[3] + s.rank[3 * d.PZ + k] + g);
            o[0] = v.x; o[1] = v.y; o[2] = v.z;
        }
    }
    // quads of point row (I, J)
    uint32_t nq[1] = {0}, tot[1];
    for (int k = k0; k < k1; k++) {
        int side;
        for (int a = 0; a < 3; a++) nq[0] += quad_at(s, d, a, k, side);
    }
    block_exclusive_scan<1>(nq, tot);
    if (!tot[0]) return;
    unsigned long long qi = (unsigned long long)__ldg(offsets + R + row_id(d, I, J)) + nq[0];
    for (int k = k0; k < k1; k++) {
        for (int a = 0; a < 3; a++) {
            int side;
            if (!quad_at(s, d, a, k, side)) continue;
            int32_t vid[4];
            float3 p[4];
            for (int t = 0; t < 4; t++) {
                int q, kk, e;
                uint16_t info;
                quad_cube(s, d, a, k, side, t, 0, q, kk, e, info);
                const int g = fc_group_of[info & 0xff][e];
                vid[t] = (int32_t)(voff[q] + s.rank[q * d.PZ + kk] + g);
                if (!QUADS) p[t] = dual_vertex(s, d, deform, I, J, q, kk, info & 0xff, g);
            }
            if (QUADS) {
                int32_t* o = faces + 4ull * qi;
                o[0] = vid[0]; o[1] = vid[1]; o[2] = vid[2]; o[3] = vid[3];
            } else {
                // diso's split: config 1 (0,1,3),(1,2,3) iff its largest corner cosine is strictly the smaller
                const float m1 = fmaxf(max_cos(p[0], p[1], p[3]), max_cos(p[1], p[2], p[3]));
                const float m2 = fmaxf(max_cos(p[0], p[1], p[2]), max_cos(p[0], p[2], p[3]));
                int32_t* o = faces + 6ull * qi;
                if (m1 < m2) {
                    o[0] = vid[0]; o[1] = vid[1]; o[2] = vid[3]; o[3] = vid[1]; o[4] = vid[2]; o[5] = vid[3];
                } else {
                    o[0] = vid[0]; o[1] = vid[1]; o[2] = vid[2]; o[3] = vid[0]; o[4] = vid[2]; o[5] = vid[3];
                }
            }
            qi++;
        }
    }
}

// one CTA per real point row (I, J) = (blockIdx.y + 1, blockIdx.x + 1)
__global__ void __launch_bounds__(DMC_MAX_THREADS) dmc_backward_kernel(const float* __restrict__ grid,
                                                                       const float* __restrict__ deform, const Dims d,
                                                                       const uint32_t* __restrict__ offsets,
                                                                       const float* __restrict__ gverts,
                                                                       float* __restrict__ ggrid,
                                                                       float* __restrict__ gdeform) {
    extern __shared__ __align__(16) char dmc_smem[];
    const Smem s = smem_layout(dmc_smem, d.PZ, true);
    const int J = blockIdx.x + 1, I = blockIdx.y + 1;
    load_rows(grid, d, I, J, s.v);
    __syncthreads();
    int k0, k1;
    seg(d, k0, k1);
    cube_rows_ranked(s, d, I, J, k0, k1);
    uint32_t voff[4];
#pragma unroll
    for (int q = 0; q < 4; q++) voff[q] = __ldg(offsets + row_id(d, I - 1 + (q >> 1), J - 1 + (q & 1)));
    const float sx = d.normalize ? (float)(d.X - 1) : 1.f, sy = d.normalize ? (float)(d.Y - 1) : 1.f,
                sz = d.normalize ? (float)(d.Z - 1) : 1.f;
    for (int k = max(k0, 1); k < min(k1, d.Z + 1); k++) {
        float gs = 0.f;
        float3 gd = make_float3(0.f, 0.f, 0.f);
        for (int a = 0; a < 3; a++) {
            for (int lo_a = 0; lo_a < 2; lo_a++) {       // 0: this point is the edge's lower end, 1: its upper end
                const int li = a == 0 ? -lo_a : 0, lj = a == 1 ? -lo_a : 0, lk = k - (a == 2 ? lo_a : 0);
                const float sl = sample(s, d, li, lj, lk);
                const float su = sample(s, d, li + (a == 0), lj + (a == 1), lk + (a == 2));
                const bool bl = sl < d.iso;
                if (bl == (su < d.iso)) continue;
                float3 ge = make_float3(0.f, 0.f, 0.f);
                bool any = false;
                for (int t = 0; t < 4; t++) {
                    int q, kk, e;
                    uint16_t info;
                    if (!quad_cube(s, d, a, k, 0, t, lo_a, q, kk, e, info)) continue;
                    const int g = fc_group_of[info & 0xff][e];
                    const float n = (float)group_size(info & 0xff, g);
                    const float* gv = gverts + 3ull * (voff[q] + s.rank[q * d.PZ + kk] + g);
                    ge.x = __fadd_rn(ge.x, __fdiv_rn(__fdiv_rn(__ldg(gv), sx), n));
                    ge.y = __fadd_rn(ge.y, __fdiv_rn(__fdiv_rn(__ldg(gv + 1), sy), n));
                    ge.z = __fadd_rn(ge.z, __fdiv_rn(__fdiv_rn(__ldg(gv + 2), sz), n));
                    any = true;
                }
                if (!any) continue;
                const float3 pl = point_pos(deform, d, I + li, J + lj, lk);
                const float3 pu = point_pos(deform, d, I + li + (a == 0), J + lj + (a == 1), lk + (a == 2));
                const float3 dp = make_float3(__fsub_rn(pu.x, pl.x), __fsub_rn(pu.y, pl.y), __fsub_rn(pu.z, pl.z));
                const float den = __fsub_rn(su, sl);
                const float t = __fdiv_rn(__fsub_rn(d.iso, sl), den);
                const float gdot = __fadd_rn(__fadd_rn(__fmul_rn(ge.x, dp.x), __fmul_rn(ge.y, dp.y)), __fmul_rn(ge.z, dp.z));
                // crossing = pl + t (pu - pl), t = (iso - sl) / (su - sl): dt/dsl = (t - 1) / den, dt/dsu = -t / den
                const float w = lo_a ? t : __fsub_rn(1.f, t);
                const float dt = lo_a ? -t : __fsub_rn(t, 1.f);
                gd.x = __fadd_rn(gd.x, __fmul_rn(ge.x, w));
                gd.y = __fadd_rn(gd.y, __fmul_rn(ge.y, w));
                gd.z = __fadd_rn(gd.z, __fmul_rn(ge.z, w));
                gs = __fadd_rn(gs, __fdiv_rn(__fmul_rn(gdot, dt), den));
            }
        }
        const long long p = ((long long)(I - 1) * d.Y + (J - 1)) * d.Z + (k - 1);
        if (ggrid) ggrid[p] = gs;
        if (gdeform) { gdeform[3 * p] = gd.x; gdeform[3 * p + 1] = gd.y; gdeform[3 * p + 2] = gd.z; }
    }
}

inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

bool dims_ok(const char* fn, int X, int Y, int Z) {
    if (X < 1 || Y < 1 || Z < 1 || Z > DMC_MAX_Z || X + 2 > 65535 || (long long)(X + 2) * (Y + 2) >= (1ll << 31)) {
        gs_set_error("%s: unsupported grid shape %dx%dx%d (each dimension >= 1, Z <= %d, X <= 65533)", fn, X, Y, Z,
                     DMC_MAX_Z);
        return false;
    }
    return true;
}

Dims make_dims(int X, int Y, int Z, float iso, int normalize) {
    return Dims{X, Y, Z, X + 2, Y + 2, Z + 2, iso, iso + 1.f, normalize};
}

int threads_for(int PZ) { return std::min(DMC_MAX_THREADS, std::max(32, ((PZ + 3) / 4 + 31) / 32 * 32)); }

long long rows(int X, int Y) { return (long long)(X + 2) * (Y + 2); }

// shared memory above the default 48 KB has to be opted into per kernel
template <typename K>
int allow_smem(K kernel, size_t smem) {
    if (smem > 48 * 1024) GS_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    return 0;
}

}  // namespace

extern "C" {

size_t ngp_b200_dmc_scratch_bytes(int32_t X, int32_t Y, int32_t Z) {
    if (X < 1 || Y < 1 || Z < 1) return 0;
    const long long R = rows(X, Y);
    return 2 * align256((size_t)R * 2 * 4) + gs_scan_seg_scratch_bytes(R, 2);
}

int32_t ngp_b200_dmc_count(const float* grid, int32_t X, int32_t Y, int32_t Z, float iso,
                           unsigned long long* totals_dev3, void* scratch, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!totals_dev3) { gs_set_error("dmc_count: NULL totals"); return 1; }
    if (!dims_ok("dmc_count", X, Y, Z)) return 1;
    if (!grid || !scratch) { gs_set_error("dmc_count: NULL grid / scratch"); return 1; }
    const long long R = rows(X, Y);
    uint32_t* counts = (uint32_t*)scratch;
    uint32_t* offsets = (uint32_t*)((char*)scratch + align256((size_t)R * 8));
    void* scan = (char*)scratch + 2 * align256((size_t)R * 8);
    const Dims d = make_dims(X, Y, Z, iso, 0);
    const int threads = threads_for(d.PZ);
    const size_t smem = 44 * (size_t)d.PZ;
    GS_CUDA_CHECK(cudaMemsetAsync(totals_dev3, 0, 3 * sizeof(unsigned long long), s));
    if (allow_smem(dmc_count_kernel, smem)) return 1;
    dmc_count_kernel<<<dim3(d.PY, d.PX), threads, smem, s>>>(grid, d, counts, totals_dev3 + 2);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    if (gs_scan_gather_seg_u32(counts, nullptr, offsets, totals_dev3, R, 2, scan, s)) return 1;
    dmc_empty_rule_kernel<<<1, 1, 0, s>>>(totals_dev3);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

static bool totals_ok(const char* fn, const unsigned long long* totals_host3) {
    if (!totals_host3) { gs_set_error("%s: NULL totals", fn); return false; }
    if (totals_host3[0] >= (1ull << 31) || totals_host3[1] >= (1ull << 31)) {
        gs_set_error("dmc: %llu vertices / %llu quads: int32 indices need fewer than 2^31 of each", totals_host3[0],
                     totals_host3[1]);
        return false;
    }
    return true;
}

int32_t ngp_b200_dmc_write(const float* grid, const float* deform, int32_t X, int32_t Y, int32_t Z, float iso,
                           int32_t quads, int32_t normalize, const unsigned long long* totals_host3, float* verts,
                           int32_t* faces, const void* scratch, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!dims_ok("dmc_write", X, Y, Z) || !totals_ok("dmc_write", totals_host3)) return 1;
    if (normalize && (X < 2 || Y < 2 || Z < 2)) {
        gs_set_error("dmc_write: normalize needs every dimension >= 2, got %dx%dx%d", X, Y, Z);
        return 1;
    }
    if (totals_host3[0] == 0) return 0;
    if (!grid || !scratch || !verts || (totals_host3[1] && !faces)) { gs_set_error("dmc_write: NULL pointer"); return 1; }
    const long long R = rows(X, Y);
    const uint32_t* offsets = (const uint32_t*)((const char*)scratch + align256((size_t)R * 8));
    const Dims d = make_dims(X, Y, Z, iso, normalize);
    const int threads = threads_for(d.PZ);
    const size_t smem = 60 * (size_t)d.PZ;
    if (quads) {
        if (allow_smem(dmc_write_kernel<true>, smem)) return 1;
        dmc_write_kernel<true><<<dim3(d.PY, d.PX), threads, smem, s>>>(grid, deform, d, offsets, verts, faces);
    } else {
        if (allow_smem(dmc_write_kernel<false>, smem)) return 1;
        dmc_write_kernel<false><<<dim3(d.PY, d.PX), threads, smem, s>>>(grid, deform, d, offsets, verts, faces);
    }
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

size_t ngp_b200_dmc_backward_workspace_bytes(int32_t X, int32_t Y, int32_t Z) {
    (void)X; (void)Y; (void)Z;
    return 0;
}

int32_t ngp_b200_dmc_backward(const float* grid, const float* deform, int32_t X, int32_t Y, int32_t Z, float iso,
                              int32_t normalize, const unsigned long long* totals_host3, const float* grad_verts,
                              float* grad_grid, float* grad_deform, const void* scratch, void* workspace,
                              void* stream) {
    (void)workspace;
    cudaStream_t s = (cudaStream_t)stream;
    if (!dims_ok("dmc_backward", X, Y, Z) || !totals_ok("dmc_backward", totals_host3)) return 1;
    if (normalize && (X < 2 || Y < 2 || Z < 2)) {
        gs_set_error("dmc_backward: normalize needs every dimension >= 2, got %dx%dx%d", X, Y, Z);
        return 1;
    }
    if (!grad_grid && !grad_deform) return 0;
    const size_t n = (size_t)X * Y * Z;
    if (totals_host3[0] == 0) {
        if (grad_grid) GS_CUDA_CHECK(cudaMemsetAsync(grad_grid, 0, n * 4, s));
        if (grad_deform) GS_CUDA_CHECK(cudaMemsetAsync(grad_deform, 0, n * 12, s));
        return 0;
    }
    if (!grid || !scratch || !grad_verts) { gs_set_error("dmc_backward: NULL pointer"); return 1; }
    const long long R = rows(X, Y);
    const uint32_t* offsets = (const uint32_t*)((const char*)scratch + align256((size_t)R * 8));
    const Dims d = make_dims(X, Y, Z, iso, normalize);
    const int threads = threads_for(d.PZ);
    const size_t smem = 60 * (size_t)d.PZ;
    if (allow_smem(dmc_backward_kernel, smem)) return 1;
    dmc_backward_kernel<<<dim3(Y, X), threads, smem, s>>>(grid, deform, d, offsets, grad_verts, grad_grid,
                                                         grad_deform);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

}  // extern "C"
