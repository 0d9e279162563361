// FlexiCubes triangle-mesh extraction on a regular grid (the FlexiCubes node's `FlexiCubes.__call__`), sm_90a.
//
// A grid edge is (grid point, axis), so no sort or unique is needed: every crossed edge, dual vertex and quad has a
// closed-form owner.  Forward: count pass over cubes -> four scans -> (host reads the totals: the one sync) -> dual
// vertex + L_dev pass -> quad pass.  Backward (no host read): quad-centre partials per quad slot -> per-cube pass
// that gathers them per dual vertex in a fixed order and writes the weight gradients and per-corner partials ->
// per-point pass that gathers the corner partials of its 8 cubes in a fixed order.  No fp32 atomics anywhere, so
// gradients are bit-identical from run to run.
//
// Attributes (the TRELLIS / Stable3DGen variant, ngp_b200_flexicubes_*_attrs): C channels per grid point, activated by
// a sigmoid, crossed on each group edge with the same end weights s * alpha as the dual vertex and averaged with the
// same beta; training quad centres take the same gamma-weighted diagonal means.  They are the `ATTRS` instantiation of the
// same passes; the C = 0 instantiation is the attribute-free extraction, unchanged.  Their backward adds their terms
// after the geometry's, writes per-corner attribute partials next to the geometry's, and the per-point pass gathers
// them in the same corner order.
//
// Numbering: point (i,j,k) = (i*Sy + j)*Sz + k, cube (i,j,k) = (i*Ry + j)*Rz + k, S = R + 1; corner c of a cube is
// the point at offset (c&1, (c>>1)&1, c>>2); case bit c = s < 0.  Output order: dual vertices by (cube, group),
// then (training) one centre per quad; quads by (owning cube, axis), the owner being the lowest of the 4 cubes, whose
// own copy of the edge is edge 6 (axis 0), 10 (axis 1) or 5 (axis 2).
//
// Algorithmic bytes per cube (forward): 4 (s, read ~once through L1/L2) + 1 (case) + 4 x 4 (counts) + 4 x 12
// (scans) + 4 x 4 (offsets re-read) + 84 (weights, surface cubes) + 12 B/dual vertex + 4 B/L_dev entry + 24 or 48
// B/quad.
#include "../../include/ngp_b200.h"
#include "gs_common.cuh"
#include "fc_table.cuh"

namespace {

constexpr int FC_THREADS = 256;

struct FcGrid {
    int Rx, Ry, Rz;
    long long Sz, Syz;   // point strides along axes 2 and 0 (axis 1 stride = Sz)
    long long F;
};

struct FcWeights {
    const float* beta; long long sb;    // raw weights, row strides; NULL = all ones
    const float* alpha; long long sa;
    const float* gamma; long long sg;
    float ws, ws_half;                  // weight_scale, (1 - weight_scale) / 2
};

struct FcAttrs {
    const float* a; long long stride;   // raw attributes, row stride (unit column stride); NULL when C = 0
    int C;
};

// axis of each cube edge, and the order of the 4 cubes around an owned edge: cube offset (along the two other axes,
// ascending) of slot t is (t >> 1, t & 1) and its local edge is fc_quad_edge[axis][t]
__device__ const unsigned char fc_edge_axis[12] = {0, 2, 0, 2, 0, 2, 0, 2, 1, 1, 1, 1};
__device__ const unsigned char fc_quad_edge[3][4] = {{6, 4, 2, 0}, {10, 9, 11, 8}, {5, 1, 7, 3}};

__device__ __forceinline__ long long cube_id(const FcGrid& g, int i, int j, int k) {
    return ((long long)i * g.Ry + j) * g.Rz + k;
}
__device__ __forceinline__ long long point_id(const FcGrid& g, int i, int j, int k) {
    return (long long)i * g.Syz + (long long)j * g.Sz + k;
}
__device__ __forceinline__ long long corner_point(const FcGrid& g, long long p0, int c) {
    return p0 + (c & 1) * g.Syz + ((c >> 1) & 1) * g.Sz + (c >> 2);
}
__device__ __forceinline__ void cube_ijk(const FcGrid& g, long long f, int& i, int& j, int& k) {
    k = (int)(f % g.Rz);
    const long long r = f / g.Rz;
    j = (int)(r % g.Ry);
    i = (int)(r / g.Ry);
}

__device__ __forceinline__ uint32_t case_of(const FcGrid& g, const float* __restrict__ s, int i, int j, int k) {
    const long long p0 = point_id(g, i, j, k);
    uint32_t c = 0;
#pragma unroll
    for (int q = 0; q < 8; q++) c |= (uint32_t)(__ldg(s + corner_point(g, p0, q)) < 0.f) << q;
    return c;
}

__device__ __forceinline__ bool is_surface(uint32_t c) { return c != 0u && c != 255u; }

__device__ __forceinline__ bool edge_crossed(uint32_t c, int e) {
    return ((c >> fc_cube_edges[e][0]) ^ (c >> fc_cube_edges[e][1])) & 1u;
}

// bit a: cube (i,j,k) with case c owns a quad along axis a (its edge crosses and all 4 cubes exist)
__device__ __forceinline__ uint32_t owned_quads(const FcGrid& g, uint32_t c, int i, int j, int k) {
    uint32_t m = 0;
    if (j + 1 < g.Ry && k + 1 < g.Rz && edge_crossed(c, 6)) m |= 1u;
    if (i + 1 < g.Rx && k + 1 < g.Rz && edge_crossed(c, 10)) m |= 2u;
    if (i + 1 < g.Rx && j + 1 < g.Ry && edge_crossed(c, 5)) m |= 4u;
    return m;
}

__device__ __forceinline__ float tanh_w(const float* w, long long stride, long long f, int c, float ws) {
    return w ? __fadd_rn(__fmul_rn(tanhf(__ldg(w + f * stride + c)), ws), 1.f) : 1.f;
}
__device__ __forceinline__ float sigmoid_f(float r) { return 1.f / (1.f + expf(-r)); }
__device__ __forceinline__ float gamma_w(const FcWeights& W, long long f) {
    if (!W.gamma) return 1.f;
    const float sg = 1.f / (1.f + expf(-__ldg(W.gamma + f * W.sg)));
    return __fadd_rn(__fmul_rn(sg, W.ws), W.ws_half);
}

// ---- forward ----------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(FC_THREADS) fc_count_kernel(const float* __restrict__ s, const FcGrid g,
                                                              uint8_t* __restrict__ cases, uint32_t* __restrict__ nvd,
                                                              uint32_t* __restrict__ nl, uint32_t* __restrict__ nq,
                                                              uint32_t* __restrict__ ns) {
    const long long f = blockIdx.x * (long long)FC_THREADS + threadIdx.x;
    if (f >= g.F) return;
    int i, j, k;
    cube_ijk(g, f, i, j, k);
    uint32_t c = case_of(g, s, i, j, k);
    const bool surf = is_surface(c);
    if (surf && fc_check[c][0]) {
        const int ni = i + fc_check[c][1], nj = j + fc_check[c][2], nk = k + fc_check[c][3];
        if (ni >= 0 && nj >= 0 && nk >= 0 && ni < g.Rx && nj < g.Ry && nk < g.Rz) {
            const uint32_t cn = case_of(g, s, ni, nj, nk);
            if (is_surface(cn) && fc_check[cn][0]) c = 255u - c;
        }
    }
    cases[f] = (uint8_t)c;
    uint32_t ne = 0;
    if (surf)
        for (int e = 0; e < 12; e++) ne += edge_crossed(c, e);
    nvd[f] = surf ? fc_num_vd[c] : 0u;
    nl[f] = ne;
    nq[f] = surf ? __popc(owned_quads(g, c, i, j, k)) : 0u;
    ns[f] = surf;
}

struct EdgeEval {
    float xa[3], xb[3];
    float sa, sb, aa, ab;    // SDF and normalised alpha at the two corners
    int ca, cb;
};

__device__ __forceinline__ void load_edge(const FcGrid& g, const float* __restrict__ x, const float* __restrict__ s,
                                          const FcWeights& W, long long f, long long p0, int e, EdgeEval& E) {
    E.ca = fc_cube_edges[e][0];
    E.cb = fc_cube_edges[e][1];
    const long long pa = corner_point(g, p0, E.ca), pb = corner_point(g, p0, E.cb);
#pragma unroll
    for (int d = 0; d < 3; d++) { E.xa[d] = __ldg(x + 3 * pa + d); E.xb[d] = __ldg(x + 3 * pb + d); }
    E.sa = __ldg(s + pa);
    E.sb = __ldg(s + pb);
    E.aa = tanh_w(W.alpha, W.sa, f, E.ca, W.ws);
    E.ab = tanh_w(W.alpha, W.sa, f, E.cb, W.ws);
}

// crossing of the edge with end weights (wa, wb): (xa wb - xb wa) / (wb - wa)
__device__ __forceinline__ void crossing(const EdgeEval& E, float wa, float wb, float* o) {
    const float den = wb - wa;
#pragma unroll
    for (int d = 0; d < 3; d++) o[d] = (E.xa[d] * wb - E.xb[d] * wa) / den;
}

// dual vertex of group (c, gi) of cube f: vd = sum(beta ue) / sum(beta); also returns ue and beta per group edge
__device__ __forceinline__ int dual_vertex(const FcGrid& g, const float* __restrict__ x, const float* __restrict__ s,
                                           const FcWeights& W, long long f, long long p0, uint32_t c, int gi,
                                           EdgeEval* E, float (*ue)[3], float* beta, float* vd, float& bsum) {
    float acc[3] = {0.f, 0.f, 0.f};
    bsum = 0.f;
    int n = 0;
    for (; n < FC_MAX_GROUP_EDGES; n++) {
        const int e = fc_groups[c][gi][n];
        if (e < 0) break;
        load_edge(g, x, s, W, f, p0, e, E[n]);
        crossing(E[n], E[n].sa * E[n].aa, E[n].sb * E[n].ab, ue[n]);
        beta[n] = tanh_w(W.beta, W.sb, f, e, W.ws);
#pragma unroll
        for (int d = 0; d < 3; d++) acc[d] += beta[n] * ue[n][d];
        bsum += beta[n];
    }
#pragma unroll
    for (int d = 0; d < 3; d++) vd[d] = acc[d] / bsum;
    return n;
}

// attribute ch crossed on group edge E with the end weights (wa, wb) of its ue: (ca wb - cb wa) / (wb - wa)
__device__ __forceinline__ float attr_crossing(const FcGrid& g, const FcAttrs& A, long long p0, const EdgeEval& E,
                                               int ch, float& ca, float& cb) {
    ca = sigmoid_f(__ldg(A.a + corner_point(g, p0, E.ca) * A.stride + ch));
    cb = sigmoid_f(__ldg(A.a + corner_point(g, p0, E.cb) * A.stride + ch));
    const float wa = E.sa * E.aa, wb = E.sb * E.ab;
    return (ca * wb - cb * wa) / (wb - wa);
}

template <bool ATTRS>
__global__ void __launch_bounds__(FC_THREADS) fc_vertex_kernel(const float* __restrict__ x, const float* __restrict__ s,
                                                               const FcGrid g, const FcWeights W, const FcAttrs A,
                                                               const uint8_t* __restrict__ cases,
                                                               const uint32_t* __restrict__ voff,
                                                               const uint32_t* __restrict__ loff,
                                                               float* __restrict__ verts, float* __restrict__ ldev,
                                                               float* __restrict__ vattrs) {
    const long long f = blockIdx.x * (long long)FC_THREADS + threadIdx.x;
    if (f >= g.F) return;
    const uint32_t c = cases[f];
    if (!is_surface(c)) return;
    int i, j, k;
    cube_ijk(g, f, i, j, k);
    const long long p0 = point_id(g, i, j, k);
    uint32_t v = voff[f], l = loff[f];
    for (int gi = 0; gi < fc_num_vd[c]; gi++, v++) {
        EdgeEval E[FC_MAX_GROUP_EDGES];
        float ue[FC_MAX_GROUP_EDGES][3], beta[FC_MAX_GROUP_EDGES], vd[3], bsum;
        const int n = dual_vertex(g, x, s, W, f, p0, c, gi, E, ue, beta, vd, bsum);
#pragma unroll
        for (int d = 0; d < 3; d++) verts[3ull * v + d] = vd[d];
        float dist[FC_MAX_GROUP_EDGES], mean = 0.f;
        for (int t = 0; t < n; t++) {
            float zc[3];
            crossing(E[t], E[t].sa, E[t].sb, zc);
            const float dx = zc[0] - vd[0], dy = zc[1] - vd[1], dz = zc[2] - vd[2];
            dist[t] = sqrtf(dx * dx + dy * dy + dz * dz);
            mean += dist[t];
        }
        mean /= (float)n;
        for (int t = 0; t < n; t++) ldev[l++] = fabsf(dist[t] - mean);
        if constexpr (ATTRS) {
            for (int ch = 0; ch < A.C; ch++) {
                float acc = 0.f, ca, cb;
                for (int t = 0; t < n; t++) acc += beta[t] * attr_crossing(g, A, p0, E[t], ch, ca, cb);
                vattrs[(long long)v * A.C + ch] = acc / bsum;
            }
        }
    }
}

// the quad cube f owns along axis a: global dual vertex per slot (cubes ascending), and the cycled order
struct Quad {
    uint32_t v[4];      // dual vertex of slot t
    long long cube[4];
    int order[4];       // cycled position -> slot
};

__device__ __forceinline__ void owned_quad(const FcGrid& g, const float* __restrict__ s,
                                           const uint8_t* __restrict__ cases, const uint32_t* __restrict__ voff,
                                           int i, int j, int k, int a, Quad& Q) {
#pragma unroll
    for (int t = 0; t < 4; t++) {
        const int u = t >> 1, w = t & 1;
        const int ci = i + (a == 0 ? 0 : u), cj = j + (a == 0 ? u : (a == 1 ? 0 : w)), ck = k + (a == 2 ? 0 : w);
        const long long cf = cube_id(g, ci, cj, ck);
        Q.cube[t] = cf;
        Q.v[t] = voff[cf] + (uint32_t)fc_group_of[cases[cf]][fc_quad_edge[a][t]];
    }
    // first end of the owner's copy of the edge (edges 6, 10, 5 list it first); y edges run from +y to -y
    const int own = fc_quad_edge[a][0], c0 = fc_cube_edges[own][0];
    const bool flip = __ldg(s + corner_point(g, point_id(g, i, j, k), c0)) > 0.f;
    const int o1[4] = {0, 1, 3, 2}, o2[4] = {2, 3, 1, 0};
#pragma unroll
    for (int t = 0; t < 4; t++) Q.order[t] = flip ? o1[t] : o2[t];
}

template <bool ATTRS>
__global__ void __launch_bounds__(FC_THREADS) fc_quad_kernel(const float* __restrict__ s, const FcGrid g,
                                                             const FcWeights W, const uint8_t* __restrict__ cases,
                                                             const uint32_t* __restrict__ voff,
                                                             const uint32_t* __restrict__ qoff, uint32_t nvd,
                                                             int training, float* __restrict__ verts,
                                                             int64_t* __restrict__ faces, int C,
                                                             float* __restrict__ vattrs) {
    const long long f = blockIdx.x * (long long)FC_THREADS + threadIdx.x;
    if (f >= g.F) return;
    const uint32_t c = cases[f];
    if (!is_surface(c)) return;
    int i, j, k;
    cube_ijk(g, f, i, j, k);
    uint32_t m = owned_quads(g, c, i, j, k), q = qoff[f];
    for (int a = 0; a < 3; a++) {
        if (!((m >> a) & 1u)) continue;
        Quad Q;
        owned_quad(g, s, cases, voff, i, j, k, a, Q);
        int64_t v[4];
        float ga[4];
#pragma unroll
        for (int t = 0; t < 4; t++) { v[t] = Q.v[Q.order[t]]; ga[t] = gamma_w(W, Q.cube[Q.order[t]]); }
        const float g02 = ga[0] * ga[2], g13 = ga[1] * ga[3];
        if (!training) {
            int64_t* o = faces + 6ll * q;
            if (g02 > g13) { o[0] = v[0]; o[1] = v[1]; o[2] = v[2]; o[3] = v[0]; o[4] = v[2]; o[5] = v[3]; }
            else           { o[0] = v[0]; o[1] = v[1]; o[2] = v[3]; o[3] = v[3]; o[4] = v[1]; o[5] = v[2]; }
        } else {
            const int64_t ctr = (int64_t)nvd + q;
            const float wsum = (g02 + g13) + 1e-8f;
#pragma unroll
            for (int d = 0; d < 3; d++) {
                const float a02 = (verts[3 * v[0] + d] + verts[3 * v[2] + d]) / 2.f;
                const float a13 = (verts[3 * v[1] + d] + verts[3 * v[3] + d]) / 2.f;
                verts[3 * ctr + d] = (a02 * g02 + a13 * g13) / wsum;
            }
            if constexpr (ATTRS) {
                for (int ch = 0; ch < C; ch++) {
                    const float a02 = (vattrs[v[0] * C + ch] + vattrs[v[2] * C + ch]) / 2.f;
                    const float a13 = (vattrs[v[1] * C + ch] + vattrs[v[3] * C + ch]) / 2.f;
                    vattrs[ctr * C + ch] = (a02 * g02 + a13 * g13) / wsum;
                }
            }
            int64_t* o = faces + 12ll * q;
#pragma unroll
            for (int t = 0; t < 4; t++) { o[3 * t] = v[t]; o[3 * t + 1] = v[(t + 1) & 3]; o[3 * t + 2] = ctr; }
        }
        q++;
    }
}

// ---- backward ---------------------------------------------------------------------------------------------------

// per quad slot (cube ascending): d loss / d (its dual vertex) in xyz, d loss / d (its cube's normalised gamma) in w;
// with attributes, w also takes their terms and qh holds d centre / d (the slot's dual vertex), the same per channel
template <bool ATTRS>
__global__ void __launch_bounds__(FC_THREADS) fc_quad_bwd_kernel(const float* __restrict__ s, const FcGrid g,
                                                                 const FcWeights W, const uint8_t* __restrict__ cases,
                                                                 const uint32_t* __restrict__ voff,
                                                                 const uint32_t* __restrict__ qoff, uint32_t nvd,
                                                                 const float* __restrict__ verts,
                                                                 const float* __restrict__ gverts,
                                                                 float4* __restrict__ qpart, int C,
                                                                 const float* __restrict__ vattrs,
                                                                 const float* __restrict__ gvattrs,
                                                                 float* __restrict__ qh) {
    const long long f = blockIdx.x * (long long)FC_THREADS + threadIdx.x;
    if (f >= g.F) return;
    const uint32_t c = cases[f];
    if (!is_surface(c)) return;
    int i, j, k;
    cube_ijk(g, f, i, j, k);
    uint32_t m = owned_quads(g, c, i, j, k), q = qoff[f];
    for (int a = 0; a < 3; a++) {
        if (!((m >> a) & 1u)) continue;
        Quad Q;
        owned_quad(g, s, cases, voff, i, j, k, a, Q);
        float ga[4], P[4][3], ctr[3], gc[3];
#pragma unroll
        for (int t = 0; t < 4; t++) {
            ga[t] = gamma_w(W, Q.cube[Q.order[t]]);
#pragma unroll
            for (int d = 0; d < 3; d++) P[t][d] = verts[3ull * Q.v[Q.order[t]] + d];
        }
        const float g02 = ga[0] * ga[2], g13 = ga[1] * ga[3], wsum = (g02 + g13) + 1e-8f;
        float d02 = 0.f, d13 = 0.f;
#pragma unroll
        for (int d = 0; d < 3; d++) {
            const float a02 = (P[0][d] + P[2][d]) / 2.f, a13 = (P[1][d] + P[3][d]) / 2.f;
            ctr[d] = verts[3ull * (nvd + q) + d];
            gc[d] = gverts[3ull * (nvd + q) + d];
            d02 += gc[d] * (a02 - ctr[d]);
            d13 += gc[d] * (a13 - ctr[d]);
        }
        if constexpr (ATTRS) {
            const uint64_t V[4] = {Q.v[Q.order[0]], Q.v[Q.order[1]], Q.v[Q.order[2]], Q.v[Q.order[3]]};
            const uint64_t ci = (uint64_t)(nvd + q) * C;
            for (int ch = 0; ch < C; ch++) {
                const float a02 = (vattrs[V[0] * C + ch] + vattrs[V[2] * C + ch]) / 2.f;
                const float a13 = (vattrs[V[1] * C + ch] + vattrs[V[3] * C + ch]) / 2.f;
                const float ct = vattrs[ci + ch], gct = gvattrs[ci + ch];
                d02 += gct * (a02 - ct);
                d13 += gct * (a13 - ct);
            }
        }
        const float gg02 = d02 / wsum, gg13 = d13 / wsum;
        const float h02 = g02 / wsum / 2.f, h13 = g13 / wsum / 2.f;
        const float gg[4] = {gg02 * ga[2], gg13 * ga[3], gg02 * ga[0], gg13 * ga[1]};
#pragma unroll
        for (int t = 0; t < 4; t++) {
            const float h = (t & 1) ? h13 : h02;
            qpart[4ull * q + Q.order[t]] = make_float4(gc[0] * h, gc[1] * h, gc[2] * h, gg[t]);
            if constexpr (ATTRS) qh[4ull * q + Q.order[t]] = h;
        }
        q++;
    }
}

__device__ __forceinline__ void crossing_bwd(const float* xa, const float* xb, float wa, float wb, const float* o,
                                             const float* go, float* gxa, float* gxb, float& gwa, float& gwb) {
    const float den = wb - wa;
    float da = 0.f, db = 0.f;
#pragma unroll
    for (int d = 0; d < 3; d++) {
        gxa[d] += go[d] * (wb / den);
        gxb[d] -= go[d] * (wa / den);
        da += go[d] * (o[d] - xb[d]);
        db += go[d] * (xa[d] - o[d]);
    }
    gwa += da / den;
    gwb += db / den;
}

// the quad that cube (i,j,k)'s crossed edge e belongs to, and the cube's slot in it; false when the edge lies on the
// grid's boundary (fewer than 4 cubes, no quad)
__device__ __forceinline__ bool quad_slot(const FcGrid& g, const uint8_t* __restrict__ cases,
                                          const uint32_t* __restrict__ qoff, int i, int j, int k, int e,
                                          uint32_t& q, int& slot) {
    const int ijk[3] = {i, j, k}, R[3] = {g.Rx, g.Ry, g.Rz};
    const int a = fc_edge_axis[e], c0 = fc_cube_edges[e][0];
    const int off[3] = {c0 & 1, (c0 >> 1) & 1, c0 >> 2};
    int o[3] = {i, j, k};
    bool interior = true;
    for (int b = 0; b < 3; b++) {
        if (b == a) continue;
        const int gp = ijk[b] + off[b];
        interior &= gp >= 1 && gp <= R[b] - 1;
        o[b] = gp - 1;
    }
    if (!interior) return false;
    const long long of = cube_id(g, o[0], o[1], o[2]);
    const uint32_t om = owned_quads(g, cases[of], o[0], o[1], o[2]);
    q = qoff[of] + __popc(om & ((1u << a) - 1u));
    const int b1 = a == 0 ? 1 : 0, b2 = a == 2 ? 1 : 2;
    slot = 2 * (1 - off[b1]) + (1 - off[b2]);
    return true;
}

// attribute inputs of the cube backward: per-vertex output gradients, the quad-centre factors (training) and the
// per-corner partials of the surface cubes (NULL when no attribute gradient is wanted)
struct FcAttrGrads {
    const float* gvattrs;
    const float* qh;
    float* cattr;
};

template <bool ATTRS>
__global__ void __launch_bounds__(FC_THREADS) fc_cube_bwd_kernel(
    const float* __restrict__ x, const float* __restrict__ s, const FcGrid g, const FcWeights W,
    const uint8_t* __restrict__ cases, const uint32_t* __restrict__ voff, const uint32_t* __restrict__ loff,
    const uint32_t* __restrict__ qoff, const uint32_t* __restrict__ soff, const float* __restrict__ gverts,
    const float* __restrict__ gldev, const float4* __restrict__ qpart, float4* __restrict__ cpart,
    float* __restrict__ gbeta, float* __restrict__ galpha, float* __restrict__ ggamma, const FcAttrs A,
    const FcAttrGrads AG, uint32_t nvd) {
    const long long f = blockIdx.x * (long long)FC_THREADS + threadIdx.x;
    if (f >= g.F) return;
    const uint32_t c = cases[f];
    float gb[12], gan[8], gx[8][3], gs[8], ggam = 0.f;
#pragma unroll
    for (int t = 0; t < 12; t++) gb[t] = 0.f;
#pragma unroll
    for (int t = 0; t < 8; t++) { gan[t] = 0.f; gs[t] = 0.f; gx[t][0] = gx[t][1] = gx[t][2] = 0.f; }
    if (is_surface(c)) {
        int i, j, k;
        cube_ijk(g, f, i, j, k);
        const long long p0 = point_id(g, i, j, k);
        float* cattr = nullptr;
        if constexpr (ATTRS) {
            if (AG.cattr) {
                cattr = AG.cattr + 8ull * soff[f] * A.C;
                for (int t = 0; t < 8 * A.C; t++) cattr[t] = 0.f;
            }
        }
        uint32_t v = voff[f], l = loff[f];
        for (int gi = 0; gi < fc_num_vd[c]; gi++, v++) {
            EdgeEval E[FC_MAX_GROUP_EDGES];
            float ue[FC_MAX_GROUP_EDGES][3], beta[FC_MAX_GROUP_EDGES], vd[3], bsum;
            const int n = dual_vertex(g, x, s, W, f, p0, c, gi, E, ue, beta, vd, bsum);
            float gvd[3] = {gverts[3ull * v], gverts[3ull * v + 1], gverts[3ull * v + 2]};
            // quad-centre partials of this dual vertex, in group edge order
            if (qpart) {
                for (int t = 0; t < n; t++) {
                    uint32_t q;
                    int slot;
                    if (!quad_slot(g, cases, qoff, i, j, k, fc_groups[c][gi][t], q, slot)) continue;
                    const float4 p = qpart[4ull * q + slot];
                    gvd[0] += p.x; gvd[1] += p.y; gvd[2] += p.z;
                    ggam += p.w;
                }
            }
            // L_dev = |d_t - mean(d)|, d_t = |zc_t - vd|
            float zc[FC_MAX_GROUP_EDGES][3], dist[FC_MAX_GROUP_EDGES], mean = 0.f;
            for (int t = 0; t < n; t++) {
                crossing(E[t], E[t].sa, E[t].sb, zc[t]);
                const float dx = zc[t][0] - vd[0], dy = zc[t][1] - vd[1], dz = zc[t][2] - vd[2];
                dist[t] = sqrtf(dx * dx + dy * dy + dz * dz);
                mean += dist[t];
            }
            mean /= (float)n;
            float sg[FC_MAX_GROUP_EDGES], msum = 0.f;
            for (int t = 0; t < n; t++) {
                const float r = dist[t] - mean;
                sg[t] = gldev[l + t] * (r > 0.f ? 1.f : (r < 0.f ? -1.f : 0.f));
                msum += sg[t];
            }
            msum /= (float)n;
            for (int t = 0; t < n; t++) {
                const float gd = sg[t] - msum;
                float gz[3] = {0.f, 0.f, 0.f};
                if (dist[t] > 0.f) {
#pragma unroll
                    for (int d = 0; d < 3; d++) {
                        gz[d] = gd * (zc[t][d] - vd[d]) / dist[t];
                        gvd[d] -= gz[d];
                    }
                }
                float gsa = 0.f, gsb = 0.f;
                crossing_bwd(E[t].xa, E[t].xb, E[t].sa, E[t].sb, zc[t], gz, gx[E[t].ca], gx[E[t].cb], gsa, gsb);
                gs[E[t].ca] += gsa;
                gs[E[t].cb] += gsb;
            }
            l += n;
            // vd = sum(beta ue) / sum(beta)
            for (int t = 0; t < n; t++) {
                const int e = fc_groups[c][gi][t];
                float gu[3], gbt = 0.f;
#pragma unroll
                for (int d = 0; d < 3; d++) {
                    gu[d] = gvd[d] * beta[t] / bsum;
                    gbt += gvd[d] * (ue[t][d] - vd[d]);
                }
                gb[e] += gbt / bsum;
                float gwa = 0.f, gwb = 0.f;
                crossing_bwd(E[t].xa, E[t].xb, E[t].sa * E[t].aa, E[t].sb * E[t].ab, ue[t], gu, gx[E[t].ca],
                             gx[E[t].cb], gwa, gwb);
                gs[E[t].ca] += gwa * E[t].aa;
                gs[E[t].cb] += gwb * E[t].ab;
                gan[E[t].ca] += gwa * E[t].sa;
                gan[E[t].cb] += gwb * E[t].sb;
            }
            // attributes, after the geometry: va = sum(beta uc) / sum(beta), uc the crossing of sigmoid(raw) with
            // the end weights of ue; the vertex's gradient takes its quad-centre terms in group edge order
            if constexpr (ATTRS) {
                long long qslot[FC_MAX_GROUP_EDGES], qctr[FC_MAX_GROUP_EDGES];
                for (int t = 0; t < n; t++) {
                    uint32_t q;
                    int slot;
                    const bool in = AG.qh && quad_slot(g, cases, qoff, i, j, k, fc_groups[c][gi][t], q, slot);
                    qslot[t] = in ? 4ll * q + slot : -1;
                    qctr[t] = in ? ((long long)nvd + q) * A.C : 0;
                }
                for (int ch = 0; ch < A.C; ch++) {
                    float gva = AG.gvattrs[(long long)v * A.C + ch];
                    for (int t = 0; t < n; t++)
                        if (qslot[t] >= 0) gva += AG.qh[qslot[t]] * AG.gvattrs[qctr[t] + ch];
                    float uc[FC_MAX_GROUP_EDGES], ca[FC_MAX_GROUP_EDGES], cb[FC_MAX_GROUP_EDGES], acc = 0.f;
                    for (int t = 0; t < n; t++) {
                        uc[t] = attr_crossing(g, A, p0, E[t], ch, ca[t], cb[t]);
                        acc += beta[t] * uc[t];
                    }
                    const float va = acc / bsum;
                    for (int t = 0; t < n; t++) {
                        gb[fc_groups[c][gi][t]] += gva * (uc[t] - va) / bsum;
                        const float gu = gva * beta[t] / bsum;
                        const float wa = E[t].sa * E[t].aa, wb = E[t].sb * E[t].ab, den = wb - wa;
                        const float gwa = gu * (uc[t] - cb[t]) / den, gwb = gu * (ca[t] - uc[t]) / den;
                        gs[E[t].ca] += gwa * E[t].aa;
                        gs[E[t].cb] += gwb * E[t].ab;
                        gan[E[t].ca] += gwa * E[t].sa;
                        gan[E[t].cb] += gwb * E[t].sb;
                        if (cattr) {
                            cattr[E[t].ca * A.C + ch] += gu * (wb / den);
                            cattr[E[t].cb * A.C + ch] -= gu * (wa / den);
                        }
                    }
                }
            }
        }
        if (cpart) {
            float4* o = cpart + 8ull * soff[f];
#pragma unroll
            for (int t = 0; t < 8; t++) o[t] = make_float4(gx[t][0], gx[t][1], gx[t][2], gs[t]);
        }
    }
    // raw weights: d tanh(r) ws + 1 = ws (1 - tanh^2); d sigmoid(r) ws + h = ws sig (1 - sig)
    if (gbeta)
        for (int e = 0; e < 12; e++) {
            const float th = tanhf(__ldg(W.beta + f * W.sb + e));
            gbeta[12 * f + e] = gb[e] * W.ws * (1.f - th * th);
        }
    if (galpha)
        for (int q = 0; q < 8; q++) {
            const float th = tanhf(__ldg(W.alpha + f * W.sa + q));
            galpha[8 * f + q] = gan[q] * W.ws * (1.f - th * th);
        }
    if (ggamma) {
        const float sgm = 1.f / (1.f + expf(-__ldg(W.gamma + f * W.sg)));
        ggamma[f] = ggam * W.ws * (sgm * (1.f - sgm));
    }
}

// per grid point: the corner partials of its (up to) 8 cubes, cube offsets (dx, dy, dz) in corner order
// (with attributes, the same for their per-corner partials, times the sigmoid's derivative at the point)
template <bool ATTRS>
__global__ void __launch_bounds__(FC_THREADS) fc_point_bwd_kernel(const FcGrid g, const uint8_t* __restrict__ cases,
                                                                  const uint32_t* __restrict__ soff,
                                                                  const float4* __restrict__ cpart, long long npts,
                                                                  float* __restrict__ gx, float* __restrict__ gs,
                                                                  const FcAttrs A, const float* __restrict__ cattr,
                                                                  float* __restrict__ gattr) {
    const long long p = blockIdx.x * (long long)FC_THREADS + threadIdx.x;
    if (p >= npts) return;
    const int k = (int)(p % g.Sz), j = (int)((p / g.Sz) % (g.Ry + 1)), i = (int)(p / g.Syz);
    float ax = 0.f, ay = 0.f, az = 0.f, as = 0.f;
#pragma unroll
    for (int c = 0; c < 8; c++) {
        const int ci = i - (c & 1), cj = j - ((c >> 1) & 1), ck = k - (c >> 2);
        if (ci < 0 || cj < 0 || ck < 0 || ci >= g.Rx || cj >= g.Ry || ck >= g.Rz) continue;
        const long long f = cube_id(g, ci, cj, ck);
        if (!is_surface(cases[f])) continue;
        const float4 v = cpart[8ull * soff[f] + c];
        ax += v.x; ay += v.y; az += v.z; as += v.w;
    }
    if (gx) { gx[3 * p] = ax; gx[3 * p + 1] = ay; gx[3 * p + 2] = az; }
    if (gs) gs[p] = as;
    if constexpr (ATTRS) {
        if (!gattr) return;
        long long base[8];
#pragma unroll
        for (int c = 0; c < 8; c++) {
            const int ci = i - (c & 1), cj = j - ((c >> 1) & 1), ck = k - (c >> 2);
            base[c] = -1;
            if (ci < 0 || cj < 0 || ck < 0 || ci >= g.Rx || cj >= g.Ry || ck >= g.Rz) continue;
            const long long f = cube_id(g, ci, cj, ck);
            if (is_surface(cases[f])) base[c] = (8ll * soff[f] + c) * A.C;
        }
        for (int ch = 0; ch < A.C; ch++) {
            float acc = 0.f;
#pragma unroll
            for (int c = 0; c < 8; c++)
                if (base[c] >= 0) acc += cattr[base[c] + ch];
            const float sg = sigmoid_f(__ldg(A.a + p * A.stride + ch));
            gattr[p * A.C + ch] = acc * (sg * (1.f - sg));
        }
    }
}

inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// scratch: cases (u8), then counts and offsets of dual vertices, L_dev entries, quads, surface cubes (u32 each)
struct FcScratch {
    uint8_t* cases;
    uint32_t *cnt[4], *off[4];
    void* scan;
};

FcScratch fc_scratch(void* base, long long F) {
    FcScratch S;
    char* p = (char*)base;
    S.cases = (uint8_t*)p;
    p += align256((size_t)F);
    for (int t = 0; t < 4; t++) { S.cnt[t] = (uint32_t*)p; p += align256((size_t)F * 4); }
    for (int t = 0; t < 4; t++) { S.off[t] = (uint32_t*)p; p += align256((size_t)F * 4); }
    S.scan = p;
    return S;
}

bool fc_dims_ok(int Rx, int Ry, int Rz) {
    return Rx >= 1 && Ry >= 1 && Rz >= 1 && (long long)(Rx + 1) * (Ry + 1) * (Rz + 1) < (1ll << 31);
}

FcGrid fc_grid(int Rx, int Ry, int Rz) {
    return FcGrid{Rx, Ry, Rz, Rz + 1, (long long)(Ry + 1) * (Rz + 1), (long long)Rx * Ry * Rz};
}

FcWeights fc_weights(const float* beta, int64_t sb, const float* alpha, int64_t sa, const float* gamma, int64_t sg,
                     double ws) {
    return FcWeights{beta, sb, alpha, sa, gamma, sg, (float)ws, (float)((1.0 - ws) / 2)};
}

inline unsigned fc_blocks(long long n) { return (unsigned)((n + FC_THREADS - 1) / FC_THREADS); }

// backward workspace: quad-centre partials (training), per-corner partials of the surface cubes, then with attributes
// the quad-centre factors (training) and the per-corner attribute partials
struct FcWork {
    size_t qpart, cpart, qh, cattr, total;
};

FcWork fc_work(const unsigned long long* totals_host4, int training, int C) {
    const unsigned long long nq = training ? totals_host4[2] : 0, ns = totals_host4[3];
    FcWork w;
    w.qpart = 0;
    w.cpart = align256(4 * nq * sizeof(float4));
    if (!C) {
        w.qh = w.cattr = w.total = w.cpart + 8 * ns * sizeof(float4);
        return w;
    }
    w.qh = w.cpart + align256(8 * ns * sizeof(float4));
    w.cattr = w.qh + align256(4 * nq * sizeof(float));
    w.total = w.cattr + 8 * ns * C * sizeof(float);
    return w;
}

bool fc_attrs_ok(const char* fn, const float* attrs, int64_t stride, int32_t C) {
    if (!attrs) { gs_set_error("%s: NULL attributes", fn); return false; }
    if (C < 1 || stride < C) {
        gs_set_error("%s: %d attribute channels with row stride %lld: need C >= 1 and stride >= C", fn, C,
                     (long long)stride);
        return false;
    }
    return true;
}

int32_t fc_write(const float* x, const float* s, const FcWeights& W, int32_t Rx, int32_t Ry, int32_t Rz,
                 int32_t training, const unsigned long long* totals_host4, float* verts, int64_t* faces, float* ldev,
                 const FcAttrs& A, float* vattrs, void* scratch, cudaStream_t st) {
    const char* fn = A.C ? "flexicubes_write_attrs" : "flexicubes_write";
    if (!fc_dims_ok(Rx, Ry, Rz)) { gs_set_error("%s: unsupported grid %dx%dx%d", fn, Rx, Ry, Rz); return 1; }
    if (!totals_host4) { gs_set_error("%s: NULL totals", fn); return 1; }
    const unsigned long long nvd = totals_host4[0], nq = totals_host4[2];
    if (nvd + nq >= (1ull << 31)) { gs_set_error("flexicubes: %llu vertices: too many", nvd + nq); return 1; }
    if (nvd == 0) return 0;
    if (!x || !s || !scratch || !verts || !ldev || (nq && !faces) || (A.C && !vattrs)) {
        gs_set_error("%s: NULL pointer", fn);
        return 1;
    }
    const FcGrid g = fc_grid(Rx, Ry, Rz);
    FcScratch S = fc_scratch(scratch, g.F);
    if (A.C)
        fc_vertex_kernel<true><<<fc_blocks(g.F), FC_THREADS, 0, st>>>(x, s, g, W, A, S.cases, S.off[0], S.off[1],
                                                                      verts, ldev, vattrs);
    else
        fc_vertex_kernel<false><<<fc_blocks(g.F), FC_THREADS, 0, st>>>(x, s, g, W, A, S.cases, S.off[0], S.off[1],
                                                                       verts, ldev, nullptr);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    if (nq) {
        if (A.C)
            fc_quad_kernel<true><<<fc_blocks(g.F), FC_THREADS, 0, st>>>(s, g, W, S.cases, S.off[0], S.off[2],
                                                                        (uint32_t)nvd, training, verts, faces, A.C,
                                                                        vattrs);
        else
            fc_quad_kernel<false><<<fc_blocks(g.F), FC_THREADS, 0, st>>>(s, g, W, S.cases, S.off[0], S.off[2],
                                                                         (uint32_t)nvd, training, verts, faces, 0,
                                                                         nullptr);
        gs_count_launches(1);
        GS_CUDA_CHECK(cudaGetLastError());
    }
    return 0;
}

int32_t fc_backward(const float* x, const float* s, const FcWeights& W, int32_t Rx, int32_t Ry, int32_t Rz,
                    int32_t training, const unsigned long long* totals_host4, const float* verts,
                    const float* grad_verts, const float* grad_ldev, float* grad_x, float* grad_s, float* grad_beta,
                    float* grad_alpha, float* grad_gamma, const FcAttrs& A, const float* vattrs,
                    const float* grad_vattrs, float* grad_attrs, void* scratch, void* workspace, cudaStream_t st) {
    const char* fn = A.C ? "flexicubes_backward_attrs" : "flexicubes_backward";
    if (!fc_dims_ok(Rx, Ry, Rz)) { gs_set_error("%s: unsupported grid %dx%dx%d", fn, Rx, Ry, Rz); return 1; }
    if (!totals_host4 || !x || !s || !scratch) { gs_set_error("%s: NULL pointer", fn); return 1; }
    if ((grad_beta && !W.beta) || (grad_alpha && !W.alpha) || (grad_gamma && !W.gamma)) {
        gs_set_error("%s: a weight gradient needs its weight", fn);
        return 1;
    }
    const unsigned long long nvd = totals_host4[0], nq = totals_host4[2];
    const FcGrid g = fc_grid(Rx, Ry, Rz);
    const long long npts = (long long)(Rx + 1) * (Ry + 1) * (Rz + 1);
    if (nvd == 0) {   // empty mesh: every gradient is zero
        if (grad_x) GS_CUDA_CHECK(cudaMemsetAsync(grad_x, 0, 12 * npts, st));
        if (grad_s) GS_CUDA_CHECK(cudaMemsetAsync(grad_s, 0, 4 * npts, st));
        if (grad_beta) GS_CUDA_CHECK(cudaMemsetAsync(grad_beta, 0, 48 * g.F, st));
        if (grad_alpha) GS_CUDA_CHECK(cudaMemsetAsync(grad_alpha, 0, 32 * g.F, st));
        if (grad_gamma) GS_CUDA_CHECK(cudaMemsetAsync(grad_gamma, 0, 4 * g.F, st));
        if (grad_attrs) GS_CUDA_CHECK(cudaMemsetAsync(grad_attrs, 0, 4 * npts * A.C, st));
        return 0;
    }
    if (!verts || !grad_verts || !grad_ldev || !workspace || (A.C && (!vattrs || !grad_vattrs))) {
        gs_set_error("%s: NULL pointer", fn);
        return 1;
    }
    FcScratch S = fc_scratch(scratch, g.F);
    const FcWork L = fc_work(totals_host4, training, A.C);
    char* w = (char*)workspace;
    float4* qpart = (training && nq) ? (float4*)(w + L.qpart) : nullptr;
    float4* cpart = (grad_x || grad_s || grad_attrs) ? (float4*)(w + L.cpart) : nullptr;
    const FcAttrGrads AG{grad_vattrs, qpart && A.C ? (const float*)(w + L.qh) : nullptr,
                         grad_attrs ? (float*)(w + L.cattr) : nullptr};
    if (qpart) {
        if (A.C)
            fc_quad_bwd_kernel<true><<<fc_blocks(g.F), FC_THREADS, 0, st>>>(
                s, g, W, S.cases, S.off[0], S.off[2], (uint32_t)nvd, verts, grad_verts, qpart, A.C, vattrs,
                grad_vattrs, (float*)AG.qh);
        else
            fc_quad_bwd_kernel<false><<<fc_blocks(g.F), FC_THREADS, 0, st>>>(
                s, g, W, S.cases, S.off[0], S.off[2], (uint32_t)nvd, verts, grad_verts, qpart, 0, nullptr, nullptr,
                nullptr);
        gs_count_launches(1);
        GS_CUDA_CHECK(cudaGetLastError());
    }
    if (A.C)
        fc_cube_bwd_kernel<true><<<fc_blocks(g.F), FC_THREADS, 0, st>>>(
            x, s, g, W, S.cases, S.off[0], S.off[1], S.off[2], S.off[3], grad_verts, grad_ldev, qpart, cpart,
            grad_beta, grad_alpha, grad_gamma, A, AG, (uint32_t)nvd);
    else
        fc_cube_bwd_kernel<false><<<fc_blocks(g.F), FC_THREADS, 0, st>>>(
            x, s, g, W, S.cases, S.off[0], S.off[1], S.off[2], S.off[3], grad_verts, grad_ldev, qpart, cpart,
            grad_beta, grad_alpha, grad_gamma, A, AG, (uint32_t)nvd);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    if (cpart) {
        if (A.C)
            fc_point_bwd_kernel<true><<<fc_blocks(npts), FC_THREADS, 0, st>>>(g, S.cases, S.off[3], cpart, npts,
                                                                              grad_x, grad_s, A, AG.cattr,
                                                                              grad_attrs);
        else
            fc_point_bwd_kernel<false><<<fc_blocks(npts), FC_THREADS, 0, st>>>(g, S.cases, S.off[3], cpart, npts,
                                                                               grad_x, grad_s, A, nullptr, nullptr);
        gs_count_launches(1);
        GS_CUDA_CHECK(cudaGetLastError());
    }
    return 0;
}

}  // namespace

extern "C" {

size_t ngp_b200_flexicubes_scratch_bytes(int32_t Rx, int32_t Ry, int32_t Rz) {
    if (!fc_dims_ok(Rx, Ry, Rz)) return 0;
    const long long F = (long long)Rx * Ry * Rz;
    return align256((size_t)F) + 8 * align256((size_t)F * 4) + gs_scan_scratch_bytes(F);
}

int32_t ngp_b200_flexicubes_count(const float* s, int32_t Rx, int32_t Ry, int32_t Rz,
                                  unsigned long long* totals_dev4, void* scratch, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (!fc_dims_ok(Rx, Ry, Rz)) { gs_set_error("flexicubes_count: unsupported grid %dx%dx%d", Rx, Ry, Rz); return 1; }
    if (!s || !totals_dev4 || !scratch) { gs_set_error("flexicubes_count: NULL pointer"); return 1; }
    const FcGrid g = fc_grid(Rx, Ry, Rz);
    FcScratch S = fc_scratch(scratch, g.F);
    fc_count_kernel<<<fc_blocks(g.F), FC_THREADS, 0, st>>>(s, g, S.cases, S.cnt[0], S.cnt[1], S.cnt[2], S.cnt[3]);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    for (int t = 0; t < 4; t++)
        if (gs_scan_gather_u32(S.cnt[t], nullptr, S.off[t], totals_dev4 + t, g.F, S.scan, st)) return 1;
    return 0;
}

int32_t ngp_b200_flexicubes_write(const float* x, const float* s, const float* beta, int64_t beta_stride,
                                  const float* alpha, int64_t alpha_stride, const float* gamma, int64_t gamma_stride,
                                  int32_t Rx, int32_t Ry, int32_t Rz, double weight_scale, int32_t training,
                                  const unsigned long long* totals_host4, float* verts, int64_t* faces, float* ldev,
                                  void* scratch, void* stream) {
    return fc_write(x, s, fc_weights(beta, beta_stride, alpha, alpha_stride, gamma, gamma_stride, weight_scale), Rx,
                    Ry, Rz, training, totals_host4, verts, faces, ldev, FcAttrs{nullptr, 0, 0}, nullptr, scratch,
                    (cudaStream_t)stream);
}

int32_t ngp_b200_flexicubes_write_attrs(const float* x, const float* s, const float* beta, int64_t beta_stride,
                                        const float* alpha, int64_t alpha_stride, const float* gamma,
                                        int64_t gamma_stride, int32_t Rx, int32_t Ry, int32_t Rz, double weight_scale,
                                        int32_t training, const unsigned long long* totals_host4, float* verts,
                                        int64_t* faces, float* ldev, const float* attrs, int64_t attr_row_stride,
                                        int32_t C, float* vattrs, void* scratch, void* stream) {
    if (!fc_attrs_ok("flexicubes_write_attrs", attrs, attr_row_stride, C)) return 1;
    return fc_write(x, s, fc_weights(beta, beta_stride, alpha, alpha_stride, gamma, gamma_stride, weight_scale), Rx,
                    Ry, Rz, training, totals_host4, verts, faces, ldev, FcAttrs{attrs, attr_row_stride, C}, vattrs,
                    scratch, (cudaStream_t)stream);
}

size_t ngp_b200_flexicubes_backward_workspace_bytes(const unsigned long long* totals_host4, int32_t training) {
    if (!totals_host4) return 0;
    return fc_work(totals_host4, training, 0).total;
}

size_t ngp_b200_flexicubes_backward_attrs_workspace_bytes(const unsigned long long* totals_host4, int32_t training,
                                                          int32_t C) {
    if (!totals_host4 || C < 1) return 0;
    return fc_work(totals_host4, training, C).total;
}

int32_t ngp_b200_flexicubes_backward(const float* x, const float* s, const float* beta, int64_t beta_stride,
                                     const float* alpha, int64_t alpha_stride, const float* gamma,
                                     int64_t gamma_stride, int32_t Rx, int32_t Ry, int32_t Rz, double weight_scale,
                                     int32_t training, const unsigned long long* totals_host4, const float* verts,
                                     const float* grad_verts, const float* grad_ldev, float* grad_x, float* grad_s,
                                     float* grad_beta, float* grad_alpha, float* grad_gamma, void* scratch,
                                     void* workspace, void* stream) {
    return fc_backward(x, s, fc_weights(beta, beta_stride, alpha, alpha_stride, gamma, gamma_stride, weight_scale),
                       Rx, Ry, Rz, training, totals_host4, verts, grad_verts, grad_ldev, grad_x, grad_s, grad_beta,
                       grad_alpha, grad_gamma, FcAttrs{nullptr, 0, 0}, nullptr, nullptr, nullptr, scratch, workspace,
                       (cudaStream_t)stream);
}

int32_t ngp_b200_flexicubes_backward_attrs(const float* x, const float* s, const float* beta, int64_t beta_stride,
                                           const float* alpha, int64_t alpha_stride, const float* gamma,
                                           int64_t gamma_stride, int32_t Rx, int32_t Ry, int32_t Rz,
                                           double weight_scale, int32_t training,
                                           const unsigned long long* totals_host4, const float* verts,
                                           const float* grad_verts, const float* grad_ldev, float* grad_x,
                                           float* grad_s, float* grad_beta, float* grad_alpha, float* grad_gamma,
                                           const float* attrs, int64_t attr_row_stride, int32_t C,
                                           const float* vattrs, const float* grad_vattrs, float* grad_attrs,
                                           void* scratch, void* workspace, void* stream) {
    if (!fc_attrs_ok("flexicubes_backward_attrs", attrs, attr_row_stride, C)) return 1;
    return fc_backward(x, s, fc_weights(beta, beta_stride, alpha, alpha_stride, gamma, gamma_stride, weight_scale),
                       Rx, Ry, Rz, training, totals_host4, verts, grad_verts, grad_ldev, grad_x, grad_s, grad_beta,
                       grad_alpha, grad_gamma, FcAttrs{attrs, attr_row_stride, C}, vattrs, grad_vattrs, grad_attrs,
                       scratch, workspace, (cudaStream_t)stream);
}

}  // extern "C"
