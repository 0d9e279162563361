// Tile compositing: front-to-back alpha blend (forward) and its back-to-front
// replay (backward).
//
// Replaces renderCUDA (forward.cu / backward.cu) of diff_gaussian_rasterization,
// semantics per SURVEY.md App. A.1.6:  alpha = min(0.99, o*exp(power)); skip
// power>0 or alpha<1/255; stop WITHOUT blending when T(1-alpha) < 1e-4;
// color = C + T*bg, depth = sum(depth*alpha*T), alpha_out = sum(alpha*T).
//
// Design — both kernels are meant to be instruction-issue bound, not HBM bound
// (48 B splat records, gathered through L2), so everything here is about
// issuing fewer instructions per (pixel, splat):
//  * one CTA per 16x16 tile, 8 warps, each warp owns an 8x4 pixel sub-rect;
//  * a batch of 256 records (3 x LDG.128 each) is staged in shared memory as
//    48 B AoS; while staging, the loading thread computes for its splat an 8-bit
//    mask "can reach alpha >= 1/255 inside warp w's sub-rect" from the exact
//    minimum of the quadratic form over the rectangle (+ slack), so each warp
//    only walks the ~11 % of (warp, splat) pairs that can touch its 32 pixels.
//    Results are unchanged: a skipped splat fails the per-pixel alpha test on
//    every lane anyway;
//  * the record holds the conic pre-scaled to log2 units (a' = -0.5*log2e*A,
//    b' = -log2e*B, c' = -0.5*log2e*C) so power is 2 FMUL + 2 FFMA + 1 FMUL and
//    exp is a bare ex2.approx (MUFU.EX2);
//  * backward: per-pixel partials are raw moment sums (sum w dx, sum w dx dx ...,
//    w = dL/dG * G) — the constant factors and the conic multiplications move to
//    the per-Gaussian preprocess backward; the 10 sums are reduced over the 32
//    lanes with a TRANSPOSE butterfly (12 SHFL instead of 50) that leaves each
//    total in its own lane, so ONE red.global.add instruction with 10 active
//    lanes updates the fp64 gradient record.
#include "gs_common.cuh"
#include <stdlib.h>

namespace {

constexpr int RB = 256;   // threads per CTA == splats per batch
constexpr float ALPHA_MIN = 1.0f / 255.0f;
constexpr uint32_t REC_BYTES = 48;

__device__ __forceinline__ float4 lds128(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, float4 v) {
    asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// power in log2 units from the pre-scaled conic; identical code in forward and
// backward so both make the same skip decisions.
__device__ __forceinline__ float power2_of(const float4 c, float dx, float dy) {
    float t = c.x * dx;
    t = fmaf(c.y, dy, t);
    float p = t * dx;
    return fmaf(c.z * dy, dy, p);
}

// 8-bit mask over the CTA's warps: bit w set if the splat may contribute in
// sub-rect w (x in [ox+8*(w&1), +7], y in [oy+4*(w>>1), +3]).
__device__ __forceinline__ uint32_t subrect_mask(const float4 g, const float4 c, int ox, int oy) {
    const float o = c.w;
    if (!(o * 255.0f >= 1.0f) || __float_as_int(g.w) <= 0) return 0u;   // can never reach 1/255 (also NaN)
    // contributes iff q(u) = 0.5(A u_x^2 + C u_y^2) + B u_x u_y <= tau (log2 units); slack covers fp32 rounding
    const float tau = __log2f(o * 255.0f) * 1.001f + 0.03f;
    const float A = -2.0f * c.x, B = -c.y, C = -2.0f * c.z;
    if (!(A > 0.f && A * C - B * B > 0.f)) return 0xFFu;   // not positive definite: no culling, per-pixel test decides
    const float invA = 1.0f / A, invC = 1.0f / C;
    uint32_t mask = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) {
        const float ux0 = (float)(ox + 8 * (w & 1)) - g.x, ux1 = ux0 + 7.0f;
        const float uy0 = (float)(oy + 4 * (w >> 1)) - g.y, uy1 = uy0 + 3.0f;
        const bool outx = (ux0 > 0.f) || (ux1 < 0.f);
        const bool outy = (uy0 > 0.f) || (uy1 < 0.f);
        float q = 0.f;
        if (outx || outy) {
            q = 3.0e38f;
            if (outx) {
                const float ue = (ux0 > 0.f) ? ux0 : ux1;
                const float uy = fminf(fmaxf(-B * ue * invC, uy0), uy1);
                q = 0.5f * (A * ue * ue + C * uy * uy) + B * ue * uy;
            }
            if (outy) {
                const float ue = (uy0 > 0.f) ? uy0 : uy1;
                const float ux = fminf(fmaxf(-B * ue * invA, ux0), ux1);
                q = fminf(q, 0.5f * (A * ux * ux + C * ue * ue) + B * ux * ue);
            }
        }
        if (!(q > tau)) mask |= 1u << w;    // NaN -> keep (conservative)
    }
    return mask;
}

// stage one batch: thread t loads record of list position (first + t)
__device__ __forceinline__ uint32_t stage_record(const SplatRec* __restrict__ recs, uint32_t id, uint32_t s_rec,
                                                 int tid, int ox, int oy) {
    const float4 g = __ldg(&recs[id].g), c = __ldg(&recs[id].c), k = __ldg(&recs[id].k);
    const uint32_t a = s_rec + tid * REC_BYTES;
    sts128(a, g); sts128(a + 16, c); sts128(a + 32, k);
    return subrect_mask(g, c, ox, oy);
}

__global__ void __launch_bounds__(RB)
render_forward_kernel(ViewArgs va, const SplatRec* __restrict__ recs, const uint32_t* __restrict__ point_list,
                      const uint32_t* __restrict__ ranges, float* __restrict__ out_color,
                      float* __restrict__ out_depth, float* __restrict__ out_alpha,
                      uint32_t* __restrict__ n_contrib, float* __restrict__ final_T) {
    __shared__ __align__(16) unsigned char s_rec_raw[RB * REC_BYTES];
    __shared__ uint32_t s_mask[RB];
    const uint32_t s_rec = (uint32_t)__cvta_generic_to_shared(s_rec_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ox = blockIdx.x * GS_TILE, oy = blockIdx.y * GS_TILE;
    const int px = ox + 8 * (warp & 1) + (lane & 7);
    const int py = oy + 4 * (warp >> 1) + (lane >> 3);
    const bool inside = px < va.W && py < va.H;
    const float pxf = (float)px, pyf = (float)py;
    const int tile = blockIdx.y * va.tiles_x + blockIdx.x;
    const uint32_t start = ranges[2 * tile], end = ranges[2 * tile + 1];

    float T = 1.f, C0 = 0.f, C1 = 0.f, C2 = 0.f, D = 0.f, Aacc = 0.f;
    uint32_t last = 0;
    bool done = !inside;

    for (uint32_t base = start; base < end; base += RB) {
        if (__syncthreads_count(done) == RB) break;
        const int n = min((uint32_t)RB, end - base);
        if (tid < n) s_mask[tid] = stage_record(recs, __ldg(point_list + base + tid), s_rec, tid, ox, oy);
        __syncthreads();
        const uint32_t pos0 = base - start + 1;
        for (int k0 = 0; k0 < n; k0 += 32) {
            const uint32_t mine = (k0 + lane < n) ? ((s_mask[k0 + lane] >> warp) & 1u) : 0u;
            uint32_t bal = __ballot_sync(0xFFFFFFFFu, mine);
            while (bal) {
                const int j = k0 + __ffs(bal) - 1;
                bal &= bal - 1;
                const uint32_t ra = s_rec + j * REC_BYTES;
                const float4 g = lds128(ra), c = lds128(ra + 16);
                const float dx = g.x - pxf, dy = g.y - pyf;
                const float p2 = power2_of(c, dx, dy);
                const float alpha = fminf(0.99f, c.w * ex2_approx(p2));
                if (done || !(p2 <= 0.f) || alpha < ALPHA_MIN) continue;
                const float test_T = T * (1.f - alpha);
                if (test_T < 0.0001f) { done = true; continue; }
                const float4 k = lds128(ra + 32);
                const float w = alpha * T;
                C0 = fmaf(k.x, w, C0); C1 = fmaf(k.y, w, C1); C2 = fmaf(k.z, w, C2);
                D = fmaf(g.z, w, D); Aacc += w;
                T = test_T;
                last = pos0 + j;
            }
            if (__all_sync(0xFFFFFFFFu, done)) break;
        }
    }
    if (inside) {
        const size_t pix = (size_t)py * va.W + px;
        const size_t plane = (size_t)va.W * va.H;
        const float bg0 = __ldg(va.bg), bg1 = __ldg(va.bg + 1), bg2 = __ldg(va.bg + 2);
        out_color[pix] = C0 + T * bg0;
        out_color[plane + pix] = C1 + T * bg1;
        out_color[2 * plane + pix] = C2 + T * bg2;
        out_depth[pix] = D;
        out_alpha[pix] = Aacc;
        n_contrib[pix] = last;
        final_T[pix] = T;
    }
}

// One butterfly stage of the transpose reduction: lanes whose `bit` is clear keep
// a (and receive the partner's a), lanes whose bit is set keep b.
__device__ __forceinline__ float xstage(float a, float b, bool hi, int m) {
    const float send = hi ? a : b;
    const float keep = hi ? b : a;
    return keep + __shfl_xor_sync(0xFFFFFFFFu, send, m);
}

template <int MINB>
__global__ void __launch_bounds__(RB, MINB)
render_backward_kernel(ViewArgs va, const SplatRec* __restrict__ recs, const uint32_t* __restrict__ point_list,
                       const uint32_t* __restrict__ ranges, const uint32_t* __restrict__ n_contrib,
                       const float* __restrict__ final_T, const float* __restrict__ dL_dcolor,
                       const float* __restrict__ dL_ddepth, const float* __restrict__ dL_dalpha,
                       SplatGrad* __restrict__ sg) {
    __shared__ __align__(16) unsigned char s_rec_raw[RB * REC_BYTES];
    __shared__ uint32_t s_mask[RB], s_id[RB];
    __shared__ uint32_t s_max;
    const uint32_t s_rec = (uint32_t)__cvta_generic_to_shared(s_rec_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ox = blockIdx.x * GS_TILE, oy = blockIdx.y * GS_TILE;
    const int px = ox + 8 * (warp & 1) + (lane & 7);
    const int py = oy + 4 * (warp >> 1) + (lane >> 3);
    const bool inside = px < va.W && py < va.H;
    const float pxf = (float)px, pyf = (float)py;
    const int tile = blockIdx.y * va.tiles_x + blockIdx.x;
    const uint32_t start = ranges[2 * tile], end = ranges[2 * tile + 1];
    if (end <= start) return;

    const size_t pix = (size_t)py * va.W + px;
    const size_t plane = (size_t)va.W * va.H;
    const float T_final = inside ? final_T[pix] : 0.f;
    const uint32_t last_contrib = inside ? n_contrib[pix] : 0u;
    float gC0 = 0.f, gC1 = 0.f, gC2 = 0.f, gD = 0.f, gA = 0.f;
    if (inside) {
        gC0 = dL_dcolor[pix]; gC1 = dL_dcolor[plane + pix]; gC2 = dL_dcolor[2 * plane + pix];
        gD = dL_ddepth[pix]; gA = dL_dalpha[pix];
    }
    const float bgT = -T_final * (__ldg(va.bg) * gC0 + __ldg(va.bg + 1) * gC1 + __ldg(va.bg + 2) * gC2);

    // transpose-reduction lane roles: value index held by this lane after the 5 stages
    const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4, h2 = lane & 2;
    const int sub = (h8 ? 3 : 0) + (h4 ? 2 : 0) + (h2 ? 1 : 0);
    const bool my_valid = !(lane & 1) && !(h8 && h4) && !(!h8 && h4 && h2);
    const int vi = (h16 ? 5 : 0) + sub;                       // 0..9
    const int my_off = vi + (vi >= 3);                        // element offset inside SplatGrad (skips g.w)

    if (tid == 0) s_max = 0;
    __syncthreads();
    uint32_t wmax = last_contrib;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xFFFFFFFFu, wmax, o));
    if (lane == 0 && wmax) atomicMax(&s_max, wmax);
    __syncthreads();
    const uint32_t nproc = s_max;        // only list positions 1..nproc were blended by some pixel of the tile
    if (nproc == 0) return;

    float T = T_final;
    // Upstream gradients are per-pixel constants and the blend is linear in the channels, so the five
    // "colour behind this splat" recurrences (r,g,b,depth,alpha) of the package collapse into ONE on the
    // projected scalar s_j = gC.rgb_j + gD*depth_j + gA:  dL/dalpha_j = T_j * (s_j - behind_j) + bg term.
    float behind = 0.f, last_alpha = 0.f, last_s = 0.f;

    // batches from the back: a batch covers 0-based list positions [lo, hi)
    for (int hi = (int)nproc; hi > 0; hi -= RB) {
        const int lo = max(0, hi - RB);
        const int n = hi - lo;
        __syncthreads();
        if (tid < n) {
            const uint32_t id = __ldg(point_list + start + lo + tid);
            s_id[tid] = id;
            s_mask[tid] = stage_record(recs, id, s_rec, tid, ox, oy);
        }
        __syncthreads();
        for (int k0 = ((n - 1) >> 5) << 5; k0 >= 0; k0 -= 32) {
            if ((uint32_t)(lo + k0) >= wmax) continue;     // whole group is past this warp's last contributor
            const uint32_t mine = (k0 + lane < n) ? ((s_mask[k0 + lane] >> warp) & 1u) : 0u;
            uint32_t bal = __ballot_sync(0xFFFFFFFFu, mine);
            while (bal) {
                const int jb = 31 - __clz(bal);
                bal &= ~(1u << jb);
                const int j = k0 + jb;
                const uint32_t ra = s_rec + j * REC_BYTES;
                const float4 g = lds128(ra), c = lds128(ra + 16);
                const float dx = g.x - pxf, dy = g.y - pyf;
                const float p2 = power2_of(c, dx, dy);
                const float G = ex2_approx(p2);
                const float alpha = fminf(0.99f, c.w * G);
                const bool active = ((uint32_t)(lo + j) < last_contrib) && (p2 <= 0.f) && !(alpha < ALPHA_MIN);
                if (!__any_sync(0xFFFFFFFFu, active)) continue;
                // raw moment sums; constants and conic factors are applied per Gaussian in preprocess_backward
                float v0 = 0.f, v1 = 0.f, v2 = 0.f, v3 = 0.f, v4 = 0.f, v5 = 0.f, v6 = 0.f, v7 = 0.f, v8 = 0.f, v9 = 0.f;
                if (active) {
                    const float4 k = lds128(ra + 32);
                    const float ria = rcp_approx(1.f - alpha);
                    T *= ria;
                    const float dchan = alpha * T;
                    float sj = fmaf(k.x, gC0, gA);
                    sj = fmaf(k.y, gC1, sj);
                    sj = fmaf(k.z, gC2, sj);
                    sj = fmaf(g.z, gD, sj);
                    behind = fmaf(last_alpha, last_s - behind, behind);
                    last_s = sj;
                    float dL_da = sj - behind;
                    dL_da = fmaf(dL_da, T, bgT * ria);      // *T, + (-T_final/(1-alpha)) * bg.dL_dpixel
                    last_alpha = alpha;
                    // straight-through min(0.99, .): gradient as if unclamped (App. A.1.6)
                    const float gda = G * dL_da;
                    const float w = c.w * gda;              // dL/dG * G
                    const float wx = w * dx, wy = w * dy;
                    v0 = wx; v1 = wy; v2 = dchan * gD;
                    v3 = wx * dx; v4 = wx * dy; v5 = wy * dy; v6 = gda;
                    v7 = dchan * gC0; v8 = dchan * gC1; v9 = dchan * gC2;
                }
                // transpose butterfly: 10 -> 5 -> 3 -> 2 -> 1 values per lane
                const float u0 = xstage(v0, v5, h16, 16), u1 = xstage(v1, v6, h16, 16), u2 = xstage(v2, v7, h16, 16),
                            u3 = xstage(v3, v8, h16, 16), u4 = xstage(v4, v9, h16, 16);
                const float t0 = xstage(u0, u3, h8, 8), t1 = xstage(u1, u4, h8, 8), t2 = xstage(u2, 0.f, h8, 8);
                const float s0 = xstage(t0, t2, h4, 4), s1 = xstage(t1, 0.f, h4, 4);
                float r = xstage(s0, s1, h2, 2);
                r += __shfl_xor_sync(0xFFFFFFFFu, r, 1);
                if (my_valid) atomicAdd(reinterpret_cast<double*>(sg + s_id[j]) + my_off, (double)r);
            }
        }
    }
}

}  // namespace

int gs_launch_render_forward_r1(const ViewArgs& va, const SplatRec* recs, const uint32_t* point_list,
                             const uint32_t* ranges, float* out_color, float* out_depth, float* out_alpha,
                             uint32_t* n_contrib, float* final_T, cudaStream_t s) {
    dim3 grid(va.tiles_x, va.tiles_y);
    render_forward_kernel<<<grid, RB, 0, s>>>(va, recs, point_list, ranges, out_color, out_depth, out_alpha,
                                              n_contrib, final_T);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int gs_launch_render_backward_r1(const ViewArgs& va, const SplatRec* recs, const uint32_t* point_list,
                              const uint32_t* ranges, const uint32_t* n_contrib, const float* final_T,
                              const float* dL_dcolor, const float* dL_ddepth, const float* dL_dalpha,
                              SplatGrad* sg, cudaStream_t s) {
    dim3 grid(va.tiles_x, va.tiles_y);
    static const int occ = getenv("GS_B200_BWD_OCC") ? atoi(getenv("GS_B200_BWD_OCC")) : 4;   // tuning knob: CTAs/SM target
    if (occ >= 5)
        render_backward_kernel<5><<<grid, RB, 0, s>>>(va, recs, point_list, ranges, n_contrib, final_T, dL_dcolor,
                                                      dL_ddepth, dL_dalpha, sg);
    else if (occ == 3)
        render_backward_kernel<3><<<grid, RB, 0, s>>>(va, recs, point_list, ranges, n_contrib, final_T, dL_dcolor,
                                                      dL_ddepth, dL_dalpha, sg);
    else
        render_backward_kernel<4><<<grid, RB, 0, s>>>(va, recs, point_list, ranges, n_contrib, final_T, dL_dcolor,
                                                      dL_ddepth, dL_dalpha, sg);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
