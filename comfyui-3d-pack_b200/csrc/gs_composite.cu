// Tile compositing, round-2 design: front-to-back alpha blend (forward) and its
// back-to-front replay (backward).
//
// Replaces renderCUDA (forward.cu / backward.cu) of diff_gaussian_rasterization,
// semantics per SURVEY.md App. A.1.6:  alpha = min(0.99, o*exp(power)); skip
// power>0 or alpha<1/255; stop WITHOUT blending when T(1-alpha) < 1e-4;
// color = C + T*bg, depth = sum(depth*alpha*T), alpha_out = sum(alpha*T).
// Called where main_3DGS_renderer.py:927-936 calls the rasterizer and where
// loss.backward() (main_3DGS.py:205) reaches its backward.
//
// Both kernels are meant to be instruction-issue bound (48 B splat records, gathered through L2),
// so the design minimises issued instructions per (pixel, splat):
//  * one CTA per 16x16 tile = 4 warps.  Warp w owns
//    the 8x8 quadrant (w&1, w>>1); every lane owns TWO pixels (x, y) and (x, y+4),
//    so dx and every per-splat operand are loaded and set up once for two
//    pixels (the pixel pair is carried as one 64-bit register pair);
//  * the tile's records are gathered by three 16 B cp.async per record (or, with
//    GS_B200_GATHER=tma, one 48 B cp.async.bulk) into a ring of shared-memory
//    stages, each completed on an mbarrier; a warp releases a stage with one
//    shared-memory atomic and the last of the four to release it refills it.
//    There is no __syncthreads() in the main loops;
//  * each warp decides by itself which records of a stage can reach
//    alpha >= 1/255 inside its quadrant (exact minimum of the quadratic form over
//    the 8x8 rectangle + slack): one test per lane and record, four ballots per
//    128-record stage, then the warp walks only the set bits;
//  * backward, per visit, only TWO values per pixel leave the lanes:
//    G*dL/dalpha and alpha*T.  They are queued in shared memory ([pixel][slot])
//    and, every 16 visits, a second phase with lanes = (slot, half-quadrant)
//    turns them into the ten per-splat sums (six image moments of G*dL/dalpha in
//    pixel-local coordinates, four colour/depth sums against per-pixel upstream
//    gradients) with plain FFMAs and no cross-lane traffic beyond one final
//    shfl.xor — the 12-SHFL transpose reduction per (warp, splat) of round 1 is
//    gone.  One fp64 red.global.add per value and (quadrant, splat) leaves the CTA
//    (SplatGrad in gs_common.cuh says why fp64).
#include "gs_common.cuh"
#include <stdlib.h>

namespace {

typedef unsigned long long u64;

constexpr int NMATH = 4;                 // warps per CTA, one per 8x8 quadrant
constexpr int NTHREADS = NMATH * 32;
constexpr int BATCH = 128;               // records per ring stage
constexpr uint32_t REC_BYTES = 48;
constexpr uint32_t STAGE_BYTES = BATCH * REC_BYTES;
constexpr float ALPHA_MIN = 1.0f / 255.0f;

// ---- pixel-pair helpers ---------------------------------------------------------------------------
// The two pixels of a lane travel as one 64-bit register pair.  sm_90 has no packed f32x2 arithmetic, so each
// helper issues two scalar IEEE operations; the explicit _rn intrinsics keep the rounding of every step (no FMA
// contraction of a mul followed by an add), so both pixels get exactly the results a packed instruction would give.
__device__ __forceinline__ u64 pk(float lo, float hi) { u64 r; asm("mov.b64 %0, {%1,%2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ u64 bc(float a) { return pk(a, a); }
__device__ __forceinline__ float lo(u64 v) { float a, b; asm("mov.b64 {%0,%1}, %2;" : "=f"(a), "=f"(b) : "l"(v)); return a; }
__device__ __forceinline__ float hi(u64 v) { float a, b; asm("mov.b64 {%0,%1}, %2;" : "=f"(a), "=f"(b) : "l"(v)); return b; }
__device__ __forceinline__ u64 fma2(u64 a, u64 b, u64 c) {
    return pk(__fmaf_rn(lo(a), lo(b), lo(c)), __fmaf_rn(hi(a), hi(b), hi(c)));
}
__device__ __forceinline__ u64 mul2(u64 a, u64 b) { return pk(__fmul_rn(lo(a), lo(b)), __fmul_rn(hi(a), hi(b))); }
__device__ __forceinline__ u64 add2(u64 a, u64 b) { return pk(__fadd_rn(lo(a), lo(b)), __fadd_rn(hi(a), hi(b))); }
__device__ __forceinline__ u64 sub2(u64 a, u64 b) { return pk(__fsub_rn(lo(a), lo(b)), __fsub_rn(hi(a), hi(b))); }

__device__ __forceinline__ float4 lds128(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ float2 lds64(uint32_t addr) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts64(uint32_t addr, float a, float b) {
    asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void sts128(uint32_t addr, float4 v) {
    asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float lg2_approx(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// ---- mbarrier / bulk-copy helpers ---------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "W_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
        "@p bra D_%=;\n\t"
        "bra W_%=;\n\t"
        "D_%=:\n\t}" ::"r"(bar), "r"(parity), "r"(1000000u) : "memory");   // suspend-time hint (ns): sleep in hardware, do not poll
}
// one record: global -> shared through the bulk-copy engine, completion counted on `bar`
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// adds the first n components of v to an fp64 double4 of a SplatGrad record (sm_90 has no vector fp64 red)
__device__ __forceinline__ void red_add_d4(double* addr, float4 v, int n) {
    atomicAdd(addr, (double)v.x); atomicAdd(addr + 1, (double)v.y); atomicAdd(addr + 2, (double)v.z);
    if (n == 4) atomicAdd(addr + 3, (double)v.w);
}
__device__ __forceinline__ uint32_t ld_volatile_s32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}

// May a splat reach alpha >= 1/255 somewhere in the 8x8 pixel square with corner (X0, Y0)?  Exact minimum of
// q(u) = 0.5(A ux^2 + C uy^2) + B ux uy (log2 units) over the rectangle, with slack for fp32 rounding and the
// approximate reciprocals; a rejected splat fails the per-pixel alpha test on every lane anyway.
__device__ __forceinline__ bool quad_hit(const float4 g, const float4 c, float X0, float Y0) {
    const float o = c.w;
    if (!(o * 255.0f >= 1.0f) || __float_as_int(g.w) <= 0) return false;    // can never reach 1/255 (also NaN)
    const float tau = lg2_approx(o * 255.0f) * 1.001f + 0.03f;
    const float A = -2.0f * c.x, B = -c.y, C = -2.0f * c.z;
    if (!(A > 0.f && A * C - B * B > 0.f)) return true;                     // not positive definite: per-pixel test decides
    const float ux0 = X0 - g.x, ux1 = ux0 + 7.0f;
    const float uy0 = Y0 - g.y, uy1 = uy0 + 7.0f;
    const bool outx = (ux0 > 0.f) || (ux1 < 0.f);
    const bool outy = (uy0 > 0.f) || (uy1 < 0.f);
    float q = 0.f;
    if (outx || outy) {
        q = 3.0e38f;
        if (outx) {
            const float ue = (ux0 > 0.f) ? ux0 : ux1;
            const float uy = fminf(fmaxf(-B * ue * rcp_approx(C), uy0), uy1);
            q = 0.5f * (A * ue * ue + C * uy * uy) + B * ue * uy;
        }
        if (outy) {
            const float ue = (uy0 > 0.f) ? uy0 : uy1;
            const float ux = fminf(fmaxf(-B * ue * rcp_approx(A), ux0), ux1);
            q = fminf(q, 0.5f * (A * ux * ux + C * ue * ue) + B * ux * ue);
        }
    }
    return !(q > tau);      // NaN -> keep (conservative)
}

// index of the highest set bit (x != 0).  `31 - __clz(x)` compiles to FLO, 31 - ., xor 31 and the mask update to a shift
// of 0x80000000, a NOT and an AND: six instructions per visit where bfind + shift + and-not do it in three.
__device__ __forceinline__ int hibit(uint32_t x) {
    int h;
    asm("bfind.u32 %0, %1;" : "=r"(h) : "r"(x));
    return h;
}

// hit masks of one stage for this warp's quadrant: bit l of m[i] <-> record i*32 + l
__device__ __forceinline__ void stage_masks(uint32_t s_rec, int n, int lane, float X0, float Y0, uint32_t m[BATCH / 32]) {
#pragma unroll
    for (int i = 0; i < BATCH / 32; i++) {
        const int j = i * 32 + lane;
        bool hit = false;
        if (j < n) {
            const uint32_t ra = s_rec + j * REC_BYTES;
            hit = quad_hit(lds128(ra), lds128(ra + 16), X0, Y0);
        }
        m[i] = __ballot_sync(0xFFFFFFFFu, hit);
    }
}

// m[i] with i known only at run time, without putting the array into local memory
__device__ __forceinline__ uint32_t pick_mask(const uint32_t m[BATCH / 32], int i) {
    static_assert(BATCH == 128, "pick_mask is written for four groups");
    return i == 0 ? m[0] : (i == 1 ? m[1] : (i == 2 ? m[2] : (i == 3 ? m[3] : 0u)));
}

// power (log2 units) of both pixels of the lane; the operation order is the scalar one of round 1
// (t = cx*dx; t = fma(cy, dy, t); p = t*dx; p = fma(cz*dy, dy, p)) so forward and backward agree bit for bit.
__device__ __forceinline__ u64 power2(const float4 c, float dx, u64 dy2) {
    const float t = c.x * dx;
    const u64 t2 = fma2(bc(c.y), dy2, bc(t));
    const u64 p = mul2(t2, bc(dx));
    const u64 q = mul2(bc(c.z), dy2);
    return fma2(q, dy2, p);
}

struct RingState {
    uint32_t stage = 0, phase = 0;
    __device__ __forceinline__ void advance(int nstages) { if (++stage == (uint32_t)nstages) { stage = 0; phase ^= 1u; } }
};

// gather of one stage: ids (coalesced LDG), then per record either three 16 B cp.async (LDGSTS) per lane with one
// cp.async.mbarrier.arrive.noinc per lane (the stage's mbarrier expects 32 arrivals) -- the default -- or
// (GS_B200_GATHER=tma) ONE 48 B bulk copy through the TMA engine (UBLKCP; completion = bytes counted on the stage's
// mbarrier, which one expect_tx arrival arms).  UBLKCP takes its operands from uniform registers, so a per-lane
// gather serialises into a ~9-instruction loop per record inside the issuing warp, whereas the three LDGSTS are one
// warp-wide instruction each.
template <bool KEEP_IDS, bool TMA>
__device__ __forceinline__ void produce_stage(const SplatRec* __restrict__ recs, const uint32_t* __restrict__ list, int n,
                                              uint32_t s_rec, uint32_t s_ids, uint32_t bar, int lane) {
    uint32_t id[BATCH / 32];
#pragma unroll
    for (int i = 0; i < BATCH / 32; i++) {
        const int j = i * 32 + lane;
        id[i] = (j < n) ? __ldg(list + j) : 0u;
    }
    if (KEEP_IDS) {
#pragma unroll
        for (int i = 0; i < BATCH / 32; i++) {
            const int j = i * 32 + lane;
            if (j < n) asm volatile("st.shared.u32 [%0], %1;" ::"r"(s_ids + j * 4), "r"(id[i]) : "memory");
        }
        __syncwarp();
    }
    if (TMA) {
        if (lane == 0) mbar_arrive_expect_tx(bar, (uint32_t)n * REC_BYTES);
        __syncwarp();
#pragma unroll
        for (int i = 0; i < BATCH / 32; i++) {
            const int j = i * 32 + lane;
            if (j < n) bulk_g2s(s_rec + j * REC_BYTES, recs + id[i], REC_BYTES, bar);
        }
    } else {
#pragma unroll
        for (int i = 0; i < BATCH / 32; i++) {
            const int j = i * 32 + lane;
            if (j < n) {
                const char* src = reinterpret_cast<const char*>(recs + id[i]);
                const uint32_t dst = s_rec + j * REC_BYTES;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + 16), "l"(src + 16) : "memory");
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + 32), "l"(src + 32) : "memory");
            }
        }
        if (KEEP_IDS) __threadfence_block();        // the ids written above must be visible to whoever sees the stage complete
        asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
    }
}
constexpr uint32_t full_count(bool tma) { return tma ? 1u : 32u; }
__device__ __forceinline__ void mbar_arrive_n(uint32_t bar, uint32_t n) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(bar), "r"(n) : "memory");
}

// ---- one visit of the forward, split into a state-free front half and the sequential blend ------------------------
struct FwdFront { u64 al2, p2; float gz; };

__device__ __forceinline__ FwdFront fwd_front(uint32_t ra, float pxf, float pyfA, float pyfB) {
    FwdFront f;
    const float4 g = lds128(ra), c = lds128(ra + 16);
    const float dx = g.x - pxf;
    const u64 dy2 = sub2(bc(g.y), pk(pyfA, pyfB));
    f.p2 = power2(c, dx, dy2);
    const u64 a2 = mul2(bc(c.w), pk(ex2_approx(lo(f.p2)), ex2_approx(hi(f.p2))));
    f.al2 = pk(fminf(0.99f, lo(a2)), fminf(0.99f, hi(a2)));
    f.gz = g.z;
    return f;
}
// contributes iff power <= 0 (a terminated pixel has a NaN power) and alpha >= 1/255
__device__ __forceinline__ bool fwd_live(float p, float al) { return (p <= 0.f) && !(al < ALPHA_MIN); }

struct FwdAcc { float c0a, c0b, c1a, c1b, c2a, c2b, da, db, aa, ab; };

__device__ __forceinline__ void fwd_back(const FwdFront& f, bool liveA, bool liveB, uint32_t ra, uint32_t pos, float& TA,
                                         float& TB, FwdAcc& acc, uint32_t& lastA, uint32_t& lastB,
                                         float& pyfA, float& pyfB) {
    const u64 T2 = pk(TA, TB);
    const u64 tt2 = mul2(T2, sub2(bc(1.f), f.al2));          // T * (1 - alpha)
    const bool stopA = liveA && (lo(tt2) < 0.0001f), stopB = liveB && (hi(tt2) < 0.0001f);
    const bool blA = liveA && !stopA, blB = liveB && !stopB;
    const u64 w2raw = mul2(f.al2, T2);
    const u64 w2 = pk(blA ? lo(w2raw) : 0.f, blB ? hi(w2raw) : 0.f);
    const float4 k = lds128(ra + 32);
    u64 t;
    t = fma2(bc(k.x), w2, pk(acc.c0a, acc.c0b)); acc.c0a = lo(t); acc.c0b = hi(t);
    t = fma2(bc(k.y), w2, pk(acc.c1a, acc.c1b)); acc.c1a = lo(t); acc.c1b = hi(t);
    t = fma2(bc(k.z), w2, pk(acc.c2a, acc.c2b)); acc.c2a = lo(t); acc.c2b = hi(t);
    t = fma2(bc(f.gz), w2, pk(acc.da, acc.db)); acc.da = lo(t); acc.db = hi(t);
    t = add2(pk(acc.aa, acc.ab), w2); acc.aa = lo(t); acc.ab = hi(t);
    TA = blA ? lo(tt2) : TA; TB = blB ? hi(tt2) : TB;
    lastA = blA ? pos : lastA; lastB = blB ? pos : lastB;
    const float QNAN = __int_as_float(0x7fc00000);           // terminated: the pixel's row coordinate becomes NaN
    pyfA = stopA ? QNAN : pyfA; pyfB = stopB ? QNAN : pyfB;
}

// Variant of fwd_back for the common case "no pixel of the warp terminates at this visit": a pixel that does not take
// the splat blends it with alpha 0 (T * (1 - 0) = T exactly, weight 0), so T and the weights need no per-pixel
// selects; T stays >= 1e-4 for every pixel that has not terminated, hence "T (1 - alpha) < 1e-4" alone identifies a
// terminating pixel and ONE warp vote per visit guards the fix-up (weight 0, T kept, row coordinate poisoned).
__device__ __forceinline__ void fwd_back_sv(const FwdFront& f, bool liveA, bool liveB, uint32_t ra, uint32_t pos, float& TA,
                                            float& TB, FwdAcc& acc, uint32_t& lastA, uint32_t& lastB,
                                            float& pyfA, float& pyfB) {
    const u64 ae2 = pk(liveA ? lo(f.al2) : 0.f, liveB ? hi(f.al2) : 0.f);
    const u64 T2 = pk(TA, TB);
    const u64 tt2 = mul2(T2, sub2(bc(1.f), ae2));            // T * (1 - alpha)
    const u64 w2r = mul2(ae2, T2);
    float wA = lo(w2r), wB = hi(w2r);
    const float oTA = TA, oTB = TB;
    TA = lo(tt2); TB = hi(tt2);
    bool blA = liveA, blB = liveB;
    if (__any_sync(0xFFFFFFFFu, fminf(TA, TB) < 0.0001f)) {
        const bool stopA = TA < 0.0001f, stopB = TB < 0.0001f;
        const float QNAN = __int_as_float(0x7fc00000);
        wA = stopA ? 0.f : wA; wB = stopB ? 0.f : wB;
        TA = stopA ? oTA : TA; TB = stopB ? oTB : TB;
        pyfA = stopA ? QNAN : pyfA; pyfB = stopB ? QNAN : pyfB;
        blA = liveA && !stopA; blB = liveB && !stopB;
    }
    lastA = blA ? pos : lastA; lastB = blB ? pos : lastB;
    const u64 w2 = pk(wA, wB);
    const float4 k = lds128(ra + 32);
    u64 t;
    t = fma2(bc(k.x), w2, pk(acc.c0a, acc.c0b)); acc.c0a = lo(t); acc.c0b = hi(t);
    t = fma2(bc(k.y), w2, pk(acc.c1a, acc.c1b)); acc.c1a = lo(t); acc.c1b = hi(t);
    t = fma2(bc(k.z), w2, pk(acc.c2a, acc.c2b)); acc.c2a = lo(t); acc.c2b = hi(t);
    t = fma2(bc(f.gz), w2, pk(acc.da, acc.db)); acc.da = lo(t); acc.db = hi(t);
    t = add2(pk(acc.aa, acc.ab), w2); acc.aa = lo(t); acc.ab = hi(t);
}

// =================================================================================================
// forward
// =================================================================================================
template <int STAGES, bool TMA, bool STOPVOTE>
__global__ void __launch_bounds__(NTHREADS)
composite_forward_kernel(ViewArgs va, const SplatRec* __restrict__ recs, const uint32_t* __restrict__ point_list,
                         const uint32_t* __restrict__ ranges, float* __restrict__ out_color,
                         float* __restrict__ out_depth, float* __restrict__ out_alpha,
                         uint32_t* __restrict__ n_contrib, float* __restrict__ final_T) {
    __shared__ __align__(128) unsigned char s_rec_raw[STAGES * STAGE_BYTES];
    __shared__ __align__(8) u64 s_full[STAGES];
    __shared__ uint32_t s_cnt[STAGES], s_stop;
    const uint32_t s_rec = (uint32_t)__cvta_generic_to_shared(s_rec_raw);
    const uint32_t a_full = (uint32_t)__cvta_generic_to_shared(s_full);
    const uint32_t a_stop = (uint32_t)__cvta_generic_to_shared(&s_stop);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tile = blockIdx.y * va.tiles_x + blockIdx.x;
    const uint32_t start = ranges[2 * tile], end = ranges[2 * tile + 1];
    const int len = (int)(end - start);
    const int nb = (len + BATCH - 1) / BATCH;

    if (tid == 0) {
        for (int i = 0; i < STAGES; i++) { mbar_init(a_full + 8 * i, full_count(TMA)); s_cnt[i] = 0; }
        s_stop = 0xFFFFFFFFu;
        mbar_fence_init();
    }
    __syncthreads();
    // first fill of the ring: warp w gathers batch w (afterwards the LAST warp to finish a stage refills it)
    if (warp < STAGES && warp < nb)
        produce_stage<false, TMA>(recs, point_list + start + warp * BATCH, min(BATCH, len - warp * BATCH), s_rec + warp * STAGE_BYTES, 0u,
                             a_full + 8 * warp, lane);

    const int X0 = blockIdx.x * GS_TILE + 8 * (warp & 1), Y0 = blockIdx.y * GS_TILE + 8 * (warp >> 1);
    const int px = X0 + (lane & 7), pyA = Y0 + (lane >> 3), pyB = pyA + 4;
    const bool inA = px < va.W && pyA < va.H, inB = px < va.W && pyB < va.H;
    const float pxf = (float)px;
    const float X0f = (float)X0, Y0f = (float)Y0;
    // A pixel that has terminated (or lies outside the image) gets a NaN row coordinate: its power is then NaN, fails
    // "power <= 0" and the pixel drops out of every later test without a per-pixel flag in the loop.
    const float QNAN = __int_as_float(0x7fc00000);
    float pyfA = inA ? (float)pyA : QNAN, pyfB = inB ? (float)pyB : QNAN;

    float TA = 1.f, TB = 1.f;
    FwdAcc acc = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    uint32_t lastA = 0, lastB = 0;
    bool warp_done = __all_sync(0xFFFFFFFFu, !inA && !inB);

    RingState rs;
    for (int b = 0; b < nb; b++) {
        mbar_wait(a_full + 8 * rs.stage, rs.phase);
        if ((uint32_t)b == ld_volatile_s32(a_stop)) break;
        if (!warp_done) {
            const int n = min(BATCH, len - b * BATCH);
            const uint32_t sr = s_rec + rs.stage * STAGE_BYTES;
            uint32_t m[BATCH / 32];
            stage_masks(sr, n, lane, X0f, Y0f, m);
#pragma unroll
            for (int i = 0; i < BATCH / 32; i++) {
                uint32_t bal = m[i];
                const uint32_t rg = sr + i * 32 * REC_BYTES;
                const uint32_t pos0 = (uint32_t)(b * BATCH + i * 32 + 1);
                // two visits per iteration: their front halves (load, power, exp, alpha) are independent and interleave;
                // the blend updates run in list order
                while (bal) {
                    const int j0 = __ffs(bal) - 1;
                    bal &= bal - 1;
                    const bool two = bal != 0;
                    const int j1 = two ? __ffs(bal) - 1 : j0;
                    bal &= bal - 1;
                    const uint32_t ra0 = rg + j0 * REC_BYTES, ra1 = rg + j1 * REC_BYTES;
                    const FwdFront f0 = fwd_front(ra0, pxf, pyfA, pyfB);
                    const FwdFront f1 = fwd_front(ra1, pxf, pyfA, pyfB);
                    // (no warp vote around the blend: 96 % of the visits have a live lane, and the branch made ptxas copy
                    // the ten accumulator registers at its join)
                    if (STOPVOTE) {
                        fwd_back_sv(f0, fwd_live(lo(f0.p2), lo(f0.al2)), fwd_live(hi(f0.p2), hi(f0.al2)), ra0, pos0 + j0,
                                    TA, TB, acc, lastA, lastB, pyfA, pyfB);
                        fwd_back_sv(f1, two && fwd_live(lo(f1.p2), lo(f1.al2)) && (pyfA == pyfA), two && fwd_live(hi(f1.p2), hi(f1.al2)) && (pyfB == pyfB),
                                    ra1, pos0 + j1, TA, TB, acc, lastA, lastB, pyfA, pyfB);
                        continue;
                    }
                    fwd_back(f0, fwd_live(lo(f0.p2), lo(f0.al2)), fwd_live(hi(f0.p2), hi(f0.al2)), ra0, pos0 + j0,
                             TA, TB, acc, lastA, lastB, pyfA, pyfB);
                    // visit 1's front half saw the row coordinates from before visit 0: drop pixels that just terminated
                    // (`two` false: j1 == j0 and the visit is masked off as a whole)
                    fwd_back(f1, two && fwd_live(lo(f1.p2), lo(f1.al2)) && (pyfA == pyfA), two && fwd_live(hi(f1.p2), hi(f1.al2)) && (pyfB == pyfB),
                             ra1, pos0 + j1, TA, TB, acc, lastA, lastB, pyfA, pyfB);
                }
                if (__all_sync(0xFFFFFFFFu, (pyfA != pyfA) && (pyfB != pyfB))) { warp_done = true; break; }
            }
        }
        // release the stage; the last of the four warps to do so refills it with batch b + STAGES.  Each release carries
        // the warp's "all my pixels have terminated" bit: when all four say so the tile is finished, nothing is gathered
        // any more and the stop batch is published (a function of b only, so concurrent refills cannot disagree).
        __syncwarp();
        uint32_t tot = 0;
        if (lane == 0) { __threadfence_block(); tot = atomicAdd(&s_cnt[rs.stage], 1u + (warp_done ? 0x100u : 0u)) + 1u + (warp_done ? 0x100u : 0u); }
        tot = __shfl_sync(0xFFFFFFFFu, tot, 0);
        if ((tot & 0xFFu) == NMATH) {
            const int nbatch = b + STAGES;
            // acquire side of the hand-over (release = the fence before each warp's atomic): the other warps' reads of
            // the stage happen before the refill below overwrites it
            if (lane == 0) { __threadfence_block(); s_cnt[rs.stage] = 0; }
            __syncwarp();
            if (nbatch < nb) {
                if ((tot >> 8) == NMATH) {
                    if (lane == 0) { atomicMin(&s_stop, (uint32_t)nbatch); __threadfence_block(); mbar_arrive_n(a_full + 8 * rs.stage, full_count(TMA)); }
                } else {
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // the stage was read through the generic proxy
                    produce_stage<false, TMA>(recs, point_list + start + nbatch * BATCH, min(BATCH, len - nbatch * BATCH),
                                         s_rec + rs.stage * STAGE_BYTES, 0u, a_full + 8 * rs.stage, lane);
                }
            }
        }
        rs.advance(STAGES);
    }
    const size_t plane = (size_t)va.W * va.H;
    const float bg0 = __ldg(va.bg), bg1 = __ldg(va.bg + 1), bg2 = __ldg(va.bg + 2);
    if (inA) {
        const size_t pix = (size_t)pyA * va.W + px;
        out_color[pix] = acc.c0a + TA * bg0; out_color[plane + pix] = acc.c1a + TA * bg1; out_color[2 * plane + pix] = acc.c2a + TA * bg2;
        out_depth[pix] = acc.da; out_alpha[pix] = acc.aa; n_contrib[pix] = lastA; final_T[pix] = TA;
    }
    if (inB) {
        const size_t pix = (size_t)pyB * va.W + px;
        out_color[pix] = acc.c0b + TB * bg0; out_color[plane + pix] = acc.c1b + TB * bg1; out_color[2 * plane + pix] = acc.c2b + TB * bg2;
        out_depth[pix] = acc.db; out_alpha[pix] = acc.ab; n_contrib[pix] = lastB; final_T[pix] = TB;
    }
}

// =================================================================================================
// backward
// =================================================================================================
// queue geometry for SLOTS queued visits per flush (8 or 16): a row = SLOTS float2 + 8 B pad (bank spread), 32 lane rows
// per array, two arrays (G dL/dalpha pairs, alpha T pairs) per warp
template <int SLOTS> struct QGeom {
    static constexpr uint32_t ROW = (SLOTS + 1) * 8;
    static constexpr uint32_t WARP = 64 * ROW;
    static constexpr int PARTS = 32 / SLOTS;       // lanes = (slot, part); a part owns SLOTS consecutive lane rows
};

// Second phase of the backward: lanes = (slot, part).  Each lane sums, over its SLOTS pixel pairs (pixel A = (x, y),
// pixel B = (x, y+4) of first-phase lane 8y+x), the queued (G*dL/dalpha, alpha*T) of its slot against pixel-local
// coordinates and the per-pixel upstream gradients; the parts are then added with shfl.xor.
template <int SLOTS>
__device__ __noinline__ void flush_queue(uint32_t q_base, uint32_t coef_base, uint32_t slot_base, int nq, int lane,
                                         float Xc, float Yc, const uint32_t* __restrict__ tile_list,
                                         const SplatRec* __restrict__ recs, SplatGrad* __restrict__ sg) {
    using Q = QGeom<SLOTS>;
    const int slot = lane & (SLOTS - 1), part = lane / SLOTS;
    // a slot remembers only the list position of its splat (one 4 B store per visit by lane 0): the id comes from the
    // tile's list and mean2D / opacity from the splat's record here -- L2 hits issued before the sums, so their latency
    // hides behind them
    uint32_t gid = 0u;
    float4 si = make_float4(0.f, 0.f, 0.f, 0.f);                // mean2D.x, mean2D.y, -, opacity
    if (slot < nq) {
        uint32_t pos;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(pos) : "r"(slot_base + slot * 4));
        gid = __ldg(tile_list + pos);
        const float4 g = __ldg(&recs[gid].g), c = __ldg(&recs[gid].c);
        si = make_float4(g.x, g.y, 0.f, c.w);
    }
    const uint32_t qg = q_base + slot * 8 + part * SLOTS * Q::ROW, qd = qg + 32 * Q::ROW;
    const uint32_t ca = coef_base + part * SLOTS * 32;
    float M0 = 0.f, M1 = 0.f, M2 = 0.f, My = 0.f, Mxy = 0.f, Myy = 0.f;
    u64 Cr2 = bc(0.f), Cg2 = bc(0.f), Cb2 = bc(0.f), Cd2 = bc(0.f);       // (pixel A, pixel B) halves, added at the end
#pragma unroll
    for (int r = 0; r < SLOTS / 8; r++) {
        u64 s0 = bc(0.f), s1 = bc(0.f), s2 = bc(0.f);                       // row sums of w, w*LX, w*LX^2 for (row of A, row of B)
#pragma unroll
        for (int x = 0; x < 8; x++) {
            const int p = r * 8 + x;
            u64 w, d, c0, c1, c2, cd;
            asm volatile("ld.shared.b64 %0, [%1];" : "=l"(w) : "r"(qg + p * Q::ROW));
            asm volatile("ld.shared.b64 %0, [%1];" : "=l"(d) : "r"(qd + p * Q::ROW));
            asm volatile("ld.shared.v2.b64 {%0,%1}, [%2];" : "=l"(c0), "=l"(c1) : "r"(ca + p * 32));
            asm volatile("ld.shared.v2.b64 {%0,%1}, [%2];" : "=l"(c2), "=l"(cd) : "r"(ca + p * 32 + 16));
            const float LX = (float)x - 3.5f;
            s0 = add2(s0, w); s1 = fma2(w, bc(LX), s1); s2 = fma2(w, bc(LX * LX), s2);
            Cr2 = fma2(d, c0, Cr2); Cg2 = fma2(d, c1, Cg2); Cb2 = fma2(d, c2, Cb2); Cd2 = fma2(d, cd, Cd2);
        }
        const float LYA = (float)(part * (SLOTS / 8) + r) - 3.5f, LYB = LYA + 4.0f;
        const float a0 = lo(s0), b0 = hi(s0), a1 = lo(s1), b1 = hi(s1);
        M0 += a0 + b0; M1 += a1 + b1; M2 += lo(s2) + hi(s2);
        My = fmaf(a0, LYA, My); Mxy = fmaf(a1, LYA, Mxy); Myy = fmaf(a0, LYA * LYA, Myy);
        My = fmaf(b0, LYB, My); Mxy = fmaf(b1, LYB, Mxy); Myy = fmaf(b0, LYB * LYB, Myy);
    }
    float Cr = lo(Cr2) + hi(Cr2), Cg = lo(Cg2) + hi(Cg2), Cb = lo(Cb2) + hi(Cb2), Cd = lo(Cd2) + hi(Cd2);
#pragma unroll
    for (int o = 16; o >= SLOTS; o >>= 1) {
#define XADD(v) v += __shfl_xor_sync(0xFFFFFFFFu, v, o)
        XADD(M0); XADD(M1); XADD(M2); XADD(My); XADD(Mxy); XADD(Myy); XADD(Cd); XADD(Cr); XADD(Cg); XADD(Cb);
#undef XADD
    }
    if (slot < nq) {
        double* dst = reinterpret_cast<double*>(sg + gid);
        // pixel = centre + L, d = mean2D - pixel = u - L with u = mean2D - centre
        const float u = si.x - Xc, v = si.y - Yc, o = si.w;
        // the ten sums of the splat = the three double4 of its SplatGrad record (ten fp64 reds per (quadrant, splat)),
        // shared between the parts of the slot
        const float4 qg = make_float4(o * (u * M0 - M1),                                   // sum w dx
                                      o * (v * M0 - My),                                   // sum w dy
                                      Cd, 0.f);                                            // dL/ddepth
        const float4 qc = make_float4(o * (fmaf(u, fmaf(u, M0, -2.f * M1), M2)),           // sum w dx dx
                                      o * (fmaf(u, fmaf(v, M0, -My), fmaf(-v, M1, Mxy))),  // sum w dx dy
                                      o * (fmaf(v, fmaf(v, M0, -2.f * My), Myy)),          // sum w dy dy
                                      M0);                                                 // dL/dopacity (sum G dL/dalpha)
        const float4 qk = make_float4(Cr, Cg, Cb, 0.f);                                    // dL/drgb
        if (Q::PARTS == 2) {
            red_add_d4(dst + (part == 0 ? 0 : 8), part == 0 ? qg : qk, 3);
            if (part == 0) red_add_d4(dst + 4, qc, 4);
        } else {
            if (part < 3) red_add_d4(dst + 4 * part, part == 0 ? qg : (part == 1 ? qc : qk), part == 1 ? 4 : 3);
        }
    }
}

// ---- one visit of the backward: recurrence-free front half, then the short sequential part ---------------------------
struct BwdFront { u64 al2, G2, ria, sj, bgr; bool any; };

__device__ __forceinline__ BwdFront bwd_front(uint32_t ra, uint32_t pos, float pxf, u64 py2, uint32_t lcA, uint32_t lcB, u64 gC0,
                                              u64 gC1, u64 gC2, u64 gD, u64 gA, u64 bgT, bool on = true) {
    BwdFront f;
    const float4 g = lds128(ra), c = lds128(ra + 16), k = lds128(ra + 32);
    const float dx = g.x - pxf;
    const u64 dy2 = sub2(bc(g.y), py2);
    const u64 p2 = power2(c, dx, dy2);
    const float pA = lo(p2), pB = hi(p2);
    float GA = ex2_approx(pA), GB = ex2_approx(pB);
    const u64 a2 = mul2(bc(c.w), pk(GA, GB));
    float alA = fminf(0.99f, lo(a2)), alB = fminf(0.99f, hi(a2));
    const bool actA = on && (pos < lcA) && (pA <= 0.f) && !(alA < ALPHA_MIN);
    const bool actB = on && (pos < lcB) && (pB <= 0.f) && !(alB < ALPHA_MIN);
    f.any = actA || actB;
    // a pixel the splat was not blended into runs the same code with alpha = G = 0: T, behind and both outputs are then
    // unchanged / zero
    alA = actA ? alA : 0.f; alB = actB ? alB : 0.f;
    GA = actA ? GA : 0.f; GB = actB ? GB : 0.f;
    f.al2 = pk(alA, alB); f.G2 = pk(GA, GB);
    const u64 om = sub2(bc(1.f), f.al2);
    f.ria = pk(rcp_approx(lo(om)), rcp_approx(hi(om)));          // alpha = 0 -> rcp(1) = 1 exactly
    u64 sj = fma2(bc(k.x), gC0, gA);                             // s_j = gC.rgb_j + gD*depth_j + gA
    sj = fma2(bc(k.y), gC1, sj);
    sj = fma2(bc(k.z), gC2, sj);
    f.sj = fma2(bc(g.z), gD, sj);
    f.bgr = mul2(bgT, f.ria);                                    // (-T_final/(1-alpha)) * bg.dL_dpixel
    return f;
}

__device__ __forceinline__ void bwd_back(const BwdFront& f, u64& T2, u64& behind, uint32_t qg, uint32_t qd) {
    T2 = mul2(T2, f.ria);                                        // T_j = T_{j+1} / (1 - alpha_j)
    const u64 dchan = mul2(f.al2, T2);                           // d pixel / d channel_j = alpha_j T_j
    const u64 ds = sub2(f.sj, behind);                           // s_j - (colour behind splat j)
    const u64 dL_da = fma2(ds, T2, f.bgr);
    behind = fma2(f.al2, ds, behind);                            // colour behind splat j-1
    // straight-through min(0.99, .): gradient as if unclamped (App. A.1.6); w = opacity * gda is applied per slot
    const u64 gda = mul2(f.G2, dL_da);
    // (two "f" operands, not one 64-bit "l": with the packed value as a single operand ptxas copied the pair into fresh
    // registers before every store -- four MOVs per visit)
    sts64(qg, lo(gda), hi(gda));
    sts64(qd, lo(dchan), hi(dchan));
}

// PAIR: every loop iteration runs BOTH visits; when the group has an odd number of hits the second one is masked off
// (alpha = G = 0: T, behind and the queued values are then unchanged / zero, and its queue slot is not consumed) and the
// queue is checked once per iteration (flushed early at SLOTS - 1) -- one branch region per iteration instead of three.
template <int STAGES, int SLOTS, int MINB, bool VOTE, bool TMA, bool PAIR>
__global__ void __launch_bounds__(NTHREADS, MINB)
composite_backward_kernel(ViewArgs va, const SplatRec* __restrict__ recs, const uint32_t* __restrict__ point_list,
                          const uint32_t* __restrict__ ranges, const uint32_t* __restrict__ n_contrib,
                          const float* __restrict__ final_T, const float* __restrict__ dL_dcolor,
                          const float* __restrict__ dL_ddepth, const float* __restrict__ dL_dalpha,
                          SplatGrad* __restrict__ sg) {
    using Q = QGeom<SLOTS>;
    // dynamic shared memory: ring | queue | per-pixel upstream gradients | slot info | barriers | counters | wmax
    extern __shared__ __align__(128) unsigned char smem[];
    const uint32_t s_rec = (uint32_t)__cvta_generic_to_shared(smem);
    const uint32_t s_q = s_rec + STAGES * STAGE_BYTES;
    const uint32_t s_coef = s_q + NMATH * Q::WARP;
    const uint32_t s_slot = s_coef + NMATH * 64 * 16;
    const uint32_t a_full = s_slot + NMATH * SLOTS * 4;
    uint32_t* s_cnt = reinterpret_cast<uint32_t*>(smem + (a_full + 8 * STAGES - s_rec));
    volatile uint32_t* s_wmax = s_cnt + STAGES;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tile = blockIdx.y * va.tiles_x + blockIdx.x;
    const uint32_t start = ranges[2 * tile], end = ranges[2 * tile + 1];
    if (end <= start) return;

    const int X0 = blockIdx.x * GS_TILE + 8 * (warp & 1), Y0 = blockIdx.y * GS_TILE + 8 * (warp >> 1);
    const int px = X0 + (lane & 7), pyA = Y0 + (lane >> 3), pyB = pyA + 4;
    const bool inA = px < va.W && pyA < va.H, inB = px < va.W && pyB < va.H;
    const size_t plane = (size_t)va.W * va.H;
    const size_t pixA = (size_t)pyA * va.W + px, pixB = (size_t)pyB * va.W + px;
    const uint32_t lcA = inA ? n_contrib[pixA] : 0u, lcB = inB ? n_contrib[pixB] : 0u;
    uint32_t wmax = max(lcA, lcB);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xFFFFFFFFu, wmax, o));
    if (lane == 0) s_wmax[warp] = wmax;
    if (tid == 0) {
        for (int i = 0; i < STAGES; i++) { mbar_init(a_full + 8 * i, full_count(TMA)); s_cnt[i] = 0; }
        mbar_fence_init();
    }
    __syncthreads();
    const uint32_t nproc = max(max(s_wmax[0], s_wmax[1]), max(s_wmax[2], s_wmax[3]));   // list positions 1..nproc were blended
    const uint32_t* __restrict__ tile_list = point_list + start;
    if (nproc == 0) return;
    const int nb = (int)((nproc + BATCH - 1) / BATCH);
    // stages are gathered from the back of the list: iteration `it` holds list positions [(nb-1-it)*BATCH, +BATCH)
    auto produce = [&](int it, uint32_t stage) {
        const int base = (nb - 1 - it) * BATCH;
        produce_stage<false, TMA>(recs, point_list + start + base, min(BATCH, (int)nproc - base), s_rec + stage * STAGE_BYTES,
                             0u, a_full + 8 * stage, lane);
    };
    if (warp < STAGES && warp < nb) produce(warp, warp);       // first fill; afterwards the last warp to finish a stage refills it

    const float pxf = (float)px;
    const u64 py2 = pk((float)pyA, (float)pyB);
    const float X0f = (float)X0, Y0f = (float)Y0;
    const float TfA = inA ? final_T[pixA] : 0.f, TfB = inB ? final_T[pixB] : 0.f;
    float gC0A = 0.f, gC1A = 0.f, gC2A = 0.f, gDA = 0.f, gAA = 0.f, gC0B = 0.f, gC1B = 0.f, gC2B = 0.f, gDB = 0.f, gAB = 0.f;
    if (inA) { gC0A = dL_dcolor[pixA]; gC1A = dL_dcolor[plane + pixA]; gC2A = dL_dcolor[2 * plane + pixA]; gDA = dL_ddepth[pixA]; gAA = dL_dalpha[pixA]; }
    if (inB) { gC0B = dL_dcolor[pixB]; gC1B = dL_dcolor[plane + pixB]; gC2B = dL_dcolor[2 * plane + pixB]; gDB = dL_ddepth[pixB]; gAB = dL_dalpha[pixB]; }
    const float bg0 = __ldg(va.bg), bg1 = __ldg(va.bg + 1), bg2 = __ldg(va.bg + 2);
    const u64 gC0 = pk(gC0A, gC0B), gC1 = pk(gC1A, gC1B), gC2 = pk(gC2A, gC2B), gD = pk(gDA, gDB), gA = pk(gAA, gAB);
    const u64 bgT = pk(-TfA * (bg0 * gC0A + bg1 * gC1A + bg2 * gC2A), -TfB * (bg0 * gC0B + bg1 * gC1B + bg2 * gC2B));

    const uint32_t q_base = s_q + warp * Q::WARP;
    const uint32_t coef_base = s_coef + warp * 64 * 16;
    const uint32_t slot_base = s_slot + warp * SLOTS * 4;
    sts128(coef_base + lane * 32, make_float4(gC0A, gC0B, gC1A, gC1B));           // (A, B) pairs per channel: the
    sts128(coef_base + lane * 32 + 16, make_float4(gC2A, gC2B, gDA, gDB));         // second phase multiplies them packed
    const uint32_t qwG = q_base + lane * Q::ROW, qwD = qwG + 32 * Q::ROW;     // this lane's rows of the two queue arrays
    const float Xc = X0f + 3.5f, Yc = Y0f + 3.5f;
    __syncwarp();

    u64 T2 = pk(TfA, TfB);
    // Upstream gradients are per-pixel constants and the blend is linear in the channels, so the five "colour behind
    // this splat" recurrences of the package collapse into ONE on the projected scalar s_j = gC.rgb_j + gD*depth_j + gA:
    // dL/dalpha_j = T_j * (s_j - behind_j) + bg term.
    u64 behind = bc(0.f);
    int nq = 0;

    RingState rs;
    for (int it = 0; it < nb; it++) {
        mbar_wait(a_full + 8 * rs.stage, rs.phase);
        const int base = (nb - 1 - it) * BATCH;
        if ((uint32_t)base < wmax) {                      // otherwise the whole stage is past this warp's last contributor
            const int n = min(BATCH, (int)nproc - base);
            const uint32_t sr = s_rec + rs.stage * STAGE_BYTES;
            uint32_t m[BATCH / 32];
            stage_masks(sr, n, lane, X0f, Y0f, m);
#pragma unroll
            for (int i = BATCH / 32 - 1; i >= 0; i--) {
                uint32_t bal = m[i];
                const uint32_t rg = sr + i * 32 * REC_BYTES, pos0 = (uint32_t)(base + i * 32);
                // two visits per iteration, from the back: everything but the T / behind recurrences and the queue slot is
                // independent between them (bwd_front), so the two instruction streams interleave
                while (bal) {
                    if (PAIR && nq > SLOTS - 2) { __syncwarp(); flush_queue<SLOTS>(q_base, coef_base, slot_base, nq, lane, Xc, Yc, tile_list, recs, sg); __syncwarp(); nq = 0; }
                    const int j0 = hibit(bal);
                    const uint32_t b0 = 1u << j0;
                    bal &= ~b0;
                    const bool two = bal != 0;
                    const int j1 = hibit(two ? bal : b0);        // (a select on the mask, not a branch around the bfind)
                    bal &= ~(1u << j1);
                    if (PAIR) {
                        const BwdFront g0 = bwd_front(rg + j0 * REC_BYTES, pos0 + j0, pxf, py2, lcA, lcB, gC0, gC1, gC2, gD, gA, bgT);
                        const BwdFront g1 = bwd_front(rg + j1 * REC_BYTES, pos0 + j1, pxf, py2, lcA, lcB, gC0, gC1, gC2, gD, gA, bgT, two);
                        bwd_back(g0, T2, behind, qwG + nq * 8, qwD + nq * 8);
                        bwd_back(g1, T2, behind, qwG + nq * 8 + 8, qwD + nq * 8 + 8);
                        if (lane == 0) {
                            asm volatile("st.shared.u32 [%0], %1;" ::"r"(slot_base + nq * 4), "r"(pos0 + j0) : "memory");
                            asm volatile("st.shared.u32 [%0+4], %1;" ::"r"(slot_base + nq * 4), "r"(pos0 + j1) : "memory");
                        }
                        nq += two ? 2 : 1;
                        continue;
                    }
                    const BwdFront f0 = bwd_front(rg + j0 * REC_BYTES, pos0 + j0, pxf, py2, lcA, lcB, gC0, gC1, gC2, gD, gA, bgT);
                    const BwdFront f1 = bwd_front(rg + j1 * REC_BYTES, pos0 + j1, pxf, py2, lcA, lcB, gC0, gC1, gC2, gD, gA, bgT);
                    if (!VOTE || __any_sync(0xFFFFFFFFu, f0.any)) {
                        bwd_back(f0, T2, behind, qwG + nq * 8, qwD + nq * 8);
                        if (lane == 0) asm volatile("st.shared.u32 [%0], %1;" ::"r"(slot_base + nq * 4), "r"(pos0 + j0) : "memory");
                        if (++nq == SLOTS) { __syncwarp(); flush_queue<SLOTS>(q_base, coef_base, slot_base, SLOTS, lane, Xc, Yc, tile_list, recs, sg); __syncwarp(); nq = 0; }
                    }
                    if (two && (!VOTE || __any_sync(0xFFFFFFFFu, f1.any))) {
                        bwd_back(f1, T2, behind, qwG + nq * 8, qwD + nq * 8);
                        if (lane == 0) asm volatile("st.shared.u32 [%0], %1;" ::"r"(slot_base + nq * 4), "r"(pos0 + j1) : "memory");
                        if (++nq == SLOTS) { __syncwarp(); flush_queue<SLOTS>(q_base, coef_base, slot_base, SLOTS, lane, Xc, Yc, tile_list, recs, sg); __syncwarp(); nq = 0; }
                    }
                }
            }
        }
        // release the stage; the last of the four warps to do so refills it
        __syncwarp();
        uint32_t tot = 0;
        if (lane == 0) { __threadfence_block(); tot = atomicAdd(&s_cnt[rs.stage], 1u) + 1u; }
        tot = __shfl_sync(0xFFFFFFFFu, tot, 0);
        if (tot == NMATH) {
            if (lane == 0) { __threadfence_block(); s_cnt[rs.stage] = 0; }       // acquire side of the stage hand-over
            __syncwarp();
            if (it + STAGES < nb) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // the stage was read through the generic proxy
                produce(it + STAGES, rs.stage);
            }
        }
        rs.advance(STAGES);
    }
    if (nq > 0) {
        __syncwarp();
        flush_queue<SLOTS>(q_base, coef_base, slot_base, nq, lane, Xc, Yc, tile_list, recs, sg);
    }
}

constexpr size_t bwd_smem_bytes(int stages, int slots) {
    return (size_t)stages * STAGE_BYTES + NMATH * 64 * (size_t)(slots + 1) * 8 + NMATH * 64 * 16 + NMATH * (size_t)slots * 4 +
           8 * (size_t)stages + 4 * (size_t)stages + 16;
}

bool gather_tma() {       // GS_B200_GATHER=tma selects the TMA bulk-copy gather instead of the cp.async default
    static const bool tma = []() { const char* e = getenv("GS_B200_GATHER"); return e && e[0] == 't'; }();
    return tma;
}

int env_int(const char* name, int dflt) {
    const char* e = getenv(name);
    return (e && *e) ? atoi(e) : dflt;
}

}  // namespace

// round-1 kernels (gs_render.cu), kept selectable for A/B measurements: GS_B200_COMPOSITE=r1
int gs_launch_render_forward_r1(const ViewArgs& va, const SplatRec* recs, const uint32_t* point_list,
                                const uint32_t* ranges, float* out_color, float* out_depth, float* out_alpha,
                                uint32_t* n_contrib, float* final_T, cudaStream_t s);
int gs_launch_render_backward_r1(const ViewArgs& va, const SplatRec* recs, const uint32_t* point_list,
                                 const uint32_t* ranges, const uint32_t* n_contrib, const float* final_T,
                                 const float* dL_dcolor, const float* dL_ddepth, const float* dL_dalpha,
                                 SplatGrad* sg, cudaStream_t s);

#include <atomic>
static std::atomic<int> g_composite_mode{[]() { const char* e = getenv("GS_B200_COMPOSITE"); return (e && e[0] == 'r') ? 1 : 0; }()};
static bool use_r1() { return g_composite_mode.load(std::memory_order_relaxed) == 1; }
extern "C" int32_t gs_b200_debug_set_composite(int32_t mode) {
    if (mode != 0 && mode != 1) { gs_set_error("composite mode must be 0 (round-2 kernels) or 1 (round-1 kernels)"); return 1; }
    g_composite_mode.store(mode);
    return 0;
}

int gs_launch_render_forward(const ViewArgs& va, const SplatRec* recs, const uint32_t* point_list,
                             const uint32_t* ranges, float* out_color, float* out_depth, float* out_alpha,
                             uint32_t* n_contrib, float* final_T, cudaStream_t s) {
    if (use_r1()) return gs_launch_render_forward_r1(va, recs, point_list, ranges, out_color, out_depth, out_alpha, n_contrib, final_T, s);
    dim3 grid(va.tiles_x, va.tiles_y);
    // ring depth: GS_B200_FWD_STAGES (2/3/4, cp.async gather); the TMA gather (GS_B200_GATHER=tma) is kept at its best
    // measured depth for A/B runs
    static const int stages = env_int("GS_B200_FWD_STAGES", 3);
    static const bool stopvote = env_int("GS_B200_FWD_STOPVOTE", 1) != 0;   // one warp vote per visit instead of per-pixel termination selects
#define FWD(ST, TM, SV) composite_forward_kernel<ST, TM, SV><<<grid, NTHREADS, 0, s>>>(va, recs, point_list, ranges, out_color, out_depth, out_alpha, n_contrib, final_T)
    if (gather_tma()) FWD(3, true, false);
    else if (stages == 2) FWD(2, false, false);
    else if (stages == 4) FWD(4, false, false);
    else if (stopvote) FWD(3, false, true);
    else FWD(3, false, false);
#undef FWD
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int gs_launch_render_backward(const ViewArgs& va, const SplatRec* recs, const uint32_t* point_list,
                              const uint32_t* ranges, const uint32_t* n_contrib, const float* final_T,
                              const float* dL_dcolor, const float* dL_ddepth, const float* dL_dalpha,
                              SplatGrad* sg, cudaStream_t s) {
    if (use_r1()) return gs_launch_render_backward_r1(va, recs, point_list, ranges, n_contrib, final_T, dL_dcolor, dL_ddepth, dL_dalpha, sg, s);
    dim3 grid(va.tiles_x, va.tiles_y);
    // Selectable: ring depth (GS_B200_BWD_STAGES 2/3) and the TMA gather (GS_B200_GATHER=tma).
    static const int stages = env_int("GS_B200_BWD_STAGES", 2);
    static const bool pair = env_int("GS_B200_BWD_PAIR", 1) != 0;      // both visits of an iteration unconditional (second masked)
#define BWD(ST, TM, PR)                                                                                                    \
    do {                                                                                                                   \
        static const cudaError_t attr = cudaFuncSetAttribute(composite_backward_kernel<ST, 16, 4, false, TM, PR>,          \
                                                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwd_smem_bytes(ST, 16)); \
        GS_CUDA_CHECK(attr);                                                                                               \
        composite_backward_kernel<ST, 16, 4, false, TM, PR><<<grid, NTHREADS, bwd_smem_bytes(ST, 16), s>>>(va, recs, point_list, ranges, n_contrib, final_T, dL_dcolor, dL_ddepth, dL_dalpha, sg); \
    } while (0)
    if (gather_tma()) BWD(2, true, false);
    else if (stages == 3) BWD(3, false, false);
    else if (pair) BWD(2, false, true);
    else BWD(2, false, false);
#undef BWD
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
