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
//  * the tile's records are gathered by three 16 B cp.async per record into a ring of
//    shared-memory stages, each completed on an mbarrier; a warp releases a stage with one
//    shared-memory atomic and the last of the four to release it refills it.
//    There is no __syncthreads() in the main loops;
//  * each warp decides by itself which records of a stage can reach
//    alpha >= 1/255 inside its quadrant (exact minimum of the quadratic form over
//    the 8x8 rectangle + slack): one test per lane and record, four ballots per
//    128-record stage, then the warp walks only the set bits;
//  * backward, per visit, only TWO values per pixel leave the lanes:
//    G*dL/dalpha and alpha*T.  They are queued in shared memory ([pixel][slot])
//    and, every 16 visits and at the end of each stage, a second phase with lanes = (slot, half-quadrant)
//    turns them into the ten per-splat sums (six image moments of G*dL/dalpha in
//    pixel-local coordinates, four colour/depth sums against per-pixel upstream
//    gradients) with plain FFMAs and no cross-lane traffic beyond one final
//    shfl.xor — the 12-SHFL transpose reduction per (warp, splat) of round 1 is
//    gone.  The sums stop in a per-stage block of fp32 partials in shared memory; when
//    the stage is released, its last warp adds the partials of the (up to four) quadrants
//    of each splat in fp64, in fixed warp order, and ONE fp64 red.global.add per value and
//    (tile, splat) leaves the CTA (SplatGrad in gs_common.cuh says why fp64).
#include "gs_common.cuh"

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

// ---- mbarrier helpers ---------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
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
__device__ __forceinline__ float lds32(uint32_t addr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t ldsu32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts32(uint32_t addr, float a) {
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(a) : "memory");
}
// fp64 add to global memory that returns nothing.  atomicAdd(double*) with its result unused compiles to a returning
// ATOMG inside combine_stage, and the warp then waits for each reply; red.global compiles to REDG, which it does not.
__device__ __forceinline__ void red_add_f64(double* p, double v) {
    asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
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

// gather of one stage: ids (coalesced LDG), then three 16 B cp.async (LDGSTS) per record and lane, and one
// cp.async.mbarrier.arrive.noinc per lane, so the stage's mbarrier expects STAGE_ARRIVALS = 32 arrivals.  (One 48 B
// bulk copy per record through the TMA engine would be fewer copies, but UBLKCP takes its operands from uniform
// registers, so a per-lane gather serialises into a ~9-instruction loop per record inside the issuing warp, whereas the
// three LDGSTS are one warp-wide instruction each.)
constexpr uint32_t STAGE_ARRIVALS = 32;
template <bool KEEP_IDS>
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

// The blend, written for the common case "no pixel of the warp terminates at this visit": a pixel that does not take
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

// Ring depth of the forward: three 6 KB stages of static shared memory (two and four were no faster, DESIGN.md 5.1).
constexpr int FWD_RING_STAGES = 3;
// The shipped backward: ring depth, queued visits per flush, CTAs per SM.  2 x 6 KB ring + 20 KB partial block + 34 KB
// queue + 4 KB upstream gradients = 70.4 KB, three CTAs per SM (an H100 SM has 228 KB of shared memory and reserves
// 1 KB per CTA).  Measured on an H100 against one partial block per stage (92.6 KB, two CTAs per SM): 0.654-0.661
// against 0.739 ms per config-1 view.  A third ring stage would take 76.5 KB and fall back to two CTAs per SM.
constexpr int BWD_STAGES = 2, BWD_SLOTS = 16, BWD_MINB = 3;

// =================================================================================================
// forward
// =================================================================================================
__global__ void __launch_bounds__(NTHREADS)
composite_forward_kernel(ViewArgs va, const SplatRec* __restrict__ recs, const uint32_t* __restrict__ point_list,
                         const uint32_t* __restrict__ ranges, float* __restrict__ out_color,
                         float* __restrict__ out_depth, float* __restrict__ out_alpha,
                         uint32_t* __restrict__ n_contrib, float* __restrict__ final_T) {
    __shared__ __align__(128) unsigned char s_rec_raw[FWD_RING_STAGES * STAGE_BYTES];
    __shared__ __align__(8) u64 s_full[FWD_RING_STAGES];
    __shared__ uint32_t s_cnt[FWD_RING_STAGES], s_stop;
    const uint32_t s_rec = (uint32_t)__cvta_generic_to_shared(s_rec_raw);
    const uint32_t a_full = (uint32_t)__cvta_generic_to_shared(s_full);
    const uint32_t a_stop = (uint32_t)__cvta_generic_to_shared(&s_stop);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tile = blockIdx.y * va.tiles_x + blockIdx.x;
    const uint32_t start = ranges[2 * tile], end = ranges[2 * tile + 1];
    const int len = (int)(end - start);
    const int nb = (len + BATCH - 1) / BATCH;

    if (tid == 0) {
        for (int i = 0; i < FWD_RING_STAGES; i++) { mbar_init(a_full + 8 * i, STAGE_ARRIVALS); s_cnt[i] = 0; }
        s_stop = 0xFFFFFFFFu;
        mbar_fence_init();
    }
    __syncthreads();
    // first fill of the ring: warp w gathers batch w (afterwards the LAST warp to finish a stage refills it)
    if (warp < FWD_RING_STAGES && warp < nb)
        produce_stage<false>(recs, point_list + start + warp * BATCH, min(BATCH, len - warp * BATCH), s_rec + warp * STAGE_BYTES, 0u,
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
                    fwd_back_sv(f0, fwd_live(lo(f0.p2), lo(f0.al2)), fwd_live(hi(f0.p2), hi(f0.al2)), ra0, pos0 + j0,
                                TA, TB, acc, lastA, lastB, pyfA, pyfB);
                    // visit 1's front half saw the row coordinates from before visit 0: drop pixels that just terminated
                    // (`two` false: j1 == j0 and the visit is masked off as a whole)
                    fwd_back_sv(f1, two && fwd_live(lo(f1.p2), lo(f1.al2)) && (pyfA == pyfA), two && fwd_live(hi(f1.p2), hi(f1.al2)) && (pyfB == pyfB),
                                ra1, pos0 + j1, TA, TB, acc, lastA, lastB, pyfA, pyfB);
                }
                if (__all_sync(0xFFFFFFFFu, (pyfA != pyfA) && (pyfB != pyfB))) { warp_done = true; break; }
            }
        }
        // release the stage; the last of the four warps to do so refills it with batch b + FWD_RING_STAGES.  Each release
        // carries the warp's "all my pixels have terminated" bit: when all four say so the tile is finished, nothing is
        // gathered any more and the stop batch is published (a function of b only, so concurrent refills cannot disagree).
        __syncwarp();
        uint32_t tot = 0;
        if (lane == 0) { __threadfence_block(); tot = atomicAdd(&s_cnt[rs.stage], 1u + (warp_done ? 0x100u : 0u)) + 1u + (warp_done ? 0x100u : 0u); }
        tot = __shfl_sync(0xFFFFFFFFu, tot, 0);
        if ((tot & 0xFFu) == NMATH) {
            const int nbatch = b + FWD_RING_STAGES;
            // acquire side of the hand-over (release = the fence before each warp's atomic): the other warps' reads of
            // the stage happen before the refill below overwrites it
            if (lane == 0) { __threadfence_block(); s_cnt[rs.stage] = 0; }
            __syncwarp();
            if (nbatch < nb) {
                if ((tot >> 8) == NMATH) {
                    if (lane == 0) { atomicMin(&s_stop, (uint32_t)nbatch); __threadfence_block(); mbar_arrive_n(a_full + 8 * rs.stage, STAGE_ARRIVALS); }
                } else {
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // the stage was read through the generic proxy
                    produce_stage<false>(recs, point_list + start + nbatch * BATCH, min(BATCH, len - nbatch * BATCH),
                                         s_rec + rs.stage * STAGE_BYTES, 0u, a_full + 8 * rs.stage, lane);
                }
            }
        }
        rs.advance(FWD_RING_STAGES);
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

// Partial block: the ten per-splat sums of every (warp, record) the warp visited in one stage, fp32,
// [warp][value][record] (value-major, so the combine's lanes = records read consecutive words).  ONE block serves both
// ring stages (see the gate in composite_backward_kernel).  Each ring stage has its own hit-mask block
// [warp][BATCH / 32], which says which partials exist (the partial block is never cleared).
constexpr int NVAL = 10;
constexpr uint32_t PART_BYTES = NMATH * NVAL * BATCH * 4;
constexpr uint32_t MASK_BYTES = NMATH * (BATCH / 32) * 4;

// Second phase of the backward: lanes = (slot, part).  Each lane sums, over its SLOTS pixel pairs (pixel A = (x, y),
// pixel B = (x, y+4) of first-phase lane 8y+x), the queued (G*dL/dalpha, alpha*T) of its slot against pixel-local
// coordinates and the per-pixel upstream gradients; the parts are then added with shfl.xor and the ten sums of each
// slot are stored, without atomics, into the warp's row of the partial block (a warp visits a record at most once per
// stage).  Those stores wait until the block is free: phase `free_parity` of the mbarrier `free_bar` has completed.
template <int SLOTS>
__device__ __noinline__ void flush_queue(uint32_t q_base, uint32_t coef_base, uint32_t slot_base, int nq, int lane,
                                         float Xc, float Yc, uint32_t s_stage, uint32_t s_part, uint32_t free_bar,
                                         uint32_t free_parity) {
    using Q = QGeom<SLOTS>;
    const int slot = lane & (SLOTS - 1), part = lane / SLOTS;
    // a slot remembers only the record index of its splat in the stage (one 4 B store per visit by lane 0); mean2D and
    // opacity come from the record, which stays in the ring until the warp releases the stage
    uint32_t rec = 0u;
    float4 si = make_float4(0.f, 0.f, 0.f, 0.f);                // mean2D.x, mean2D.y, -, opacity
    if (slot < nq) {
        rec = ldsu32(slot_base + slot * 4);
        const float4 g = lds128(s_stage + rec * REC_BYTES);
        si = make_float4(g.x, g.y, 0.f, lds32(s_stage + rec * REC_BYTES + 28));
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
    mbar_wait(free_bar, free_parity);
    if (slot < nq) {
        // pixel = centre + L, d = mean2D - pixel = u - L with u = mean2D - centre
        const float u = si.x - Xc, v = si.y - Yc, o = si.w;
        // the ten sums of the splat, in the order of the non-padding doubles of its SplatGrad record
        const float val[NVAL] = {o * (u * M0 - M1),                                   // sum w dx
                                 o * (v * M0 - My),                                   // sum w dy
                                 Cd,                                                  // dL/ddepth
                                 o * (fmaf(u, fmaf(u, M0, -2.f * M1), M2)),           // sum w dx dx
                                 o * (fmaf(u, fmaf(v, M0, -My), fmaf(-v, M1, Mxy))),  // sum w dx dy
                                 o * (fmaf(v, fmaf(v, M0, -2.f * My), Myy)),          // sum w dy dy
                                 M0,                                                  // dL/dopacity (sum G dL/dalpha)
                                 Cr, Cg, Cb};                                         // dL/drgb
        // every part of the slot holds all ten sums: each stores every PARTS-th of them
#pragma unroll
        for (int k = 0; k < NVAL; k++)
            if (k % Q::PARTS == part) sts32(s_part + (k * BATCH + rec) * 4, val[k]);
    }
}

// The stage's splats leave the CTA here, run by the last warp to release the stage; lanes = records.  Per record hit
// by any quadrant, the partials of the warps that hit it are converted to fp64 and added in warp order 0, 1, 2, 3, then
// ONE set of ten fp64 reds goes to its SplatGrad record (sm_90 has no vector fp64 red).  A sum of up to four fp32 values
// in fp64 is exact unless their exponents lie more than 29 bits apart, so SplatGrad receives, to fp64 rounding, what
// one set of reds per (quadrant, splat) would add -- with one set per (tile, splat) instead.
__device__ __noinline__ void combine_stage(uint32_t s_part, uint32_t s_mask, int lane, const uint32_t* __restrict__ list,
                                           SplatGrad* __restrict__ sg) {
    uint32_t hit[BATCH / 32], gid[BATCH / 32];
#pragma unroll
    for (int i = 0; i < BATCH / 32; i++) {              // bit w of hit[i]: warp w holds a partial of record i*32 + lane
        uint32_t h = 0u;
#pragma unroll
        for (int w = 0; w < NMATH; w++) h |= ((ldsu32(s_mask + (w * (BATCH / 32) + i) * 4) >> lane) & 1u) << w;
        hit[i] = h;
        gid[i] = h ? __ldg(list + i * 32 + lane) : 0u;
    }
#pragma unroll
    for (int i = 0; i < BATCH / 32; i++) {
        if (!hit[i]) continue;
        double* dst = reinterpret_cast<double*>(sg + gid[i]);
        const uint32_t pa = s_part + (i * 32 + lane) * 4;
#pragma unroll
        for (int k = 0; k < NVAL; k++) {
            double s = 0.0;
#pragma unroll
            for (int w = 0; w < NMATH; w++) {           // absent partials are stale words: selected away, never added
                const float p = lds32(pa + (w * NVAL + k) * BATCH * 4);
                s += ((hit[i] >> w) & 1u) ? (double)p : 0.0;
            }
            red_add_f64(dst + (k < 3 ? k : k + 1), s);   // skips the padding double after dL/ddepth
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

// Every loop iteration runs BOTH visits; when the group has an odd number of hits the second one is masked off
// (alpha = G = 0: T, behind and the queued values are then unchanged / zero, and its queue slot is not consumed) and the
// queue is checked once per iteration (flushed early at SLOTS - 1) -- one branch region per iteration instead of three.
//
// One partial block serves every iteration, behind a gate: the mbarrier a_free completes phase `it` when the combine of
// iteration `it` has read the block, and flush_queue waits for phase it - 1 before it stores partials of iteration
// `it`.  A warp waits there only when it has partials to store, so a warp that runs ahead still computes its stage
// masks, its first-phase visits and the second-phase sums of its first flush before it blocks.  No deadlock: a waiting
// warp in iteration `it` has released stage it - 1, so the last warp to release it, which runs that combine, is not
// among the waiters; and the warps still in iteration it - 1 wait (if at all) for the combine of it - 2, which has
// completed, because stage `it` was refilled after it.  That also bounds the phases in flight: when a warp enters
// iteration `it`, at most the combine of it - 1 is pending (the refill of a stage follows its combine), so the parity
// wait cannot alias an older phase -- which holds for a ring of at most two stages.
template <int STAGES, int SLOTS, int MINB>
__global__ void __launch_bounds__(NTHREADS, MINB)
composite_backward_kernel(ViewArgs va, const SplatRec* __restrict__ recs, const uint32_t* __restrict__ point_list,
                          const uint32_t* __restrict__ ranges, const uint32_t* __restrict__ n_contrib,
                          const float* __restrict__ final_T, const float* __restrict__ dL_dcolor,
                          const float* __restrict__ dL_ddepth, const float* __restrict__ dL_dalpha,
                          SplatGrad* __restrict__ sg) {
    static_assert(STAGES <= 2, "the partial-block gate waits on mbarrier parity: one combine in flight at most");
    using Q = QGeom<SLOTS>;
    // dynamic shared memory: ring | partial block | hit masks per stage | queue | per-pixel upstream gradients |
    // slot info | barriers (full per stage, free) | counters | wmax
    extern __shared__ __align__(128) unsigned char smem[];
    const uint32_t s_rec = (uint32_t)__cvta_generic_to_shared(smem);
    const uint32_t s_part = s_rec + STAGES * STAGE_BYTES;
    const uint32_t s_mask = s_part + PART_BYTES;
    const uint32_t s_q = s_mask + STAGES * MASK_BYTES;
    const uint32_t s_coef = s_q + NMATH * Q::WARP;
    const uint32_t s_slot = s_coef + NMATH * 64 * 16;
    const uint32_t a_full = s_slot + NMATH * SLOTS * 4;
    const uint32_t a_free = a_full + 8 * STAGES;
    uint32_t* s_cnt = reinterpret_cast<uint32_t*>(smem + (a_free + 8 - s_rec));
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
        for (int i = 0; i < STAGES; i++) { mbar_init(a_full + 8 * i, STAGE_ARRIVALS); s_cnt[i] = 0; }
        mbar_init(a_free, 1);
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
        produce_stage<false>(recs, point_list + start + base, min(BATCH, (int)nproc - base), s_rec + stage * STAGE_BYTES,
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
        const uint32_t sr = s_rec + rs.stage * STAGE_BYTES;
        const uint32_t msk = s_mask + rs.stage * MASK_BYTES;
        const uint32_t s_pw = s_part + warp * NVAL * BATCH * 4;      // this warp's rows of the partial block
        // phase it - 1 of a_free: the combine of iteration it - 1 has read the block (for it = 0, parity 1 of a fresh
        // mbarrier counts as complete)
        const uint32_t free_par = (uint32_t)(it + 1) & 1u;
        if ((uint32_t)base < wmax) {                      // otherwise the whole stage is past this warp's last contributor
            const int n = min(BATCH, (int)nproc - base);
            uint32_t m[BATCH / 32];
            stage_masks(sr, n, lane, X0f, Y0f, m);
            // the stage's own mask block: its last reader, the combine of iteration it - STAGES, ran before the refill
            if (lane == 0)
                asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(msk + warp * 16), "r"(m[0]), "r"(m[1]),
                             "r"(m[2]), "r"(m[3]) : "memory");
#pragma unroll
            for (int i = BATCH / 32 - 1; i >= 0; i--) {
                uint32_t bal = m[i];
                const uint32_t rg = sr + i * 32 * REC_BYTES, r0 = (uint32_t)(i * 32), pos0 = (uint32_t)base + r0;
                // two visits per iteration, from the back: everything but the T / behind recurrences and the queue slot is
                // independent between them (bwd_front), so the two instruction streams interleave
                while (bal) {
                    if (nq > SLOTS - 2) { __syncwarp(); flush_queue<SLOTS>(q_base, coef_base, slot_base, nq, lane, Xc, Yc, sr, s_pw, a_free, free_par); __syncwarp(); nq = 0; }
                    const int j0 = hibit(bal);
                    const uint32_t b0 = 1u << j0;
                    bal &= ~b0;
                    const bool two = bal != 0;
                    const int j1 = hibit(two ? bal : b0);        // (a select on the mask, not a branch around the bfind)
                    bal &= ~(1u << j1);
                    const BwdFront g0 = bwd_front(rg + j0 * REC_BYTES, pos0 + j0, pxf, py2, lcA, lcB, gC0, gC1, gC2, gD, gA, bgT);
                    const BwdFront g1 = bwd_front(rg + j1 * REC_BYTES, pos0 + j1, pxf, py2, lcA, lcB, gC0, gC1, gC2, gD, gA, bgT, two);
                    bwd_back(g0, T2, behind, qwG + nq * 8, qwD + nq * 8);
                    bwd_back(g1, T2, behind, qwG + nq * 8 + 8, qwD + nq * 8 + 8);
                    if (lane == 0) {
                        asm volatile("st.shared.u32 [%0], %1;" ::"r"(slot_base + nq * 4), "r"(r0 + j0) : "memory");
                        asm volatile("st.shared.u32 [%0+4], %1;" ::"r"(slot_base + nq * 4), "r"(r0 + j1) : "memory");
                    }
                    nq += two ? 2 : 1;
                }
            }
            // every visit of the stage is flushed before the stage is released, so the partial block holds the whole
            // stage once all four warps have released it
            if (nq > 0) { __syncwarp(); flush_queue<SLOTS>(q_base, coef_base, slot_base, nq, lane, Xc, Yc, sr, s_pw, a_free, free_par); nq = 0; }
        } else if (lane == 0) {
            asm volatile("st.shared.v4.u32 [%0], {%1,%1,%1,%1};" ::"r"(msk + warp * 16), "r"(0u) : "memory");
        }
        // release the stage; the last of the four warps to do so combines the partial block, frees it and refills the
        // stage
        __syncwarp();
        uint32_t tot = 0;
        if (lane == 0) { __threadfence_block(); tot = atomicAdd(&s_cnt[rs.stage], 1u) + 1u; }
        tot = __shfl_sync(0xFFFFFFFFu, tot, 0);
        if (tot == NMATH) {
            if (lane == 0) { __threadfence_block(); s_cnt[rs.stage] = 0; }       // acquire side of the stage hand-over
            __syncwarp();
            combine_stage(s_part, msk, lane, tile_list + base, sg);
            __syncwarp();
            if (lane == 0) mbar_arrive(a_free);          // release: the combine's reads of the block precede later stores
            // the refill comes after the combine: the stage's mask block is rewritten once its records arrive, and a warp
            // can enter iteration it + STAGES only when the combine of iteration it is complete (see the gate above)
            if (it + STAGES < nb) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // the stage was read through the generic proxy
                produce(it + STAGES, rs.stage);
            }
        }
        rs.advance(STAGES);
    }
}

constexpr size_t bwd_smem_bytes(int stages, int slots) {
    return (size_t)stages * (STAGE_BYTES + MASK_BYTES) + PART_BYTES + NMATH * 64 * (size_t)(slots + 1) * 8 +
           NMATH * 64 * 16 + NMATH * (size_t)slots * 4 + 8 * (size_t)stages + 8 + 4 * (size_t)stages + 16;
}

constexpr size_t BWD_SMEM = bwd_smem_bytes(BWD_STAGES, BWD_SLOTS);
static_assert(BWD_MINB * (BWD_SMEM + 1024) <= 228 * 1024, "the backward's shared memory must fit BWD_MINB CTAs per SM");
#define BWD_KERNEL composite_backward_kernel<BWD_STAGES, BWD_SLOTS, BWD_MINB>

// Dynamic shared memory beyond 48 KB must be allowed per kernel, and three CTAs of 70 KB need the largest shared-memory
// carveout (228 KB) of the unified L1.  Set once, before the first launch or occupancy query.
cudaError_t bwd_kernel_attributes() {
    static const cudaError_t err = []() {
        cudaError_t e = cudaFuncSetAttribute(BWD_KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_SMEM);
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(BWD_KERNEL, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        return e;
    }();
    return err;
}

}  // namespace

int gs_launch_render_forward(const ViewArgs& va, const SplatRec* recs, const uint32_t* point_list,
                             const uint32_t* ranges, float* out_color, float* out_depth, float* out_alpha,
                             uint32_t* n_contrib, float* final_T, cudaStream_t s) {
    dim3 grid(va.tiles_x, va.tiles_y);
    composite_forward_kernel<<<grid, NTHREADS, 0, s>>>(va, recs, point_list, ranges, out_color, out_depth, out_alpha,
                                                       n_contrib, final_T);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int gs_launch_render_backward(const ViewArgs& va, const SplatRec* recs, const uint32_t* point_list,
                              const uint32_t* ranges, const uint32_t* n_contrib, const float* final_T,
                              const float* dL_dcolor, const float* dL_ddepth, const float* dL_dalpha,
                              SplatGrad* sg, cudaStream_t s) {
    dim3 grid(va.tiles_x, va.tiles_y);
    GS_CUDA_CHECK(bwd_kernel_attributes());
    BWD_KERNEL<<<grid, NTHREADS, BWD_SMEM, s>>>(va, recs, point_list, ranges, n_contrib, final_T, dL_dcolor, dL_ddepth,
                                                dL_dalpha, sg);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

extern "C" int32_t gs_b200_composite_bwd_occupancy(int32_t* ctas_per_sm, int32_t* smem_bytes) {
    if (!ctas_per_sm || !smem_bytes) { gs_set_error("composite_bwd_occupancy: NULL"); return 1; }
    GS_CUDA_CHECK(bwd_kernel_attributes());
    int n = 0;
    GS_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, BWD_KERNEL, NTHREADS, BWD_SMEM));
    *ctas_per_sm = n;
    *smem_bytes = (int32_t)BWD_SMEM;
    return 0;
}
