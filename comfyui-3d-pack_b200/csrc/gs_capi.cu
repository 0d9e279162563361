// C ABI of the rasterizer (include/gs_b200.h): orchestration of the kernels.
// Replaces RasterizeGaussiansCUDA / RasterizeGaussiansBackwardCUDA of
// diff_gaussian_rasterization (reached from main_3DGS_renderer.py:927-936 and
// main_3DGS.py:205).
#include "../../include/gs_b200.h"
#include "gs_common.cuh"

#include <stdarg.h>
#include <string.h>
#include <algorithm>
#include <memory>
#include <vector>

static thread_local char g_err[512] = "";

void gs_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

#include <atomic>
#include <mutex>
static std::atomic<long long> g_launches{0};
void gs_count_launches(int n) { g_launches += n; }

namespace {

// ---- per-stage CUDA-event timing (off by default; bench.py turns it on for a profiling pass)
struct StageEv { int stage; cudaEvent_t a, b; };
static std::mutex g_prof_mu;
static bool g_prof_on = false;
static std::vector<StageEv> g_prof;
struct StageTimer {
    cudaStream_t s; int idx = -1;
    StageTimer(int stage, cudaStream_t s_) : s(s_) {
        if (!g_prof_on) return;
        std::lock_guard<std::mutex> l(g_prof_mu);
        StageEv e; e.stage = stage;
        if (cudaEventCreate(&e.a) != cudaSuccess || cudaEventCreate(&e.b) != cudaSuccess) return;
        cudaEventRecord(e.a, s);
        g_prof.push_back(e); idx = (int)g_prof.size() - 1;
    }
    ~StageTimer() {
        if (idx < 0) return;
        std::lock_guard<std::mutex> l(g_prof_mu);
        if (idx < (int)g_prof.size()) cudaEventRecord(g_prof[idx].b, s);
    }
};

struct Allocator {
    gs_b200_alloc_fn fn;
    void* user;
    cudaStream_t stream;
    std::vector<void*> scratch;     // internally allocated scratch, freed at scope end
    bool failed = false;

    void* get(int tag, size_t bytes, void** owned_slot = nullptr) {
        if (bytes == 0) bytes = 256;
        bytes = (bytes + 255) & ~(size_t)255;
        void* p = nullptr;
        if (fn) {
            p = fn(user, tag, bytes);
            if (!p) { failed = true; gs_set_error("allocator callback returned NULL for %zu bytes (tag %d)", bytes, tag); }
            return p;
        }
        static thread_local int pool_dev = -1;      // keep freed blocks in the pool across stream syncs
        int devn = 0;
        cudaGetDevice(&devn);
        if (pool_dev != devn) {
            cudaMemPool_t pool;
            if (cudaDeviceGetDefaultMemPool(&pool, devn) == cudaSuccess) {
                unsigned long long thr = ~0ull;
                cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
            }
            pool_dev = devn;
        }
        cudaError_t e = cudaMallocAsync(&p, bytes, stream);
        if (e != cudaSuccess) { failed = true; gs_set_error("cudaMallocAsync(%zu) -> %s", bytes, cudaGetErrorString(e)); return nullptr; }
        if (tag == GS_B200_BUF_SCRATCH) scratch.push_back(p);
        else if (owned_slot) *owned_slot = p;
        return p;
    }
    ~Allocator() {
        for (void* p : scratch) cudaFreeAsync(p, stream);
    }
};

// carve sub-buffers out of one allocation
struct Carver {
    char* base; size_t off = 0;
    explicit Carver(void* b) : base((char*)b) {}
    template <typename T> T* take(size_t count) {
        T* p = (T*)(base + off);
        off += (count * sizeof(T) + 255) & ~(size_t)255;
        return p;
    }
    static size_t need(size_t count, size_t elem) { return (count * elem + 255) & ~(size_t)255; }
};

// fn: the entry point named in the error message
int make_view_args(const char* fn, const gs_b200_view* v, ViewArgs& va) {
    if (!v || !v->bg || !v->viewmatrix || !v->projmatrix || !v->campos) { gs_set_error("%s: NULL view field", fn); return 1; }
    if (v->image_height <= 0 || v->image_width <= 0) { gs_set_error("%s: bad image size", fn); return 1; }
    if (v->sh_degree < 0 || v->sh_degree > 3) { gs_set_error("%s: sh_degree must be 0..3", fn); return 1; }
    va.view = v->viewmatrix; va.proj = v->projmatrix; va.campos = v->campos; va.bg = v->bg;
    va.tanfovx = v->tanfovx; va.tanfovy = v->tanfovy;
    va.W = v->image_width; va.H = v->image_height;
    // fp32 focal, as the oracle: S / (2 tan)
    va.focal_x = (float)va.W / (2.0f * va.tanfovx);
    va.focal_y = (float)va.H / (2.0f * va.tanfovy);
    va.scale_modifier = v->scale_modifier;
    va.tiles_x = (va.W + GS_TILE - 1) / GS_TILE;
    va.tiles_y = (va.H + GS_TILE - 1) / GS_TILE;
    va.sh_degree = v->sh_degree;
    return 0;
}

// fn: the entry point named in the error message (the package's own two messages are kept word for word)
int check_inputs(const char* fn, int N, int M, int sh_degree, const float* means3D, const float* shs,
                 const float* colors_precomp, const float* opacities, const float* scales, const float* rotations,
                 const float* cov3D_precomp) {
    if (N < 0) { gs_set_error("%s: N < 0", fn); return 1; }
    if (N == 0) return 0;      // empty cloud: pointers of empty arrays may legitimately be NULL
    if (!means3D || !opacities) { gs_set_error("%s: means3D/opacities NULL", fn); return 1; }
    if ((shs == nullptr) == (colors_precomp == nullptr)) {
        gs_set_error("Please provide excatly one of either SHs or precomputed colors!"); return 1;
    }
    const bool sr = scales != nullptr || rotations != nullptr;
    if ((sr && cov3D_precomp) || (!sr && !cov3D_precomp) || (sr && (!scales || !rotations))) {
        gs_set_error("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!"); return 1;
    }
    if (shs && M < (sh_degree + 1) * (sh_degree + 1)) { gs_set_error("%s: shs has %d coefficients, sh_degree %d needs %d", fn, M, sh_degree, (sh_degree + 1) * (sh_degree + 1)); return 1; }
    if (shs && M > 16) { gs_set_error("%s: at most 16 SH coefficients (degree 3) supported, got %d", fn, M); return 1; }
    return 0;
}

// The multi-view step's view chunks: nchunks balanced chunks of <= VB views (VB <= 16, one batched preprocess, binning
// and preprocess backward each); chunk k holds views [first(k), first(k) + count(k)).
struct StepChunks {
    int V, nchunks, VB;
    explicit StepChunks(int V_) : V(V_) {
        const int maxv = std::min(gs_preprocess_multi_max_views(), GS_MAX_SEGS);
        nchunks = (V + maxv - 1) / maxv;
        VB = nchunks > 0 ? (V + nchunks - 1) / nchunks : 0;
    }
    int first(int k) const { return VB * k; }
    int count(int k) const { return std::min(VB, V - first(k)); }
};

int bits_for(int n) { int b = 0; while ((1 << b) < n) b++; return b < 1 ? 1 : b; }

unsigned long long* pinned_u64() {
    static thread_local unsigned long long* p = nullptr;
    if (!p) { if (cudaHostAlloc((void**)&p, 64, cudaHostAllocDefault) != cudaSuccess) p = nullptr; }
    return p;
}

#define STAGE_CHECK(dbg, s, what)                                                                     \
    do {                                                                                              \
        if (dbg) {                                                                                    \
            cudaError_t _e = cudaStreamSynchronize(s);                                                \
            if (_e == cudaSuccess) _e = cudaGetLastError();                                           \
            if (_e != cudaSuccess) { gs_set_error("stage %s failed: %s", what, cudaGetErrorString(_e)); return 1; } \
        }                                                                                             \
    } while (0)

}  // namespace

extern "C" {

int32_t gs_b200_abi_version(void) { return GS_B200_ABI_VERSION; }

// tile culling mode: 0 = off (the package's tile lists everywhere), 1 = multi-view step entries only (default),
// 2 = also gs_b200_rasterize_forward.  Images are bit-identical in every mode; see tight_spans() in gs_preprocess.cu.
static int tile_culling_init() {
    const char* e = getenv("GS_B200_TILE_CULLING");
    if (e && *e) { int v = atoi(e); return v < 0 ? 0 : (v > 2 ? 2 : v); }
    return 1;
}
static std::atomic<int> g_tile_culling{tile_culling_init()};
int32_t gs_b200_set_tile_culling(int32_t mode) {
    GS_REQ(mode >= 0 && mode <= 2, "tile culling mode must be 0, 1 or 2");
    g_tile_culling.store(mode);
    return 0;
}
int32_t gs_b200_get_tile_culling(void) { return g_tile_culling.load(); }
int64_t gs_b200_launch_count(void) { return (int64_t)g_launches.load(); }
void gs_b200_profile_enable(int32_t on) {
    std::lock_guard<std::mutex> l(g_prof_mu);
    for (auto& e : g_prof) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); }
    g_prof.clear();
    g_prof_on = on != 0;
}
int32_t gs_b200_profile_read(float* ms_out, int32_t* calls_out) {
    std::lock_guard<std::mutex> l(g_prof_mu);
    for (int i = 0; i < GS_B200_NSTAGES; i++) { if (ms_out) ms_out[i] = 0.f; if (calls_out) calls_out[i] = 0; }
    for (auto& e : g_prof) {
        if (cudaEventSynchronize(e.b) != cudaSuccess) { gs_set_error("profile_read: event sync failed"); return 1; }
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, e.a, e.b) != cudaSuccess) { gs_set_error("profile_read: elapsed failed"); return 1; }
        if (ms_out) ms_out[e.stage] += ms;
        if (calls_out) calls_out[e.stage] += 1;
    }
    return 0;
}
const char* gs_b200_last_error(void) { return g_err; }

// ---- binning of nv views ----------------------------------------------------------------------------------
// Inputs are the preprocess's [nv][N] arrays (one view: the single-view entries; a chunk of views: the multi-view
// step).  Every stage is one launch (or one launch per digit pass) over all nv views.
// Phase A: segmented depth sort -> segmented gather-scan -> ONE D2H of the nv pair totals.
// Phase B (the host has the totals, to size the pair buffers): emit (which also counts the tile sort's digit
// histograms) -> segmented tile sort -> ranges.  View v's pairs are [base[v], base[v+1]) of one chunk buffer.
struct BinA {
    int nv = 0, N = 0, dbg = 0;
    uint32_t *tiles = nullptr, *dkeys = nullptr, *ids = nullptr;          // [nv][N] from the preprocess
    const uint32_t* minkeys = nullptr; int minkey_stride = 0;             // depth-key bias of view v: minkeys[v * stride]
    uint32_t *dkeys_alt = nullptr, *ids_alt = nullptr, *offsets = nullptr;
    unsigned long long* totals = nullptr;                                 // [nv] on the device
    void *sort_scratch = nullptr, *scan_scratch = nullptr;
    const uint32_t *sorted_ids = nullptr, *sorted_dkeys = nullptr;       // [nv][N], set by bin_a
};
static size_t bin_a_bytes(int nv, int N) {
    const size_t nn = (size_t)nv * N;
    return Carver::need(nn, 4) * 3 + Carver::need(nv, 8) + Carver::need(gs_sort_seg_scratch_bytes(nv, (int64_t)nn), 1) +
           Carver::need(gs_scan_seg_scratch_bytes(N, nv), 1);
}
static void carve_bin_a(Carver& c, BinA& b, int nv, int N) {
    const size_t nn = (size_t)nv * N;
    b.nv = nv; b.N = N;
    b.dkeys_alt = c.take<uint32_t>(nn); b.ids_alt = c.take<uint32_t>(nn); b.offsets = c.take<uint32_t>(nn);
    b.totals = c.take<unsigned long long>(nv);
    b.sort_scratch = c.take<char>(gs_sort_seg_scratch_bytes(nv, (int64_t)nn));
    b.scan_scratch = c.take<char>(gs_scan_seg_scratch_bytes(N, nv));
}
static int bin_a(BinA& b, unsigned long long* host_totals, cudaStream_t s) {
    SortSegs sg; sg.n = b.nv;
    for (int v = 0; v <= b.nv; v++) sg.off[v] = (int64_t)v * b.N;
    int in_alt = 0;
    { StageTimer t(1, s);
    if (gs_sort_pairs_segmented(b.dkeys, b.dkeys_alt, b.ids, b.ids_alt, sg, 0, 32, b.sort_scratch, &in_alt, b.minkeys,
                                b.minkey_stride, false, s)) return 1; }
    STAGE_CHECK(b.dbg, s, "depth sort");
    b.sorted_ids = in_alt ? b.ids_alt : b.ids;
    b.sorted_dkeys = in_alt ? b.dkeys_alt : b.dkeys;
    { StageTimer t(2, s);
    if (gs_scan_gather_seg_u32(b.tiles, b.sorted_ids, b.offsets, b.totals, b.N, b.nv, b.scan_scratch, s)) return 1; }
    GS_CUDA_CHECK(cudaMemcpyAsync(host_totals, b.totals, (size_t)b.nv * 8, cudaMemcpyDeviceToHost, s));
    return 0;
}
// per-view pair bases from the totals phase A copied to the host
static int view_spans(int nv, const unsigned long long* host_totals, ViewSpans& vs) {
    vs.n = nv; vs.base[0] = 0;
    for (int v = 0; v < nv; v++) {
        if (host_totals[v] > (unsigned long long)GS_MAX_SEG_KEYS) {
            gs_set_error("too many (tile,splat) pairs in one view: %llu (at most %lld)", host_totals[v], (long long)GS_MAX_SEG_KEYS);
            return 1;
        }
        vs.base[v + 1] = vs.base[v] + (int64_t)host_totals[v];
    }
    return 0;
}
struct BinB { uint32_t *point_list = nullptr, *tile_keys = nullptr, *keys_alt = nullptr, *vals_alt = nullptr; void* sort_scratch = nullptr; };
static size_t bin_b_scratch_bytes(int nv, int64_t P) {
    return Carver::need(P, 4) * 2 + Carver::need(gs_sort_seg_scratch_bytes(nv, P), 1);
}
static void carve_bin_b_scratch(Carver& c, BinB& o, int nv, int64_t P) {
    o.keys_alt = c.take<uint32_t>(P); o.vals_alt = c.take<uint32_t>(P);
    o.sort_scratch = c.take<char>(gs_sort_seg_scratch_bytes(nv, P));
}
// ranges: [nv][tiles][2], zeroed by the caller
static int bin_b(const BinA& a, const ViewSpans& vs, int tiles_x, int tiles_y, const SplatRec* recs, const uint4* spans,
          const BinB& o, uint32_t* ranges, cudaStream_t s) {
    const int64_t P = vs.base[vs.n];
    if (P <= 0) return 0;
    const int ntiles = tiles_x * tiles_y;
    const int tbits = bits_for(ntiles);
    const int npasses = (tbits + 7) / 8;
    // start in the buffer that makes the last pass land in the saved pair
    uint32_t *k0 = (npasses & 1) ? o.keys_alt : o.tile_keys, *v0 = (npasses & 1) ? o.vals_alt : o.point_list;
    uint32_t *k1 = (npasses & 1) ? o.tile_keys : o.keys_alt, *v1 = (npasses & 1) ? o.point_list : o.vals_alt;
    GS_CUDA_CHECK(cudaMemsetAsync(o.sort_scratch, 0, gs_sort_hist_bytes(vs.n), s));
    { StageTimer t(3, s);
    if (gs_launch_emit_multi(recs, spans, a.sorted_ids, a.offsets, a.N, tiles_x, tiles_y, vs, k0, v0,
                             (uint32_t*)o.sort_scratch, npasses, s)) return 1; }
    STAGE_CHECK(a.dbg, s, "emit");
    SortSegs sg; sg.n = vs.n;
    for (int v = 0; v <= vs.n; v++) sg.off[v] = vs.base[v];
    int in_alt = 0;
    { StageTimer t(4, s);
    if (gs_sort_pairs_segmented(k0, k1, v0, v1, sg, 0, tbits, o.sort_scratch, &in_alt, nullptr, 0, true, s)) return 1; }
    STAGE_CHECK(a.dbg, s, "tile sort");
    { StageTimer t(5, s);
    if (gs_launch_ranges_multi(o.tile_keys, vs, ntiles, ranges, s)) return 1; }
    STAGE_CHECK(a.dbg, s, "ranges");
    return 0;
}

// ---- single-view forward: preprocess -> binning phase A (one view) -> D2H of the pair count -> the one host
// round-trip (the pair count sizes the binning buffers) -> binning phase B -> composite.
int32_t gs_b200_rasterize_forward(const gs_b200_view* view, int32_t N, int32_t M, const float* means3D,
                                  const float* shs, const float* colors_precomp, const float* opacities,
                                  const float* scales, const float* rotations, const float* cov3D_precomp,
                                  float* out_color, float* out_depth, float* out_alpha, int32_t* radii,
                                  gs_b200_alloc_fn alloc, void* alloc_user, gs_b200_state* state, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    ViewArgs va;
    if (make_view_args(__func__, view, va)) return 1;
    if (check_inputs(__func__, N, M, view->sh_degree, means3D, shs, colors_precomp, opacities, scales, rotations,
                     cov3D_precomp)) return 1;
    GS_REQ(out_color && out_depth && out_alpha && (N == 0 || radii) && state, "NULL output");
    unsigned long long* host_total = pinned_u64();
    if (!host_total) { gs_set_error("cudaHostAlloc failed"); return 1; }
    const int dbg = view->debug;
    memset(state, 0, sizeof(*state));
    state->num_gaussians = N; state->tiles_x = va.tiles_x; state->tiles_y = va.tiles_y;
    Allocator A{alloc, alloc_user, s};
    const size_t npix = (size_t)va.W * va.H;
    const int ntiles = va.tiles_x * va.tiles_y;

    const size_t img_bytes = Carver::need((size_t)ntiles * 2, 4) + Carver::need(npix, 4) * 2;
    void* img = A.get(GS_B200_BUF_IMAGE, img_bytes, &state->owned[GS_B200_BUF_IMAGE]);
    if (A.failed) return 1;
    Carver ci(img);
    state->ranges = ci.take<uint32_t>((size_t)ntiles * 2);
    state->n_contrib = ci.take<uint32_t>(npix);
    state->final_T = ci.take<float>(npix);
    GS_CUDA_CHECK(cudaMemsetAsync(state->ranges, 0, (size_t)ntiles * 2 * 4, s));

    SplatRec* recs = (SplatRec*)A.get(GS_B200_BUF_GEOM, (size_t)N * sizeof(SplatRec), &state->owned[GS_B200_BUF_GEOM]);
    if (A.failed) return 1;
    state->geom = recs;
    BinA b;
    uint4* spans = nullptr;                        // tile culling: per-row tile spans (NULL = full squares)
    *host_total = 0;
    if (N > 0) {
        const bool own_spans = g_tile_culling.load() == 2;
        const size_t sc_bytes = Carver::need(N, 4) * 3 + Carver::need(1, 8) + bin_a_bytes(1, N) + (own_spans ? Carver::need(N, 16) : 0);
        void* sc = A.get(GS_B200_BUF_SCRATCH, sc_bytes);
        if (A.failed) return 1;
        Carver cv(sc);
        spans = own_spans ? cv.take<uint4>(N) : nullptr;
        b.tiles = cv.take<uint32_t>(N);
        b.dkeys = cv.take<uint32_t>(N);
        b.ids = cv.take<uint32_t>(N);
        uint32_t* min_key = (uint32_t*)cv.take<unsigned long long>(1);
        carve_bin_a(cv, b, 1, N);
        b.minkeys = min_key; b.dbg = dbg;
        GS_CUDA_CHECK(cudaMemsetAsync(min_key, 0xFF, 4, s));
        { StageTimer t(0, s);
        if (gs_launch_preprocess(va, N, M, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                                 recs, radii, b.tiles, b.dkeys, b.ids, min_key, spans, s)) return 1; }
        STAGE_CHECK(dbg, s, "preprocess");
        if (bin_a(b, host_total, s)) return 1;
    }
    GS_CUDA_CHECK(cudaStreamSynchronize(s));

    ViewSpans vs;
    if (view_spans(1, host_total, vs)) return 1;
    const int64_t P = vs.base[1];
    state->num_rendered = P;
    void* bin = A.get(GS_B200_BUF_BINNING, Carver::need(P, 4) * 2, &state->owned[GS_B200_BUF_BINNING]);
    if (A.failed) return 1;
    Carver cb(bin);
    BinB o;
    o.point_list = state->point_list = cb.take<uint32_t>(P);
    o.tile_keys = state->tile_keys = cb.take<uint32_t>(P);
    if (P > 0) {
        void* sc2 = A.get(GS_B200_BUF_SCRATCH, bin_b_scratch_bytes(1, P));
        if (A.failed) return 1;
        Carver c2(sc2);
        carve_bin_b_scratch(c2, o, 1, P);
        if (bin_b(b, vs, va.tiles_x, va.tiles_y, recs, spans, o, state->ranges, s)) return 1;
    }
    { StageTimer t(6, s);
    if (gs_launch_render_forward(va, recs, state->point_list, state->ranges, out_color, out_depth, out_alpha,
                                 state->n_contrib, state->final_T, s)) return 1; }
    STAGE_CHECK(dbg, s, "render");
    return 0;
}

int32_t gs_b200_rasterize_backward(const gs_b200_view* view, int32_t N, int32_t M, const float* means3D,
                                   const float* shs, const float* colors_precomp, const float* opacities,
                                   const float* scales, const float* rotations, const float* cov3D_precomp,
                                   const int32_t* radii, const gs_b200_state* state, const float* dL_dcolor,
                                   const float* dL_ddepth, const float* dL_dalpha, float* dL_dmeans3D,
                                   float* dL_dmeans2D, float* dL_dshs, float* dL_dcolors, float* dL_dopacities,
                                   float* dL_dscales, float* dL_drotations, float* dL_dcov3D, int32_t accumulate,
                                   gs_b200_alloc_fn alloc, void* alloc_user, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    ViewArgs va;
    if (make_view_args(__func__, view, va)) return 1;
    if (check_inputs(__func__, N, M, view->sh_degree, means3D, shs, colors_precomp, opacities, scales, rotations,
                     cov3D_precomp)) return 1;
    GS_REQ(state && dL_dcolor && dL_ddepth && dL_dalpha, "NULL state/upstream gradient");
    if (N == 0) return 0;
    GS_REQ(radii && dL_dmeans3D && dL_dmeans2D && dL_dopacities && (!shs || dL_dshs) && (!colors_precomp || dL_dcolors) &&
           (!scales || (dL_dscales && dL_drotations)) && (!cov3D_precomp || dL_dcov3D), "NULL gradient output");
    if (state->num_gaussians != N) { gs_set_error("%s: state is for N=%d, got %d", __func__, state->num_gaussians, N); return 1; }
    const int dbg = view->debug;
    Allocator A{alloc, alloc_user, s};
    SplatGrad* sg = (SplatGrad*)A.get(GS_B200_BUF_SCRATCH, (size_t)N * sizeof(SplatGrad));
    if (A.failed) return 1;
    GS_CUDA_CHECK(cudaMemsetAsync(sg, 0, (size_t)N * sizeof(SplatGrad), s));
    if (state->num_rendered > 0) {
        { StageTimer t(7, s);
        if (gs_launch_render_backward(va, (const SplatRec*)state->geom, state->point_list, state->ranges,
                                      state->n_contrib, state->final_T, dL_dcolor, dL_ddepth, dL_dalpha, sg, s)) return 1; }
        STAGE_CHECK(dbg, s, "render backward");
    }
    { StageTimer t(8, s);
    if (gs_launch_preprocess_backward(va, N, M, means3D, shs, colors_precomp, opacities, scales, rotations,
                                      cov3D_precomp, radii, sg, dL_dmeans3D, dL_dmeans2D, dL_dshs, dL_dcolors,
                                      dL_dopacities, dL_dscales, dL_drotations, dL_dcov3D, accumulate, s)) return 1; }
    STAGE_CHECK(dbg, s, "preprocess backward");
    return 0;
}

int32_t gs_b200_state_free(gs_b200_state* state, void* stream_) {
    if (!state) return 0;
    for (int i = 0; i < 4; i++)
        if (state->owned[i]) { cudaFreeAsync(state->owned[i], (cudaStream_t)stream_); state->owned[i] = nullptr; }
    return 0;
}

int32_t gs_b200_debug_sorted_keys(const gs_b200_state* state, uint64_t* keys_out, void* stream_) {
    GS_REQ(state && keys_out, "NULL argument");
    return gs_launch_sorted_keys((const SplatRec*)state->geom, state->point_list, state->tile_keys,
                                 state->num_rendered, keys_out, (cudaStream_t)stream_);
}

int32_t gs_b200_debug_preprocess_backward(const gs_b200_view* view, int32_t N, int32_t M, const float* means3D,
                                          const float* shs, const float* colors_precomp, const float* opacities,
                                          const float* scales, const float* rotations, const float* cov3D_precomp,
                                          const int32_t* radii, const double* splat_grads, float* dL_dmeans3D,
                                          float* dL_dmeans2D, float* dL_dshs, float* dL_dcolors, float* dL_dopacities,
                                          float* dL_dscales, float* dL_drotations, float* dL_dcov3D, int32_t accumulate,
                                          void* stream_) {
    ViewArgs va;
    if (make_view_args(__func__, view, va)) return 1;
    if (check_inputs(__func__, N, M, view->sh_degree, means3D, shs, colors_precomp, opacities, scales, rotations,
                     cov3D_precomp)) return 1;
    GS_REQ(N == 0 || (radii && splat_grads), "NULL radii/splat_grads");
    return gs_launch_preprocess_backward(va, N, M, means3D, shs, colors_precomp, opacities, scales, rotations,
                                         cov3D_precomp, radii, (const SplatGrad*)splat_grads, dL_dmeans3D, dL_dmeans2D,
                                         dL_dshs, dL_dcolors, dL_dopacities, dL_dscales, dL_drotations, dL_dcov3D,
                                         accumulate, (cudaStream_t)stream_);
}

int32_t gs_b200_step_view_chunks(int32_t V, int32_t* bounds) {
    if (V <= 0 || !bounds) { gs_set_error("%s: bad argument", __func__); return -1; }
    const StepChunks ch(V);
    for (int k = 0; k < ch.nchunks; k++) bounds[k] = ch.first(k);
    bounds[ch.nchunks] = V;
    return ch.nchunks;
}

// ---------------------------------------------------------------------------------
// Multi-view optimisation step (device-resident or host buffers).
//
// Views are handled in chunks.  An auxiliary stream projects and bins every view of a chunk in batched launches
// (one host wait for the chunk's pair counts); the views' composite kernels then run on TWO slot streams with
// per-slot grow-only workspaces (no allocation in steady state), so that one view's forward overlaps the other's
// backward.
// ---------------------------------------------------------------------------------
namespace {

struct Region { void* p = nullptr; size_t cap = 0; };
struct Slot {
    cudaStream_t stream = nullptr;
    Region image, loss_ws, nc;       // nc: n_contrib + final_T of the view on the slot
    cudaEvent_t evDone = nullptr;

    static int ensure(Region& r, size_t bytes, cudaStream_t st) {
        if (r.cap >= bytes) return 0;
        if (r.p) { cudaStreamSynchronize(st); cudaFree(r.p); r.p = nullptr; r.cap = 0; }
        const size_t want = bytes + bytes / 4 + 4096;
        if (cudaMalloc(&r.p, want) != cudaSuccess) { gs_set_error("cudaMalloc(%zu) failed", want); return 1; }
        r.cap = want;
        return 0;
    }
};

// The step's packed parameter and gradient buffers: six groups of N rows, means | shs | opacities | scales | rotations
// | means2D (gradients only), of 3, 3M, 1, 3, 4 and 3 floats a row.  Group g starts at off[g]; off[5] floats hold the
// parameters and off[6] the gradients.
struct PackedLayout { size_t off[7], width[6]; };
PackedLayout packed_layout(size_t N, size_t M) {
    const size_t width[6] = {3, 3 * M, 1, 3, 4, 3};
    PackedLayout L;
    L.off[0] = 0;
    for (int g = 0; g < 6; g++) { L.width[g] = width[g]; L.off[g + 1] = L.off[g] + N * width[g]; }
    return L;
}
struct PackedPtrs { float *means, *shs, *opac, *scales, *rots, *m2d; float* colors = nullptr; /* [N,3] instead of shs: forward-only */ };
PackedPtrs carve_packed(float* base, size_t N, size_t M, bool with_m2d) {
    const PackedLayout L = packed_layout(N, M);
    PackedPtrs p;
    p.means = base + L.off[0]; p.shs = base + L.off[1]; p.opac = base + L.off[2]; p.scales = base + L.off[3];
    p.rots = base + L.off[4]; p.m2d = with_m2d ? base + L.off[5] : nullptr;
    return p;
}
// the parameters as the entries take them: five arrays (and, for a forward-only caller, precomputed colours)
PackedPtrs param_ptrs(const float* means, const float* shs, const float* opac, const float* scales, const float* rots,
                      const float* colors = nullptr) {
    PackedPtrs p;
    p.means = (float*)means; p.shs = (float*)shs; p.opac = (float*)opac; p.scales = (float*)scales; p.rots = (float*)rots;
    p.m2d = nullptr; p.colors = (float*)colors;
    return p;
}

// Gradient sink: fn(user, first, count, stream) is called after each Gaussian range [first, first + count) of the
// step's LAST preprocess-backward has been enqueued on `stream`; that pass runs over nchunks such ranges.
struct GradSink { gs_b200_grad_sink fn = nullptr; void* user = nullptr; int nchunks = 1; };
thread_local GradSink g_grad_sink;       // gs_b200_set_grad_sink: a data-parallel caller's all-reduce

// What every view chunk of one multi-view step shares: the views (views_dev: [V][40] floats, in chunks ch), image and
// SH sizes, and the parameters.  geom_only: the preprocess leaves the records' colours to a pass after the binning,
// which first waits for shs_ready (if set): the host-buffer step's SH block is still being uploaded.
struct StepScene {
    StepChunks ch;
    const float* views_dev;
    int W, H, tiles_x, tiles_y, sh_degree;
    float scale_modifier;
    int N, M;
    PackedPtrs par;
    bool geom_only;
    cudaEvent_t shs_ready;
    StepScene(int V, int H_, int W_, int sh_degree_, float scale_modifier_, const float* views_dev_, int N_, int M_,
              const PackedPtrs& par_, bool geom_only_ = false, cudaEvent_t shs_ready_ = nullptr)
        : ch(V), views_dev(views_dev_), W(W_), H(H_), tiles_x((W_ + GS_TILE - 1) / GS_TILE),
          tiles_y((H_ + GS_TILE - 1) / GS_TILE), sh_degree(sh_degree_), scale_modifier(scale_modifier_), N(N_), M(M_),
          par(par_), geom_only(geom_only_), shs_ready(shs_ready_) {}
    const float* views(int k) const { return views_dev + (size_t)ch.first(k) * 40; }
};

size_t chunk_pairs_bytes(int nv, int64_t P) { return Carver::need(P, 4) * 2 + bin_b_scratch_bytes(nv, P); }

// Workspace of one view chunk of the multi-view step, in six grow-only regions that are freed with it: [VB][N]
// preprocess outputs and depth sort, the binning scratch and [VB][tiles][2] ranges, and the chunk's pair lists.
struct ChunkWS {
    Region r_recs, r_sg, r_u32, r_spans, r_bin, r_pairs;
    SplatRec* recs; SplatGrad* sg; int32_t* radii; uint32_t *minkeys, *ranges; uint4* spans; BinA bin;
    ViewSpans vs; BinB pairs;           // the chunk's per-view pair bases and pair lists (chunk_bin)

    ChunkWS() = default;
    ChunkWS(const ChunkWS&) = delete;
    ChunkWS& operator=(const ChunkWS&) = delete;
    ~ChunkWS() {
        for (Region* r : {&r_recs, &r_sg, &r_u32, &r_spans, &r_bin, &r_pairs}) if (r->p) cudaFree(r->p);
    }
    // sized for the scene's largest chunk; tight: with the tile culling's spans
    int setup(const StepScene& sc, bool tight, cudaStream_t s) {
        const int VB = sc.ch.VB, ntiles = sc.tiles_x * sc.tiles_y;
        const size_t nvb = (size_t)VB * sc.N;
        if (Slot::ensure(r_recs, nvb * sizeof(SplatRec), s) || Slot::ensure(r_sg, nvb * sizeof(SplatGrad), s) ||
            Slot::ensure(r_u32, nvb * 4 * 4 + 256 * 4, s) ||
            Slot::ensure(r_bin, bin_a_bytes(VB, sc.N) + Carver::need((size_t)VB * ntiles * 2, 4), s)) return 1;
        if (tight && Slot::ensure(r_spans, nvb * sizeof(uint4), s)) return 1;
        uint32_t* u32 = (uint32_t*)r_u32.p;
        recs = (SplatRec*)r_recs.p; sg = (SplatGrad*)r_sg.p; radii = (int32_t*)u32;
        minkeys = u32 + 4 * nvb;        // [VB] stride 2 words
        spans = tight ? (uint4*)r_spans.p : nullptr;
        bin.tiles = u32 + nvb; bin.dkeys = u32 + 2 * nvb; bin.ids = u32 + 3 * nvb;
        bin.minkeys = minkeys; bin.minkey_stride = 2;
        Carver cb(r_bin.p);
        ranges = cb.take<uint32_t>((size_t)VB * ntiles * 2);
        carve_bin_a(cb, bin, VB, sc.N);
        return 0;
    }
};

// ---- the three per-chunk stages of the multi-view step.  step_core runs them on its aux stream; the test entries run
// them on one stream.
// Projection of chunk k: preprocess, depth sort, scan, and the D2H of the views' pair counts to host_totals.
int chunk_project(ChunkWS& w, const StepScene& sc, int k, unsigned long long* host_totals, cudaStream_t s) {
    const PackedPtrs& p = sc.par;
    const int nv = sc.ch.count(k);
    GS_CUDA_CHECK(cudaMemsetAsync(w.minkeys, 0xFF, 256 * 4, s));
    { StageTimer t(0, s);
    if (gs_launch_preprocess_multi(sc.views(k), nv, sc.W, sc.H, sc.sh_degree, sc.scale_modifier, sc.N, sc.M, p.means,
                                   p.shs, p.colors, p.opac, p.scales, p.rots, w.recs, w.radii, w.bin.tiles, w.bin.dkeys,
                                   w.bin.ids, w.minkeys, w.spans, s, sc.geom_only ? 1 : 0)) return 1; }
    w.bin.nv = nv;
    return bin_a(w.bin, host_totals, s);
}
// Binning of chunk k, once host_totals holds its pair counts: the per-view pair bases (view_spans), the pair lists in
// the grow-only pairs region (fill_pairs: pre-filled with 0xFF bytes, so a slot the emit leaves unwritten reads
// 0xFFFFFFFF after the sort), ranges, emit, tile sort; then, for a geom_only scene, the records' colours.
int chunk_bin(ChunkWS& w, const StepScene& sc, int k, const unsigned long long* host_totals, bool fill_pairs,
              cudaStream_t s) {
    const int nv = sc.ch.count(k);
    if (view_spans(nv, host_totals, w.vs)) return 1;
    const int64_t P = w.vs.base[nv];
    const size_t bytes = chunk_pairs_bytes(nv, P);
    if (Slot::ensure(w.r_pairs, bytes, s)) return 1;
    if (fill_pairs) GS_CUDA_CHECK(cudaMemsetAsync(w.r_pairs.p, 0xFF, bytes, s));
    Carver cp(w.r_pairs.p);
    w.pairs.point_list = cp.take<uint32_t>(P); w.pairs.tile_keys = cp.take<uint32_t>(P);
    carve_bin_b_scratch(cp, w.pairs, nv, P);
    GS_CUDA_CHECK(cudaMemsetAsync(w.ranges, 0, (size_t)nv * sc.tiles_x * sc.tiles_y * 2 * 4, s));
    if (bin_b(w.bin, w.vs, sc.tiles_x, sc.tiles_y, w.recs, w.spans, w.pairs, w.ranges, s)) return 1;
    if (sc.geom_only) {
        if (sc.shs_ready) GS_CUDA_CHECK(cudaStreamWaitEvent(s, sc.shs_ready, 0));
        const PackedPtrs& p = sc.par;
        if (gs_launch_sh_colour_multi(sc.views(k), nv, sc.sh_degree, sc.N, sc.M, p.means, p.shs, w.radii, w.recs, s)) return 1;
    }
    return 0;
}
// Preprocess backward of chunk k from its views' [count(k)][N] radii and SplatGrad: the first chunk writes the
// gradients grd, later ones add to them.  Run over `nparts` Gaussian ranges whose starts are multiples of the kernel's
// 128-Gaussian CTA; the sink (optional) follows each range's launch.
int chunk_backward(const StepScene& sc, int k, const int32_t* radii, const SplatGrad* sg, const PackedPtrs& grd,
                   int nparts, const GradSink* sink, cudaStream_t s) {
    const PackedPtrs& p = sc.par;
    const int N = sc.N;
    const int per = (((N + nparts - 1) / nparts) + 127) / 128 * 128;
    for (int first = 0; first < N; first += per) {
        const int count = std::min(per, N - first);
        { StageTimer t(8, s);
        if (gs_launch_preprocess_backward_multi(sc.views(k), sc.ch.count(k), sc.W, sc.H, sc.sh_degree, sc.scale_modifier,
                                                N, sc.M, p.means, p.shs, p.scales, p.rots, radii, sg, grd.means, grd.m2d,
                                                grd.shs, grd.opac, grd.scales, grd.rots, k > 0 ? 1 : 0, first, count,
                                                s)) return 1; }
        if (sink) sink->fn(sink->user, first, count, (void*)s);
    }
    return 0;
}

constexpr int NSLOTS = 2;       // the composites of a chunk's views alternate between two slot streams
struct StepCache {
    Slot slot[NSLOTS];
    bool init = false;
    cudaStream_t copy_stream = nullptr, d2h_stream = nullptr, aux_stream = nullptr;
    cudaEvent_t evFork = nullptr, evPB = nullptr, evGeom = nullptr, evD2H = nullptr, evAux = nullptr;
    cudaEvent_t evBinA[2] = {nullptr, nullptr}, evBin[2] = {nullptr, nullptr};
    unsigned long long* host_totals[2] = {nullptr, nullptr};     // pinned: per-view pair counts of a chunk
    std::vector<cudaEvent_t> up_ready;          // per view: upstream gradient resident
    Region host_stage;                           // device copies of host inputs (step_host)
    bool busy = false;                           // a view hook must not re-enter the step entries on this thread
    ChunkWS ws[2];                               // two chunk workspaces that alternate between chunks
    int ensure_init() {
        if (init) return 0;
        for (int i = 0; i < NSLOTS; i++) {
            GS_CUDA_CHECK(cudaStreamCreateWithFlags(&slot[i].stream, cudaStreamNonBlocking));
            GS_CUDA_CHECK(cudaEventCreateWithFlags(&slot[i].evDone, cudaEventDisableTiming));
        }
        GS_CUDA_CHECK(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking));
        GS_CUDA_CHECK(cudaStreamCreateWithFlags(&d2h_stream, cudaStreamNonBlocking));
        GS_CUDA_CHECK(cudaStreamCreateWithFlags(&aux_stream, cudaStreamNonBlocking));
        GS_CUDA_CHECK(cudaEventCreateWithFlags(&evAux, cudaEventDisableTiming));
        for (int i = 0; i < 2; i++) {
            GS_CUDA_CHECK(cudaEventCreateWithFlags(&evBinA[i], cudaEventDisableTiming));
            GS_CUDA_CHECK(cudaEventCreateWithFlags(&evBin[i], cudaEventDisableTiming));
            GS_CUDA_CHECK(cudaHostAlloc((void**)&host_totals[i], GS_MAX_SEGS * sizeof(unsigned long long), cudaHostAllocDefault));
        }
        GS_CUDA_CHECK(cudaEventCreateWithFlags(&evD2H, cudaEventDisableTiming));
        GS_CUDA_CHECK(cudaEventCreateWithFlags(&evFork, cudaEventDisableTiming));
        GS_CUDA_CHECK(cudaEventCreateWithFlags(&evPB, cudaEventDisableTiming));
        GS_CUDA_CHECK(cudaEventCreateWithFlags(&evGeom, cudaEventDisableTiming));
        init = true;
        return 0;
    }
};
// one pipeline state per (thread, device): streams, events and workspaces belong to the device that was current when
// they were created, so a thread that drives a second GPU gets a second set instead of launching onto the first one's
StepCache& step_cache() {
    thread_local std::unique_ptr<StepCache> caches[64];
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (!caches[dev]) caches[dev].reset(new StepCache());
    return *caches[dev];
}

// Device-resident core.  views_host gives tanfov per view (host side), views_dev the matrices.
// Views are handled in chunks of <= VB.  Per chunk, on the aux stream: ONE multi-view preprocess pass over the
// Gaussians (parameters read once), then the batched binning of all its views (segmented depth sort, gather-scan,
// one host wait for the pair counts, emit, segmented tile sort, ranges).  Then per view, on the slot streams:
// composite forward -> view hook -> SplatGrad zeroing -> composite backward.  Then ONE multi-view
// preprocess-backward pass (parameters read once, gradients written once).
// view hook (optional): called on the host after view v's forward has been enqueued on its slot stream and before
// its backward is; the callee enqueues, on that stream, whatever turns images[v] into dL_dout[v] (the loss).
// forward_only: no backward at all (render entry).  radii_out (optional): [V][N] per-view radii.
// shs_ready (optional, host-buffer step): the SH block is still being uploaded when the step starts -- `user` is ordered
// after the geometry parameters only.  Projection and binning of each chunk run first (colour-free), the colours are
// filled in when the event fires (sh_colour_multi on the aux stream), then the composites follow.
// sink (optional): follows the ranges of the final preprocess-backward (the host-buffer step starts the D2H of each
// range there while the next one computes); without one, the sink set by gs_b200_set_grad_sink, if any.
struct StepOpts { gs_b200_view_hook hook = nullptr; void* hook_user = nullptr; bool forward_only = false; int32_t* radii_out = nullptr;
                  cudaEvent_t shs_ready = nullptr; GradSink sink; };

int step_core(int V, int H, int W, int sh_degree, float scale_modifier, const float* views_host,
              const float* views_dev, int N, int M, const PackedPtrs& par, const float* dL_dout_dev,
              const cudaEvent_t* up_ready, const PackedPtrs& grd, float* images_dev, int64_t* num_rendered_out,
              cudaStream_t user, const StepOpts& O = StepOpts()) {
    StepCache& C = step_cache();
    if (C.busy) { gs_set_error("step: re-entrant call from a view hook (the per-thread pipeline state is in use)"); return 1; }
    struct BusyGuard { bool& b; explicit BusyGuard(bool& x) : b(x) { b = true; } ~BusyGuard() { b = false; } } busy_guard(C.busy);
    if (C.ensure_init()) return 1;
    const GradSink& sink = O.sink.fn ? O.sink : g_grad_sink;
    const size_t npix = (size_t)H * W;
    // View chunks: one batched preprocess + binning / preprocess-backward per chunk of <= 16 views, on the aux stream:
    //   aux stream:   pre+bin(0) | pre+bin(1) ......... bwd(0) | pre+bin(2) ...... bwd(1) | ... | bwd(last)
    //   slot streams:             views of chunk 0 ............. views of chunk 1 .......
    // pre+bin(k+1) is enqueued when chunk k's views start (its second half, after the host has read the pair counts,
    // once they have all been enqueued), bwd(k) after that; two workspace sets alternate and the aux stream's own
    // order (bwd(k-1) before pre(k+1)) protects their reuse.
    const bool late = O.shs_ready && par.shs && !par.colors;
    const StepScene sc(V, H, W, sh_degree, scale_modifier, views_dev, N, M, par, late, late ? O.shs_ready : nullptr);
    const int nchunks = sc.ch.nchunks, ntiles = sc.tiles_x * sc.tiles_y;
    const bool tight = g_tile_culling.load() >= 1;
    if (O.shs_ready && !late) GS_CUDA_CHECK(cudaStreamWaitEvent(user, O.shs_ready, 0));
    const int nsets = nchunks > 1 ? 2 : 1;
    for (int i = 0; i < nsets; i++)
        if (C.ws[i].setup(sc, tight, user)) return 1;
    cudaStream_t aux = C.aux_stream;
    // everything is ordered after the caller's stream
    GS_CUDA_CHECK(cudaEventRecord(C.evFork, user));
    GS_CUDA_CHECK(cudaStreamWaitEvent(aux, C.evFork, 0));

    int64_t rendered = 0;
    auto enqueue_pre = [&](int k) -> int {
        if (chunk_project(C.ws[k & (nsets - 1)], sc, k, C.host_totals[k & 1], aux)) return 1;
        GS_CUDA_CHECK(cudaEventRecord(C.evBinA[k & 1], aux));
        return 0;
    };
    auto enqueue_bin = [&](int k) -> int {
        ChunkWS& w = C.ws[k & (nsets - 1)];
        GS_CUDA_CHECK(cudaEventSynchronize(C.evBinA[k & 1]));
        // grow-only: the pair lists of all the chunk's views live until its last composite backward
        if (chunk_bin(w, sc, k, C.host_totals[k & 1], false, aux)) return 1;
        rendered += w.vs.base[w.vs.n];
        GS_CUDA_CHECK(cudaEventRecord(C.evBin[k & 1], aux));
        return 0;
    };

    int rc = enqueue_pre(0);
    if (!rc) rc = enqueue_bin(0);
    for (int k = 0; k < nchunks && !rc; k++) {
        const int v0 = sc.ch.first(k), nv = sc.ch.count(k);
        const ChunkWS& w = C.ws[k & (nsets - 1)];
        // the slot streams continue after this chunk's binning ...
        for (int i = 0; i < NSLOTS; i++) GS_CUDA_CHECK(cudaStreamWaitEvent(C.slot[i].stream, C.evBin[k & 1], 0));
        // ... while the next chunk's preprocess and depth sort already run beside them
        if (k + 1 < nchunks && (rc = enqueue_pre(k + 1))) break;

        for (int j = 0; j < nv && !rc; j++) {
            Slot& S = C.slot[j & 1];
            const int v = v0 + j;
            if (!images_dev && Slot::ensure(S.image, 5 * npix * 4, S.stream)) { rc = 1; break; }
            if (Slot::ensure(S.nc, Carver::need(npix, 4) * 2, S.stream)) { rc = 1; break; }
            const float* vh = views_host + (size_t)v * 40;
            const float* vd = views_dev + (size_t)v * 40;
            gs_b200_view vw;
            vw.image_height = H; vw.image_width = W; vw.tanfovx = vh[38]; vw.tanfovy = vh[39];
            vw.bg = vd + 35; vw.scale_modifier = scale_modifier; vw.viewmatrix = vd; vw.projmatrix = vd + 16;
            vw.sh_degree = sh_degree; vw.campos = vd + 32; vw.prefiltered = 0; vw.debug = 0;
            ViewArgs va;
            if ((rc = make_view_args("step", &vw, va))) break;
            float* img = images_dev ? images_dev + (size_t)v * 5 * npix : (float*)S.image.p;
            Carver cn(S.nc.p);
            uint32_t* n_contrib = cn.take<uint32_t>(npix);
            float* final_T = cn.take<float>(npix);
            const size_t off = (size_t)j * N;
            const SplatRec* recs = w.recs + off;
            const uint32_t* point_list = w.pairs.point_list + w.vs.base[j];
            const uint32_t* ranges = w.ranges + (size_t)j * ntiles * 2;
            { StageTimer t(6, S.stream);
            if ((rc = gs_launch_render_forward(va, recs, point_list, ranges, img, img + 3 * npix, img + 4 * npix,
                                               n_contrib, final_T, S.stream))) break; }
            if (O.forward_only) continue;
            if (O.hook && O.hook(O.hook_user, v, (void*)S.stream) != 0) { gs_set_error("step: view hook failed at view %d", v); rc = 1; break; }
            const float* up = dL_dout_dev + (size_t)v * 5 * npix;
            if (up_ready) GS_CUDA_CHECK(cudaStreamWaitEvent(S.stream, up_ready[v], 0));
            // The view's SplatGrad slice is zeroed here, on its slot stream, so the write overlaps the other slot's
            // composites.  Also for a view without pairs, whose composite backward is skipped: the batched
            // preprocess-backward reads the slice for every Gaussian with radii > 0.
            GS_CUDA_CHECK(cudaMemsetAsync(w.sg + off, 0, (size_t)N * sizeof(SplatGrad), S.stream));
            if (w.vs.base[j + 1] > w.vs.base[j]) {
                StageTimer t(7, S.stream);
                if ((rc = gs_launch_render_backward(va, recs, point_list, ranges, n_contrib, final_T, up, up + 3 * npix,
                                                    up + 4 * npix, w.sg + off, S.stream))) break;
            }
        }
        // the next chunk's binning, now that this chunk's views are queued behind it
        if (!rc && k + 1 < nchunks) rc = enqueue_bin(k + 1);
        // the aux stream picks up after this chunk's views (batched backward, radii copy, workspace hand-over)
        for (int i = 0; i < NSLOTS; i++) {
            cudaEventRecord(C.slot[i].evDone, C.slot[i].stream);
            cudaStreamWaitEvent(aux, C.slot[i].evDone, 0);
        }
        if (rc) break;
        if (O.radii_out) GS_CUDA_CHECK(cudaMemcpyAsync(O.radii_out + (size_t)v0 * N, w.radii, (size_t)nv * N * 4, cudaMemcpyDeviceToDevice, aux));
        if (O.forward_only) continue;
        const GradSink* last = k + 1 == nchunks && sink.fn ? &sink : nullptr;       // the sink follows the last pass
        rc = chunk_backward(sc, k, w.radii, w.sg, grd, last ? last->nchunks : 1, last, aux);
    }
    // join: the caller's stream continues after the aux stream (which has waited for both slot streams)
    for (int i = 0; i < NSLOTS; i++) {          // (on an error path the slots may not have been joined into aux yet)
        cudaEventRecord(C.slot[i].evDone, C.slot[i].stream);
        cudaStreamWaitEvent(aux, C.slot[i].evDone, 0);
    }
    cudaEventRecord(C.evAux, aux);
    cudaStreamWaitEvent(user, C.evAux, 0);
    if (num_rendered_out) *num_rendered_out = rendered;
    return rc;
}

// fn: the entry point named in the error message
int step_host_impl(const char* fn, int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                   const float* views_host, int32_t N, int32_t M, const float* means3D_host,
                   const float* shs_host, const float* opacities_host, const float* scales_host,
                   const float* rotations_host, const float* dL_dout_host, float* grads_host, float* grads_dev,
                   float* images_host, int64_t* num_rendered_out, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    if (V <= 0 || N <= 0 || !views_host || !means3D_host || !shs_host || !opacities_host || !scales_host ||
        !rotations_host || !dL_dout_host || (!grads_host && !grads_dev)) { gs_set_error("%s: bad argument", fn); return 1; }
    StepCache& C = step_cache();
    if (C.ensure_init()) return 1;
    const size_t npix = (size_t)H * W;
    const PackedLayout L = packed_layout(N, M);
    const size_t n_par = L.off[5], n_grad = L.off[6];
    const size_t need = Carver::need(n_par, 4) + Carver::need(n_grad, 4) + Carver::need((size_t)V * 40, 4) +
                        Carver::need((size_t)V * 5 * npix, 4) * (images_host ? 2 : 1);
    if (Slot::ensure(C.host_stage, need, s)) return 1;
    Carver c(C.host_stage.p);
    float* d_par = c.take<float>(n_par);
    float* d_grad = c.take<float>(n_grad);
    float* d_views = c.take<float>((size_t)V * 40);
    float* d_up = c.take<float>((size_t)V * 5 * npix);
    float* d_img = images_host ? c.take<float>((size_t)V * 5 * npix) : nullptr;
    const PackedPtrs par = carve_packed(d_par, N, M, false), grd = carve_packed(d_grad, N, M, true);
    while ((int)C.up_ready.size() < V) {
        cudaEvent_t e; GS_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); C.up_ready.push_back(e);
    }
    // H2D order on the copy stream: geometry parameters FIRST (projection, sorting and binning need nothing else), then
    // the SH block (192 of the 236 B per Gaussian at degree 3; only the colours and the backward need it -- step_core
    // bins every view while it is on its way, StepOpts::shs_ready), then the upstream gradients view by view (needed only
    // at each view's backward), so they stream in behind the compute.
    GS_CUDA_CHECK(cudaEventRecord(C.evFork, s));
    GS_CUDA_CHECK(cudaStreamWaitEvent(C.copy_stream, C.evFork, 0));
    GS_CUDA_CHECK(cudaMemcpyAsync(d_views, views_host, (size_t)V * 160, cudaMemcpyHostToDevice, C.copy_stream));
    GS_CUDA_CHECK(cudaMemcpyAsync(par.means, means3D_host, (size_t)N * 12, cudaMemcpyHostToDevice, C.copy_stream));
    GS_CUDA_CHECK(cudaMemcpyAsync(par.opac, opacities_host, (size_t)N * 4, cudaMemcpyHostToDevice, C.copy_stream));
    GS_CUDA_CHECK(cudaMemcpyAsync(par.scales, scales_host, (size_t)N * 12, cudaMemcpyHostToDevice, C.copy_stream));
    GS_CUDA_CHECK(cudaMemcpyAsync(par.rots, rotations_host, (size_t)N * 16, cudaMemcpyHostToDevice, C.copy_stream));
    GS_CUDA_CHECK(cudaEventRecord(C.evGeom, C.copy_stream));
    GS_CUDA_CHECK(cudaMemcpyAsync(par.shs, shs_host, (size_t)N * 12 * M, cudaMemcpyHostToDevice, C.copy_stream));
    GS_CUDA_CHECK(cudaEventRecord(C.evPB, C.copy_stream));
    for (int v = 0; v < V; v++) {
        GS_CUDA_CHECK(cudaMemcpyAsync(d_up + (size_t)v * 5 * npix, dL_dout_host + (size_t)v * 5 * npix, 5 * npix * 4,
                                      cudaMemcpyHostToDevice, C.copy_stream));
        GS_CUDA_CHECK(cudaEventRecord(C.up_ready[v], C.copy_stream));
    }
    GS_CUDA_CHECK(cudaStreamWaitEvent(s, C.evGeom, 0));
    StepOpts opts;
    opts.shs_ready = C.evPB;
    // D2H of the summed gradients is chunked over Gaussian ranges and starts as soon as a range is final.  The sink is
    // set with device gradients too (it then copies nothing), so a sink from gs_b200_set_grad_sink never applies here.
    struct SinkCtx { StepCache* C; float* host; float* dev; PackedLayout L; } sctx{&C, grads_host, d_grad, L};
    opts.sink.user = &sctx;
    opts.sink.nchunks = grads_host ? 4 : 1;
    opts.sink.fn = [](void* vp, int32_t first, int32_t count, void* st) {
        SinkCtx* q = (SinkCtx*)vp;
        if (!q->host) return;
        StepCache& C2 = *q->C;
        cudaEventRecord(C2.evD2H, (cudaStream_t)st);
        cudaStreamWaitEvent(C2.d2h_stream, C2.evD2H, 0);
        for (int g = 0; g < 6; g++) {
            const size_t off = q->L.off[g] + (size_t)first * q->L.width[g];
            cudaMemcpyAsync(q->host + off, q->dev + off, (size_t)count * q->L.width[g] * 4, cudaMemcpyDeviceToHost, C2.d2h_stream);
        }
    };
    // no memset of the gradient buffer: the first view chunk's preprocess-backward writes every element (accumulate = 0)
    if (step_core(V, H, W, sh_degree, scale_modifier, views_host, d_views, N, M, par, d_up, C.up_ready.data(), grd,
                  d_img, num_rendered_out, s, opts)) return 1;
    if (grads_dev) GS_CUDA_CHECK(cudaMemcpyAsync(grads_dev, d_grad, n_grad * 4, cudaMemcpyDeviceToDevice, s));
    if (images_host) GS_CUDA_CHECK(cudaMemcpyAsync(images_host, d_img, (size_t)V * 5 * npix * 4, cudaMemcpyDeviceToHost, s));
    if (grads_host) GS_CUDA_CHECK(cudaStreamSynchronize(C.d2h_stream));
    if (grads_host || images_host) GS_CUDA_CHECK(cudaStreamSynchronize(s));
    return 0;
}
}  // namespace

int32_t gs_b200_set_grad_sink(gs_b200_grad_sink sink, void* user, int32_t nchunks) {
    GS_REQ(!sink || (nchunks >= 1 && nchunks <= 64), "nchunks must be 1..64");
    g_grad_sink.fn = sink; g_grad_sink.user = user; g_grad_sink.nchunks = sink ? nchunks : 1;
    return 0;
}

int32_t gs_b200_step_device(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                            const float* views_host, const float* views_dev, int32_t N, int32_t M,
                            const float* means3D, const float* shs, const float* opacities, const float* scales,
                            const float* rotations, const float* dL_dout, float* grads, float* images,
                            int64_t* num_rendered_out, void* stream_) {
    GS_REQ(V > 0 && N > 0 && views_host && views_dev && means3D && shs && opacities && scales && rotations && dL_dout &&
           grads, "bad argument");
    // grads need no memset: the first chunk's preprocess-backward writes every element
    return step_core(V, H, W, sh_degree, scale_modifier, views_host, views_dev, N, M,
                     param_ptrs(means3D, shs, opacities, scales, rotations), dL_dout, nullptr,
                     carve_packed(grads, N, M, true), images, num_rendered_out, (cudaStream_t)stream_);
}

int32_t gs_b200_step_device_hook(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                                 const float* views_host, const float* views_dev, int32_t N, int32_t M,
                                 const float* means3D, const float* shs, const float* opacities, const float* scales,
                                 const float* rotations, float* dL_dout, float* grads, float* images, int32_t* radii,
                                 gs_b200_view_hook hook, void* hook_user, int64_t* num_rendered_out, void* stream_) {
    GS_REQ(V > 0 && N > 0 && views_host && views_dev && means3D && shs && opacities && scales && rotations && dL_dout &&
           grads && images && hook, "bad argument");
    StepOpts o; o.hook = hook; o.hook_user = hook_user; o.radii_out = radii;
    return step_core(V, H, W, sh_degree, scale_modifier, views_host, views_dev, N, M,
                     param_ptrs(means3D, shs, opacities, scales, rotations), dL_dout, nullptr,
                     carve_packed(grads, N, M, true), images, num_rendered_out, (cudaStream_t)stream_, o);
}

namespace {
struct TrainLossCtx {
    int H, W; const float *ref, *mask; float ls, la, scale; float *dL, *images, *losses;
};
int32_t train_loss_hook(void* user, int32_t v, void* stream_) {
    TrainLossCtx* q = (TrainLossCtx*)user;
    cudaStream_t s = (cudaStream_t)stream_;
    StepCache& C = step_cache();
    Slot* S = &C.slot[0];
    for (int i = 1; i < NSLOTS; i++) if (s == C.slot[i].stream) S = &C.slot[i];
    if (Slot::ensure(S->loss_ws, gs_image_loss_scratch_bytes(q->H, q->W), s)) return 1;
    const size_t npix = (size_t)q->H * q->W;
    return gs_launch_image_loss(q->H, q->W, q->images + (size_t)v * 5 * npix, q->ref + (size_t)v * 3 * npix,
                                q->mask + (size_t)v * npix, q->ls, q->la, q->scale, q->dL + (size_t)v * 5 * npix,
                                q->losses + v, S->loss_ws.p, s);
}
thread_local Region g_loss_ws;
}  // namespace

int32_t gs_b200_image_loss(int32_t H, int32_t W, const float* image, const float* ref_image, const float* ref_mask,
                           float lambda_ssim, float lambda_alpha, float scale, float* dL_dimage, float* loss_out,
                           void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    GS_REQ(image && ref_image && ref_mask && dL_dimage && loss_out, "NULL argument");
    if (Slot::ensure(g_loss_ws, gs_image_loss_scratch_bytes(H, W), s)) return 1;
    return gs_launch_image_loss(H, W, image, ref_image, ref_mask, lambda_ssim, lambda_alpha, scale, dL_dimage, loss_out,
                                g_loss_ws.p, s);
}

int32_t gs_b200_step_device_train(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                                  const float* views_host, const float* views_dev, int32_t N, int32_t M,
                                  const float* means3D, const float* shs, const float* opacities, const float* scales,
                                  const float* rotations, const float* ref_images, const float* ref_masks,
                                  float lambda_ssim, float lambda_alpha, float loss_scale, float* dL_dout, float* grads,
                                  float* images, int32_t* radii, float* losses, int64_t* num_rendered_out, void* stream_) {
    GS_REQ(V > 0 && N > 0 && views_host && views_dev && means3D && shs && opacities && scales && rotations &&
           ref_images && ref_masks && dL_dout && grads && images && losses, "bad argument");
    GS_REQ(!(lambda_ssim > 0.f) || (H > 160 && W > 160), "MS-SSIM needs image sides > 160");
    TrainLossCtx ctx{H, W, ref_images, ref_masks, lambda_ssim, lambda_alpha, loss_scale, dL_dout, images, losses};
    StepOpts o; o.hook = train_loss_hook; o.hook_user = &ctx; o.radii_out = radii;
    return step_core(V, H, W, sh_degree, scale_modifier, views_host, views_dev, N, M,
                     param_ptrs(means3D, shs, opacities, scales, rotations), dL_dout, nullptr,
                     carve_packed(grads, N, M, true), images, num_rendered_out, (cudaStream_t)stream_, o);
}

int32_t gs_b200_render_views(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                             const float* views_host, const float* views_dev, int32_t N, int32_t M,
                             const float* means3D, const float* shs, const float* colors_precomp, const float* opacities,
                             const float* scales, const float* rotations, float* images, int32_t* radii,
                             int64_t* num_rendered_out, void* stream_) {
    GS_REQ(V > 0 && N > 0 && views_host && views_dev && means3D && opacities && scales && rotations && images,
           "bad argument");
    if ((shs == nullptr) == (colors_precomp == nullptr)) { gs_set_error("Please provide excatly one of either SHs or precomputed colors!"); return 1; }
    StepOpts o; o.forward_only = true; o.radii_out = radii;
    return step_core(V, H, W, sh_degree, scale_modifier, views_host, views_dev, N, M,
                     param_ptrs(means3D, shs, opacities, scales, rotations, colors_precomp), nullptr, nullptr,
                     PackedPtrs{}, images, num_rendered_out, (cudaStream_t)stream_, o);
}

// ---- test entries of the binning stage and of the multi-view step's chunk stages ----------------------------------

int32_t gs_b200_debug_sort_segmented(uint32_t* keys, uint32_t* keys_alt, uint32_t* vals, uint32_t* vals_alt,
                                     const int64_t* seg_off, int32_t nseg, int32_t begin_bit, int32_t end_bit,
                                     const uint32_t* key_bias, int32_t bias_stride, int32_t* result_in_alt, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    GS_REQ(seg_off && nseg >= 1 && nseg <= GS_MAX_SEGS && result_in_alt, "bad argument");
    SortSegs sg; sg.n = nseg;
    for (int i = 0; i <= nseg; i++) sg.off[i] = seg_off[i];
    void* scratch = nullptr;
    const size_t bytes = gs_sort_seg_scratch_bytes(nseg, std::max<int64_t>(seg_off[nseg], 0));
    GS_CUDA_CHECK(cudaMallocAsync(&scratch, bytes, s));
    int r = 0;
    const int rc = gs_sort_pairs_segmented(keys, keys_alt, vals, vals_alt, sg, begin_bit, end_bit, scratch, &r, key_bias,
                                           bias_stride, false, s);
    cudaFreeAsync(scratch, s);
    *result_in_alt = r;
    return rc;
}

// The multi-view step's projection and binning, as step_core runs them (chunk_project, chunk_bin), on `stream` alone,
// with the pair buffers pre-filled with 0xFF bytes and every intermediate list copied out.  Without point_list (the
// first call of two) only the [V][N] arrays and the totals, from which the caller sizes the pair lists.
int32_t gs_b200_debug_bin_views(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                                const float* views_dev, int32_t N, int32_t M, const float* means3D, const float* shs,
                                const float* opacities, const float* scales, const float* rotations, int32_t tight,
                                int32_t* radii, uint32_t* tiles_touched, uint32_t* spans, uint32_t* sorted_dkeys,
                                uint32_t* sorted_ids, uint32_t* offsets, int64_t* totals, uint32_t* ranges,
                                uint32_t* point_list, uint32_t* tile_keys, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    GS_REQ(V > 0 && N > 0 && M >= (sh_degree + 1) * (sh_degree + 1) && M <= 16 && views_dev && means3D && shs &&
           opacities && scales && rotations && radii && tiles_touched && (!tight || spans) && sorted_dkeys &&
           sorted_ids && offsets && totals && (!point_list || (tile_keys && ranges)), "bad argument");
    const StepScene sc(V, H, W, sh_degree, scale_modifier, views_dev, N, M,
                       param_ptrs(means3D, shs, opacities, scales, rotations));
    const int ntiles = sc.tiles_x * sc.tiles_y;
    ChunkWS w;
    if (w.setup(sc, tight != 0, s)) return 1;
    unsigned long long host_totals[GS_MAX_SEGS];
    int64_t pair0 = 0;        // the chunk's first pair in point_list / tile_keys
    for (int k = 0; k < sc.ch.nchunks; k++) {
        const int v0 = sc.ch.first(k), nv = sc.ch.count(k);
        const size_t o = (size_t)v0 * N, n = (size_t)nv * N;
        if (chunk_project(w, sc, k, host_totals, s)) return 1;
        GS_CUDA_CHECK(cudaMemcpyAsync(radii + o, w.radii, n * 4, cudaMemcpyDeviceToDevice, s));
        GS_CUDA_CHECK(cudaMemcpyAsync(tiles_touched + o, w.bin.tiles, n * 4, cudaMemcpyDeviceToDevice, s));
        if (tight) GS_CUDA_CHECK(cudaMemcpyAsync(spans + 4 * o, w.spans, n * 16, cudaMemcpyDeviceToDevice, s));
        GS_CUDA_CHECK(cudaMemcpyAsync(sorted_dkeys + o, w.bin.sorted_dkeys, n * 4, cudaMemcpyDeviceToDevice, s));
        GS_CUDA_CHECK(cudaMemcpyAsync(sorted_ids + o, w.bin.sorted_ids, n * 4, cudaMemcpyDeviceToDevice, s));
        GS_CUDA_CHECK(cudaMemcpyAsync(offsets + o, w.bin.offsets, n * 4, cudaMemcpyDeviceToDevice, s));
        GS_CUDA_CHECK(cudaStreamSynchronize(s));
        for (int j = 0; j < nv; j++) totals[v0 + j] = (int64_t)host_totals[j];
        if (chunk_bin(w, sc, k, host_totals, true, s)) return 1;
        if (point_list) {
            const int64_t P = w.vs.base[nv];
            GS_CUDA_CHECK(cudaMemcpyAsync(ranges + (size_t)v0 * ntiles * 2, w.ranges, (size_t)nv * ntiles * 8, cudaMemcpyDeviceToDevice, s));
            if (P > 0) {
                GS_CUDA_CHECK(cudaMemcpyAsync(point_list + pair0, w.pairs.point_list, (size_t)P * 4, cudaMemcpyDeviceToDevice, s));
                GS_CUDA_CHECK(cudaMemcpyAsync(tile_keys + pair0, w.pairs.tile_keys, (size_t)P * 4, cudaMemcpyDeviceToDevice, s));
            }
            pair0 += P;
        }
        GS_CUDA_CHECK(cudaStreamSynchronize(s));
    }
    return 0;
}

// The multi-view step's batched preprocess, as step_core runs it (chunk_project, chunk_bin; with geom_only the
// host-buffer step's colour-free projection and the colour pass after the binning), with the records copied out.
int32_t gs_b200_debug_preprocess_views(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                                       const float* views_dev, int32_t N, int32_t M, const float* means3D,
                                       const float* shs, const float* colors_precomp, const float* opacities,
                                       const float* scales, const float* rotations, int32_t geom_only, float* recs_out,
                                       void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    GS_REQ(V > 0 && N > 0 && sh_degree >= 0 && sh_degree <= 3 && views_dev && means3D && opacities && scales &&
           rotations && recs_out && (shs == nullptr) != (colors_precomp == nullptr) && (!geom_only || shs) &&
           (!shs || (M >= (sh_degree + 1) * (sh_degree + 1) && M <= 16)), "bad argument");
    const StepScene sc(V, H, W, sh_degree, scale_modifier, views_dev, N, M,
                       param_ptrs(means3D, shs, opacities, scales, rotations, colors_precomp), geom_only != 0);
    ChunkWS w;
    if (w.setup(sc, g_tile_culling.load() >= 1, s)) return 1;
    unsigned long long host_totals[GS_MAX_SEGS];
    for (int k = 0; k < sc.ch.nchunks; k++) {
        if (chunk_project(w, sc, k, host_totals, s)) return 1;
        GS_CUDA_CHECK(cudaStreamSynchronize(s));
        if (chunk_bin(w, sc, k, host_totals, false, s)) return 1;
        GS_CUDA_CHECK(cudaMemcpyAsync(recs_out + (size_t)sc.ch.first(k) * N * 12, w.recs,
                                      (size_t)sc.ch.count(k) * N * sizeof(SplatRec), cudaMemcpyDeviceToDevice, s));
        GS_CUDA_CHECK(cudaStreamSynchronize(s));
    }
    return 0;
}

// The preprocess backward of the multi-view step, as step_core runs it (chunk_backward), from the caller's [V][N]
// radii and SplatGrad; the last chunk over `nparts` Gaussian ranges as with a gradient sink.
int32_t gs_b200_debug_preprocess_backward_multi(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                                                const float* views_dev, int32_t N, int32_t M, const float* means3D,
                                                const float* shs, const float* scales, const float* rotations,
                                                const int32_t* radii, const double* splat_grads, float* grads_dev,
                                                int32_t nparts, void* stream_) {
    GS_REQ(V > 0 && N > 0 && M >= (sh_degree + 1) * (sh_degree + 1) && M <= 16 && nparts >= 1 && views_dev &&
           means3D && shs && scales && rotations && radii && splat_grads && grads_dev, "bad argument");
    const StepScene sc(V, H, W, sh_degree, scale_modifier, views_dev, N, M,
                       param_ptrs(means3D, shs, nullptr, scales, rotations));
    const PackedPtrs grd = carve_packed(grads_dev, N, M, true);
    for (int k = 0; k < sc.ch.nchunks; k++) {
        const size_t o = (size_t)sc.ch.first(k) * N;
        if (chunk_backward(sc, k, radii + o, (const SplatGrad*)splat_grads + o, grd, k + 1 == sc.ch.nchunks ? nparts : 1,
                           nullptr, (cudaStream_t)stream_)) return 1;
    }
    return 0;
}

int32_t gs_b200_step_host(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                          const float* views_host, int32_t N, int32_t M, const float* means3D_host,
                          const float* shs_host, const float* opacities_host, const float* scales_host,
                          const float* rotations_host, const float* dL_dout_host, float* grads_host,
                          float* images_host, int64_t* num_rendered_out, void* stream_) {
    return step_host_impl(__func__, V, H, W, sh_degree, scale_modifier, views_host, N, M, means3D_host, shs_host,
                          opacities_host, scales_host, rotations_host, dL_dout_host, grads_host, nullptr,
                          images_host, num_rendered_out, stream_);
}

int32_t gs_b200_step_host_dev_grads(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                          const float* views_host, int32_t N, int32_t M, const float* means3D_host,
                          const float* shs_host, const float* opacities_host, const float* scales_host,
                          const float* rotations_host, const float* dL_dout_host, float* grads_dev,
                          float* images_host, int64_t* num_rendered_out, void* stream_) {
    return step_host_impl(__func__, V, H, W, sh_degree, scale_modifier, views_host, N, M, means3D_host, shs_host,
                          opacities_host, scales_host, rotations_host, dL_dout_host, nullptr, grads_dev,
                          images_host, num_rendered_out, stream_);
}

}  // extern "C"
