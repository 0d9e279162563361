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

int make_view_args(const gs_b200_view* v, ViewArgs& va) {
    if (!v || !v->bg || !v->viewmatrix || !v->projmatrix || !v->campos) { gs_set_error("view: NULL field"); return 1; }
    if (v->image_height <= 0 || v->image_width <= 0) { gs_set_error("view: bad image size"); return 1; }
    if (v->sh_degree < 0 || v->sh_degree > 3) { gs_set_error("view: sh_degree must be 0..3"); return 1; }
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

int check_inputs(int N, int M, int sh_degree, const float* means3D, const float* shs, const float* colors_precomp,
                 const float* opacities, const float* scales, const float* rotations, const float* cov3D_precomp) {
    if (N < 0) { gs_set_error("N < 0"); return 1; }
    if (N == 0) return 0;      // empty cloud: pointers of empty arrays may legitimately be NULL
    if (!means3D || !opacities) { gs_set_error("means3D/opacities NULL"); return 1; }
    if ((shs == nullptr) == (colors_precomp == nullptr)) {
        gs_set_error("Please provide excatly one of either SHs or precomputed colors!"); return 1;
    }
    const bool sr = scales != nullptr || rotations != nullptr;
    if ((sr && cov3D_precomp) || (!sr && !cov3D_precomp) || (sr && (!scales || !rotations))) {
        gs_set_error("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!"); return 1;
    }
    if (shs && M < (sh_degree + 1) * (sh_degree + 1)) { gs_set_error("shs has %d coefficients, sh_degree %d needs %d", M, sh_degree, (sh_degree + 1) * (sh_degree + 1)); return 1; }
    if (shs && M > 16) { gs_set_error("at most 16 SH coefficients (degree 3) supported, got %d", M); return 1; }
    return 0;
}

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
    if (mode < 0 || mode > 2) { gs_set_error("tile culling mode must be 0, 1 or 2"); return 1; }
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

size_t gs_b200_sort_scratch_bytes(int64_t n) { return gs_sort_scratch_bytes(n); }

int32_t gs_b200_sort_pairs_u32(uint32_t* keys, uint32_t* keys_alt, uint32_t* vals, uint32_t* vals_alt, int64_t n,
                               int32_t begin_bit, int32_t end_bit, void* scratch, int32_t* result_in_alt,
                               void* stream) {
    int r = 0;
    int rc = gs_sort_pairs_u32(keys, keys_alt, vals, vals_alt, n, begin_bit, end_bit, scratch, &r, (cudaStream_t)stream);
    if (result_in_alt) *result_in_alt = r;
    return rc;
}

// ---- forward, split at the one host round-trip (number of (tile,splat) pairs) -----------------
// Phase A: preprocess -> depth sort -> gather-scan -> async D2H of the pair count.
// Phase B (needs P on the host to size the binning buffers): emit -> tile sort -> ranges -> composite.
struct FwdCtx {
    ViewArgs va; int N = 0, M = 0, dbg = 0;
    Allocator A;
    gs_b200_state* state = nullptr;
    SplatRec* recs = nullptr;
    uint32_t *sorted_ids = nullptr, *offsets = nullptr;
    uint4* spans = nullptr;                        // tile culling: per-row tile spans (NULL = full squares)
    unsigned long long* host_total = nullptr;      // pinned
    float *out_color = nullptr, *out_depth = nullptr, *out_alpha = nullptr;
    cudaStream_t s = nullptr;
    FwdCtx(gs_b200_alloc_fn fn, void* user, cudaStream_t st) : A{fn, user, st}, s(st) {}
};

// per-view arrays already produced by the multi-view preprocess (gs_launch_preprocess_multi)
struct PreView { SplatRec* recs; uint32_t *tiles, *dkeys, *ids, *min_key; uint4* spans; };

static int fwd_phase_a(FwdCtx& c, const gs_b200_view* view, int32_t N, int32_t M, const float* means3D,
                       const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                       const float* rotations, const float* cov3D_precomp, float* out_color, float* out_depth,
                       float* out_alpha, int32_t* radii, gs_b200_state* state, unsigned long long* host_total,
                       const PreView* pre = nullptr) {
    cudaStream_t s = c.s;
    if (make_view_args(view, c.va)) return 1;
    if (check_inputs(N, M, view->sh_degree, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp)) return 1;
    if (!out_color || !out_depth || !out_alpha || (N > 0 && !radii) || !state) { gs_set_error("forward: NULL output"); return 1; }
    const ViewArgs& va = c.va;
    c.N = N; c.M = M; c.dbg = view->debug; c.state = state; c.host_total = host_total;
    c.out_color = out_color; c.out_depth = out_depth; c.out_alpha = out_alpha;
    memset(state, 0, sizeof(*state));
    state->num_gaussians = N; state->tiles_x = va.tiles_x; state->tiles_y = va.tiles_y;
    Allocator& A = c.A;
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

    if (pre) c.recs = pre->recs;
    else c.recs = (SplatRec*)A.get(GS_B200_BUF_GEOM, (size_t)N * sizeof(SplatRec), &state->owned[GS_B200_BUF_GEOM]);
    if (A.failed) return 1;
    state->geom = c.recs;
    *host_total = 0;
    if (N > 0) {
        const size_t sort_b = gs_sort_scratch_bytes(N), scan_b = gs_scan_scratch_bytes(N);
        const bool own_spans = !pre && g_tile_culling.load() == 2;
        const size_t sc_bytes = Carver::need(N, 4) * 6 + Carver::need(1, 8) * 2 + Carver::need(sort_b, 1) + Carver::need(scan_b, 1) +
                                (own_spans ? Carver::need(N, 16) : 0);
        void* sc = A.get(GS_B200_BUF_SCRATCH, sc_bytes);
        if (A.failed) return 1;
        Carver cv(sc);
        c.spans = pre ? pre->spans : (own_spans ? cv.take<uint4>(N) : nullptr);
        uint32_t* tiles = cv.take<uint32_t>(N);
        uint32_t* dkeys = cv.take<uint32_t>(N);
        uint32_t* ids = cv.take<uint32_t>(N);
        if (pre) { tiles = pre->tiles; dkeys = pre->dkeys; ids = pre->ids; }
        uint32_t* dkeys_alt = cv.take<uint32_t>(N);
        uint32_t* ids_alt = cv.take<uint32_t>(N);
        c.offsets = cv.take<uint32_t>(N);
        unsigned long long* total = cv.take<unsigned long long>(1);
        uint32_t* min_key = (uint32_t*)cv.take<unsigned long long>(1);
        void* sort_scratch = cv.take<char>(sort_b);
        void* scan_scratch = cv.take<char>(scan_b);
        if (pre) {
            min_key = pre->min_key;       // the multi-view pass has already written records, keys, tiles, spans and radii
        } else {
            GS_CUDA_CHECK(cudaMemsetAsync(min_key, 0xFF, 4, s));
            StageTimer t(0, s);
            if (gs_launch_preprocess(va, N, M, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                                     c.recs, radii, tiles, dkeys, ids, min_key, c.spans, s)) return 1;
        }
        STAGE_CHECK(c.dbg, s, "preprocess");
        int in_alt = 0;
        { StageTimer t(1, s);
        if (gs_sort_pairs_u32_biased(dkeys, dkeys_alt, ids, ids_alt, N, 0, 32, sort_scratch, &in_alt, min_key, s)) return 1; }
        STAGE_CHECK(c.dbg, s, "depth sort");
        c.sorted_ids = in_alt ? ids_alt : ids;
        { StageTimer t(2, s);
        if (gs_scan_gather_u32(tiles, c.sorted_ids, c.offsets, total, N, scan_scratch, s)) return 1; }
        GS_CUDA_CHECK(cudaMemcpyAsync(host_total, total, 8, cudaMemcpyDeviceToHost, s));
    }
    return 0;
}

// caller has made sure the D2H of phase A completed (stream or event sync).  Binning half: emit -> tile sort -> ranges.
static int fwd_phase_b_bin(FwdCtx& c) {
    cudaStream_t s = c.s;
    const ViewArgs& va = c.va;
    gs_b200_state* state = c.state;
    Allocator& A = c.A;
    const unsigned long long P = *c.host_total;
    const int ntiles = va.tiles_x * va.tiles_y;
    if (P >= (1ull << 30)) { gs_set_error("too many (tile,splat) pairs: %llu", P); return 1; }
    state->num_rendered = (int64_t)P;
    const size_t bin_bytes = Carver::need(P, 4) * 2;
    void* bin = A.get(GS_B200_BUF_BINNING, bin_bytes, &state->owned[GS_B200_BUF_BINNING]);
    if (A.failed) return 1;
    Carver cb(bin);
    state->point_list = cb.take<uint32_t>(P);
    state->tile_keys = cb.take<uint32_t>(P);
    if (P > 0) {
        const size_t sort_b = gs_sort_scratch_bytes((int64_t)P);
        void* sc2 = A.get(GS_B200_BUF_SCRATCH, Carver::need(P, 4) * 2 + Carver::need(sort_b, 1));
        if (A.failed) return 1;
        Carver c2(sc2);
        uint32_t* keys_b = c2.take<uint32_t>(P);
        uint32_t* vals_b = c2.take<uint32_t>(P);
        void* sort_scratch = c2.take<char>(sort_b);
        const int tbits = bits_for(ntiles);
        const int npasses = (tbits + 7) / 8;
        // start in the buffer that makes the last pass land in the saved pair
        uint32_t *k0 = (npasses & 1) ? keys_b : state->tile_keys, *v0 = (npasses & 1) ? vals_b : state->point_list;
        uint32_t *k1 = (npasses & 1) ? state->tile_keys : keys_b, *v1 = (npasses & 1) ? state->point_list : vals_b;
        { StageTimer t(3, s);
        if (gs_launch_emit(c.recs, c.spans, c.sorted_ids, c.offsets, c.N, va.tiles_x, va.tiles_y, k0, v0, s)) return 1; }
        STAGE_CHECK(c.dbg, s, "emit");
        int in_alt = 0;
        { StageTimer t(4, s);
        if (gs_sort_pairs_u32(k0, k1, v0, v1, (int64_t)P, 0, tbits, sort_scratch, &in_alt, s)) return 1; }
        STAGE_CHECK(c.dbg, s, "tile sort");
        { StageTimer t(5, s);
        if (gs_launch_ranges(state->tile_keys, (int64_t)P, state->ranges, s)) return 1; }
        STAGE_CHECK(c.dbg, s, "ranges");
    }
    return 0;
}
// composite half of phase B (the only part of the forward that reads the colours in the records)
static int fwd_phase_b_render(FwdCtx& c) {
    cudaStream_t s = c.s;
    const ViewArgs& va = c.va;
    gs_b200_state* state = c.state;
    { StageTimer t(6, s);
    if (gs_launch_render_forward(va, c.recs, state->point_list, state->ranges, c.out_color, c.out_depth, c.out_alpha,
                                 state->n_contrib, state->final_T, s)) return 1; }
    STAGE_CHECK(c.dbg, s, "render");
    return 0;
}
static int fwd_phase_b(FwdCtx& c) { return fwd_phase_b_bin(c) || fwd_phase_b_render(c); }

int32_t gs_b200_rasterize_forward(const gs_b200_view* view, int32_t N, int32_t M, const float* means3D,
                                  const float* shs, const float* colors_precomp, const float* opacities,
                                  const float* scales, const float* rotations, const float* cov3D_precomp,
                                  float* out_color, float* out_depth, float* out_alpha, int32_t* radii,
                                  gs_b200_alloc_fn alloc, void* alloc_user, gs_b200_state* state, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    unsigned long long* hp = pinned_u64();
    if (!hp) { gs_set_error("cudaHostAlloc failed"); return 1; }
    FwdCtx c(alloc, alloc_user, s);
    if (fwd_phase_a(c, view, N, M, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                    out_color, out_depth, out_alpha, radii, state, hp)) return 1;
    GS_CUDA_CHECK(cudaStreamSynchronize(s));
    return fwd_phase_b(c);
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
    if (make_view_args(view, va)) return 1;
    if (check_inputs(N, M, view->sh_degree, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp)) return 1;
    if (!state || !dL_dcolor || !dL_ddepth || !dL_dalpha) { gs_set_error("backward: NULL state/upstream gradient"); return 1; }
    if (N == 0) return 0;
    if (!radii || !dL_dmeans3D || !dL_dmeans2D || !dL_dopacities || (shs && !dL_dshs) || (colors_precomp && !dL_dcolors) ||
        (scales && (!dL_dscales || !dL_drotations)) || (cov3D_precomp && !dL_dcov3D)) {
        gs_set_error("backward: NULL gradient output"); return 1;
    }
    if (state->num_gaussians != N) { gs_set_error("backward: state is for N=%d, got %d", state->num_gaussians, N); return 1; }
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
    if (!state || !keys_out) { gs_set_error("debug_sorted_keys: NULL"); return 1; }
    return gs_launch_sorted_keys((const SplatRec*)state->geom, state->point_list, state->tile_keys,
                                 state->num_rendered, keys_out, (cudaStream_t)stream_);
}

int32_t gs_b200_knn_mean_dist2(const float* points, int32_t N, float* out, void* stream_) {
    return gs_launch_knn(points, N, out, (cudaStream_t)stream_);
}

// ---------------------------------------------------------------------------------
// Multi-view optimisation step (device-resident or host buffers).
//
// Views are software-pipelined over TWO internal streams with per-slot grow-only
// workspaces (no allocation in steady state): while view v's composite kernels
// (instruction-issue bound) run on one stream, view v+1's preprocess / sorts
// (memory bound) run on the other, and the host's wait for v+1's pair count is
// hidden behind the GPU work already queued for v.
// ---------------------------------------------------------------------------------
namespace {

struct Region { void* p = nullptr; size_t cap = 0; };
struct Slot {
    cudaStream_t stream = nullptr;
    Region saved[3];                 // GEOM, BINNING, IMAGE
    Region arena; size_t arena_off = 0, arena_want = 0;
    std::vector<void*> overflow;
    Region sgrad, radii, image, loss_ws;
    unsigned long long* host_total = nullptr;
    cudaEvent_t evA = nullptr, evDone = nullptr;
    bool failed = false;

    static int ensure(Region& r, size_t bytes, cudaStream_t st) {
        if (r.cap >= bytes) return 0;
        if (r.p) { cudaStreamSynchronize(st); cudaFree(r.p); r.p = nullptr; r.cap = 0; }
        const size_t want = bytes + bytes / 4 + 4096;
        if (cudaMalloc(&r.p, want) != cudaSuccess) { gs_set_error("cudaMalloc(%zu) failed", want); return 1; }
        r.cap = want;
        return 0;
    }
    void begin_call() {
        // grow the arena to what the previous call needed in total (so overflow is a warm-up-only path)
        if (arena_want > arena.cap) { release_overflow(); ensure(arena, arena_want, stream); }
        arena_off = 0; arena_want = 0;
    }
    void release_overflow() {
        if (overflow.empty()) return;
        cudaStreamSynchronize(stream);
        for (void* p : overflow) cudaFree(p);
        overflow.clear();
    }
    void* alloc(int tag, size_t bytes) {
        bytes = (bytes + 255) & ~(size_t)255;
        if (tag != GS_B200_BUF_SCRATCH) {
            if (ensure(saved[tag], bytes, stream)) { failed = true; return nullptr; }
            return saved[tag].p;
        }
        arena_want += bytes;
        if (arena_off + bytes <= arena.cap) { void* p = (char*)arena.p + arena_off; arena_off += bytes; return p; }
        void* p = nullptr;
        if (cudaMalloc(&p, bytes) != cudaSuccess) { failed = true; gs_set_error("cudaMalloc(%zu) failed", bytes); return nullptr; }
        overflow.push_back(p);
        return p;
    }
};
void* slot_alloc_cb(void* user, int32_t tag, size_t bytes) { return ((Slot*)user)->alloc(tag, bytes); }

constexpr int NSLOTS = 8;       // the device-resident step alternates between slots 0 and 1; the host-buffer step bins up to 8 views ahead
struct StepCache {
    Slot slot[NSLOTS];
    bool init = false;
    cudaStream_t copy_stream = nullptr, d2h_stream = nullptr, aux_stream = nullptr;
    cudaEvent_t evFork = nullptr, evPB = nullptr, evGeom = nullptr, evColour = nullptr, evD2H = nullptr, evAux = nullptr, evPre[2] = {nullptr, nullptr};
    std::vector<cudaEvent_t> up_ready;          // per view: upstream gradient resident
    Region host_stage;                           // device copies of host inputs (step_host)
    bool busy = false;                           // a view hook must not re-enter the step entries on this thread
    Region ws_recs[2], ws_sg[2], ws_u32[2], ws_spans[2];               // per-chunk [VB][N] arrays of the multi-view step
    int ensure_init() {
        if (init) return 0;
        for (int i = 0; i < NSLOTS; i++) {
            GS_CUDA_CHECK(cudaStreamCreateWithFlags(&slot[i].stream, cudaStreamNonBlocking));
            GS_CUDA_CHECK(cudaEventCreateWithFlags(&slot[i].evA, cudaEventDisableTiming));
            GS_CUDA_CHECK(cudaEventCreateWithFlags(&slot[i].evDone, cudaEventDisableTiming));
            GS_CUDA_CHECK(cudaHostAlloc((void**)&slot[i].host_total, 64, cudaHostAllocDefault));
        }
        GS_CUDA_CHECK(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking));
        GS_CUDA_CHECK(cudaStreamCreateWithFlags(&d2h_stream, cudaStreamNonBlocking));
        GS_CUDA_CHECK(cudaStreamCreateWithFlags(&aux_stream, cudaStreamNonBlocking));
        GS_CUDA_CHECK(cudaEventCreateWithFlags(&evAux, cudaEventDisableTiming));
        for (int i = 0; i < 2; i++) GS_CUDA_CHECK(cudaEventCreateWithFlags(&evPre[i], cudaEventDisableTiming));
        GS_CUDA_CHECK(cudaEventCreateWithFlags(&evD2H, cudaEventDisableTiming));
        GS_CUDA_CHECK(cudaEventCreateWithFlags(&evFork, cudaEventDisableTiming));
        GS_CUDA_CHECK(cudaEventCreateWithFlags(&evPB, cudaEventDisableTiming));
        GS_CUDA_CHECK(cudaEventCreateWithFlags(&evGeom, cudaEventDisableTiming));
        GS_CUDA_CHECK(cudaEventCreateWithFlags(&evColour, cudaEventDisableTiming));
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
struct UserSink { gs_b200_grad_sink fn = nullptr; void* user = nullptr; int nchunks = 1; };
thread_local UserSink g_user_sink;

struct PackedPtrs { float *means, *shs, *opac, *scales, *rots, *m2d; float* colors = nullptr; /* [N,3] instead of shs: forward-only */ };
PackedPtrs carve_packed(float* base, size_t N, size_t M, bool with_m2d) {
    PackedPtrs p;
    p.means = base; p.shs = p.means + N * 3; p.opac = p.shs + N * 3 * M; p.scales = p.opac + N;
    p.rots = p.scales + N * 3; p.m2d = with_m2d ? p.rots + N * 4 : nullptr;
    return p;
}

// Device-resident core.  views_host gives tanfov per view (host side), views_dev the matrices.
// Views are handled in chunks of <= VB: ONE multi-view preprocess pass over the Gaussians for the chunk
// (parameters read once), then per view [depth sort -> scan -> (host: pair count) -> emit -> tile sort ->
// ranges -> composite fwd -> composite bwd] pipelined over the two slot streams, then ONE multi-view
// preprocess-backward pass (parameters read once, gradients written once).
// grad_sink (optional): called after each Gaussian range [first, first+count) of the FINAL preprocess-backward has
// been enqueued on `user`, so a host-buffer caller can start the D2H of that range while the next one computes.
struct GradSink { void (*fn)(void* ctx, int first, int count, cudaStream_t user); void* ctx; int nchunks; };
// view hook (optional): called on the host after view v's forward has been enqueued on its slot stream and before
// its backward is; the callee enqueues, on that stream, whatever turns images[v] into dL_dout[v] (the loss).
// forward_only: no backward at all (render entry).  radii_out (optional): [V][N] per-view radii.
// shs_ready (optional, host-buffer step): the SH block is still being uploaded when the step starts -- `user` is ordered
// after the geometry parameters only.  Projection, depth sort and binning of every view run first (colour-free), the
// colours are filled in when the event fires, then the composites follow.  Needs one slot per view: V <= NSLOTS, else
// the step simply waits for the event first.
struct StepOpts { gs_b200_view_hook hook = nullptr; void* hook_user = nullptr; bool forward_only = false; int32_t* radii_out = nullptr;
                  cudaEvent_t shs_ready = nullptr; };

int step_core(int V, int H, int W, int sh_degree, float scale_modifier, const float* views_host,
              const float* views_dev, int N, int M, const PackedPtrs& par, const float* dL_dout_dev,
              const cudaEvent_t* up_ready, const PackedPtrs& grd, float* images_dev, int64_t* num_rendered_out,
              cudaStream_t user, const GradSink* sink = nullptr, const StepOpts* opts = nullptr) {
    StepCache& C = step_cache();
    if (C.busy) { gs_set_error("step: re-entrant call from a view hook (the per-thread pipeline state is in use)"); return 1; }
    struct BusyGuard { bool& b; explicit BusyGuard(bool& x) : b(x) { b = true; } ~BusyGuard() { b = false; } } busy_guard(C.busy);
    const StepOpts defaults;
    const StepOpts& O = opts ? *opts : defaults;
    if (C.ensure_init()) return 1;
    GradSink user_sink;
    if (!sink && g_user_sink.fn && !O.forward_only) {      // data-parallel caller: all-reduce chunks behind the last pass
        user_sink.ctx = &g_user_sink;
        user_sink.nchunks = g_user_sink.nchunks;
        user_sink.fn = [](void* vp, int first, int count, cudaStream_t st) {
            UserSink* u = (UserSink*)vp;
            u->fn(u->user, first, count, (void*)st);
        };
        sink = &user_sink;
    }
    const size_t npix = (size_t)H * W;
    // View chunks: one batched preprocess / preprocess-backward pass per chunk of <= 16 views, on the aux stream:
    //   aux stream:   pre(0) | pre(1) ............ bwd(0) | pre(2) ....... bwd(1) | ... | bwd(last)
    //   slot streams:          views of chunk 0 ........... views of chunk 1 ......
    // pre(k+1) is enqueued when chunk k's views start, bwd(k) when they have all been enqueued; two workspace sets
    // alternate and the aux stream's own order (bwd(k-1) before pre(k+1)) protects their reuse.
    // GS_B200_STEP_OVERLAP=1 additionally cuts a step of >= 6 views into two chunks so that the batched passes overlap
    // the composites instead of running alone at the head and tail of the step.  Measured on C1 (8 views): 12.25-12.33
    // ms vs 12.09-12.10 ms without — every kernel of the step is issue-bound, so the overlapped passes only take
    // issue slots from the composites, and the second chunk re-reads the parameters.  Off by default.
    const int maxv = std::min(gs_preprocess_multi_max_views(), 16);
    static const bool overlap = []() { const char* e = getenv("GS_B200_STEP_OVERLAP"); return e && e[0] == '1'; }();
    const int nchunks = std::max((overlap && V >= 6) ? 2 : 1, (V + maxv - 1) / maxv);
    const int VB = (V + nchunks - 1) / nchunks;
    const size_t nvb = (size_t)VB * N;
    const bool tight = g_tile_culling.load() >= 1;
    const bool late = O.shs_ready && nchunks == 1 && V <= NSLOTS && par.shs && !par.colors;
    if (O.shs_ready && !late) GS_CUDA_CHECK(cudaStreamWaitEvent(user, O.shs_ready, 0));
    const int nslots_used = late ? V : 2;
    auto slot_of = [&](int j) { return late ? j : (j & 1); };
    struct WS { SplatRec* recs; SplatGrad* sg; int32_t* radii; uint32_t *tiles, *dkeys, *ids, *minkeys; uint4* spans; } ws[2];
    const int nsets = nchunks > 1 ? 2 : 1;
    for (int i = 0; i < nsets; i++) {
        if (Slot::ensure(C.ws_recs[i], nvb * sizeof(SplatRec), user) || Slot::ensure(C.ws_sg[i], nvb * sizeof(SplatGrad), user) ||
            Slot::ensure(C.ws_u32[i], nvb * 4 * 4 + 256 * 4, user)) return 1;
        if (tight && Slot::ensure(C.ws_spans[i], nvb * sizeof(uint4), user)) return 1;
        uint32_t* u32 = (uint32_t*)C.ws_u32[i].p;
        ws[i] = WS{(SplatRec*)C.ws_recs[i].p, (SplatGrad*)C.ws_sg[i].p, (int32_t*)u32, u32 + nvb, u32 + 2 * nvb, u32 + 3 * nvb,
                   u32 + 4 * nvb /* [VB] stride 2 words */, tight ? (uint4*)C.ws_spans[i].p : nullptr};
    }
    cudaStream_t aux = C.aux_stream;
    // everything is ordered after the caller's stream
    GS_CUDA_CHECK(cudaEventRecord(C.evFork, user));
    GS_CUDA_CHECK(cudaStreamWaitEvent(aux, C.evFork, 0));

    auto enqueue_pre = [&](int k) -> int {           // batched preprocess of chunk k on the aux stream
        const int v0 = k * VB, nv = std::min(VB, V - v0);
        const WS& w = ws[k & (nsets - 1)];
        GS_CUDA_CHECK(cudaMemsetAsync(w.minkeys, 0xFF, 256 * 4, aux));
        { StageTimer t(0, aux);
        if (gs_launch_preprocess_multi(views_dev + (size_t)v0 * 40, nv, W, H, sh_degree, scale_modifier, N, M, par.means,
                                       par.shs, par.colors, par.opac, par.scales, par.rots, w.recs, w.radii, w.tiles, w.dkeys, w.ids,
                                       w.minkeys, w.spans, aux, late ? 1 : 0)) return 1; }
        GS_CUDA_CHECK(cudaEventRecord(C.evPre[k & 1], aux));
        return 0;
    };

    gs_b200_state st[NSLOTS];
    gs_b200_view view[NSLOTS];
    std::unique_ptr<FwdCtx> ctx[NSLOTS];            // released on every exit path
    int64_t rendered = 0;
    int rc = enqueue_pre(0);

    for (int k = 0; k < nchunks && !rc; k++) {
        const int v0 = k * VB, nv = std::min(VB, V - v0);
        const WS& w = ws[k & (nsets - 1)];
        // the slot streams continue after this chunk's preprocess ...
        for (int i = 0; i < nslots_used; i++) GS_CUDA_CHECK(cudaStreamWaitEvent(C.slot[i].stream, C.evPre[k & 1], 0));
        // ... while the next chunk's preprocess already runs beside them
        if (k + 1 < nchunks && (rc = enqueue_pre(k + 1))) break;

        auto launch_a = [&](int j) -> int {          // j: view index inside the chunk
            const int q = slot_of(j);
            Slot& S = C.slot[q];
            S.begin_call();
            if (!images_dev && Slot::ensure(S.image, 5 * npix * 4, S.stream)) return 1;
            const int v = v0 + j;
            const float* vh = views_host + (size_t)v * 40;
            const float* vd = views_dev + (size_t)v * 40;
            gs_b200_view& vw = view[q];
            vw.image_height = H; vw.image_width = W; vw.tanfovx = vh[38]; vw.tanfovy = vh[39];
            vw.bg = vd + 35; vw.scale_modifier = scale_modifier; vw.viewmatrix = vd; vw.projmatrix = vd + 16;
            vw.sh_degree = sh_degree; vw.campos = vd + 32; vw.prefiltered = 0; vw.debug = 0;
            float* img = images_dev ? images_dev + (size_t)v * 5 * npix : (float*)S.image.p;
            ctx[q].reset(new FwdCtx(slot_alloc_cb, &S, S.stream));
            const size_t o = (size_t)j * N;
            PreView pre{w.recs + o, w.tiles + o, w.dkeys + o, w.ids + o, w.minkeys + 2 * j, w.spans ? w.spans + o : nullptr};
            if (fwd_phase_a(*ctx[q], &vw, N, M, par.means, par.shs, par.colors, par.opac, par.scales, par.rots, nullptr,
                            img, img + 3 * npix, img + 4 * npix, w.radii + o, &st[q], S.host_total, &pre)) return 1;
            GS_CUDA_CHECK(cudaEventRecord(S.evA, S.stream));
            // The view's SplatGrad slice is zeroed here, on its slot stream, so the write overlaps the other slot's
            // composites instead of delaying the batched preprocess.  Also for a view without pairs, whose composite
            // backward is skipped: the batched preprocess-backward reads the slice for every Gaussian with radii > 0.
            // (Placed after evA, so the host's wait for the pair count does not wait for it too.)
            if (!O.forward_only) GS_CUDA_CHECK(cudaMemsetAsync(w.sg + o, 0, (size_t)N * sizeof(SplatGrad), S.stream));
            return S.failed ? 1 : 0;
        };

        // after view j's forward has been enqueued: loss hook, upstream-gradient wait, composite backward
        auto finish_view = [&](int j) -> int {
            const int q = slot_of(j);
            Slot& S = C.slot[q];
            const int v = v0 + j;
            if (O.forward_only) return S.failed ? 1 : 0;
            if (O.hook && O.hook(O.hook_user, v, (void*)S.stream) != 0) { gs_set_error("step: view hook failed at view %d", v); return 1; }
            const float* up = dL_dout_dev + (size_t)v * 5 * npix;
            if (up_ready) GS_CUDA_CHECK(cudaStreamWaitEvent(S.stream, up_ready[v], 0));
            if (st[q].num_rendered > 0) {
                StageTimer t(7, S.stream);
                if (gs_launch_render_backward(ctx[q]->va, (const SplatRec*)st[q].geom, st[q].point_list, st[q].ranges, st[q].n_contrib,
                                              st[q].final_T, up, up + 3 * npix, up + 4 * npix, w.sg + (size_t)j * N, S.stream)) return 1;
            }
            return S.failed ? 1 : 0;
        };
        if (late) {
            // every view's depth sort and binning first (one slot per view, no colour needed) ...
            for (int j = 0; j < nv && !rc; j++) rc = launch_a(j);
            for (int j = 0; j < nv && !rc; j++) {
                GS_CUDA_CHECK(cudaEventSynchronize(C.slot[j].evA));
                if ((rc = fwd_phase_b_bin(*ctx[j]))) break;
                rendered += st[j].num_rendered;
            }
            // ... the colours as soon as the SH block has arrived, then the composites
            if (!rc) {
                GS_CUDA_CHECK(cudaStreamWaitEvent(aux, O.shs_ready, 0));
                rc = gs_launch_sh_colour_multi(views_dev + (size_t)v0 * 40, nv, sh_degree, N, M, par.means, par.shs, w.radii, w.recs, aux);
                if (!rc) GS_CUDA_CHECK(cudaEventRecord(C.evColour, aux));
            }
            for (int j = 0; j < nv && !rc; j++) {
                GS_CUDA_CHECK(cudaStreamWaitEvent(C.slot[j].stream, C.evColour, 0));
                if ((rc = fwd_phase_b_render(*ctx[j]))) break;
                rc = finish_view(j);
            }
        } else {
            rc = launch_a(0);
            for (int j = 0; j < nv && !rc; j++) {
                Slot& S = C.slot[j & 1];
                if (j + 1 < nv) { rc = launch_a(j + 1); if (rc) break; }
                GS_CUDA_CHECK(cudaEventSynchronize(S.evA));
                if ((rc = fwd_phase_b(*ctx[j & 1]))) break;
                rendered += st[j & 1].num_rendered;
                rc = finish_view(j);
            }
        }
        for (int i = 0; i < NSLOTS; i++) ctx[i].reset();
        // the aux stream picks up after this chunk's views (batched backward, radii copy, workspace hand-over)
        for (int i = 0; i < nslots_used; i++) {
            cudaEventRecord(C.slot[i].evDone, C.slot[i].stream);
            cudaStreamWaitEvent(aux, C.slot[i].evDone, 0);
        }
        if (rc) break;
        if (O.radii_out) GS_CUDA_CHECK(cudaMemcpyAsync(O.radii_out + (size_t)v0 * N, w.radii, (size_t)nv * N * 4, cudaMemcpyDeviceToDevice, aux));
        if (O.forward_only) continue;
        const bool last_chunk = k + 1 == nchunks;
        const int nparts = (sink && last_chunk && sink->nchunks > 1) ? sink->nchunks : 1;
        const int per = (((N + nparts - 1) / nparts) + 127) / 128 * 128;
        for (int first = 0; first < N && !rc; first += per) {
            const int count = std::min(per, N - first);
            { StageTimer t(8, aux);
            rc = gs_launch_preprocess_backward_multi(views_dev + (size_t)v0 * 40, nv, W, H, sh_degree, scale_modifier, N, M,
                                                     par.means, par.shs, par.scales, par.rots, w.radii, w.sg, grd.means,
                                                     grd.m2d, grd.shs, grd.opac, grd.scales, grd.rots, k > 0 ? 1 : 0, first,
                                                     count, aux); }
            if (!rc && sink && last_chunk) sink->fn(sink->ctx, first, count, aux);
        }
    }
    // join: the caller's stream continues after the aux stream (which has waited for both slot streams)
    for (int i = 0; i < nslots_used; i++) {          // (on an error path the slots may not have been joined into aux yet)
        cudaEventRecord(C.slot[i].evDone, C.slot[i].stream);
        cudaStreamWaitEvent(aux, C.slot[i].evDone, 0);
    }
    cudaEventRecord(C.evAux, aux);
    cudaStreamWaitEvent(user, C.evAux, 0);
    if (num_rendered_out) *num_rendered_out = rendered;
    return rc;
}

int step_host_impl(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                   const float* views_host, int32_t N, int32_t M, const float* means3D_host,
                   const float* shs_host, const float* opacities_host, const float* scales_host,
                   const float* rotations_host, const float* dL_dout_host, float* grads_host, float* grads_dev,
                   float* images_host, int64_t* num_rendered_out, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    if (V <= 0 || N <= 0 || !views_host || !means3D_host || !shs_host || !opacities_host || !scales_host ||
        !rotations_host || !dL_dout_host || (!grads_host && !grads_dev)) { gs_set_error("step_host: bad argument"); return 1; }
    StepCache& C = step_cache();
    if (C.ensure_init()) return 1;
    const size_t npix = (size_t)H * W;
    const size_t n_par = (size_t)N * (3 + 3 * (size_t)M + 1 + 3 + 4);
    const size_t n_grad = n_par + (size_t)N * 3;
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
    // at each view's backward), so they stream in behind the compute.  GS_B200_HOST_LATE_SH=0: wait for everything first.
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
    static const bool late_sh = []() { const char* e = getenv("GS_B200_HOST_LATE_SH"); return !(e && e[0] == '0'); }();
    GS_CUDA_CHECK(cudaStreamWaitEvent(s, late_sh ? C.evGeom : C.evPB, 0));
    StepOpts opts;
    if (late_sh) opts.shs_ready = C.evPB;
    // D2H of the summed gradients is chunked over Gaussian ranges and starts as soon as a range is final
    struct SinkCtx { StepCache* C; float* host; float* dev; size_t N, M; } sctx{&C, grads_host, d_grad, (size_t)N, (size_t)M};
    GradSink sink;
    sink.ctx = &sctx; sink.nchunks = grads_host ? 4 : 1;
    sink.fn = [](void* vp, int first, int count, cudaStream_t user) {
        SinkCtx* q = (SinkCtx*)vp;
        if (!q->host) return;
        StepCache& C2 = *q->C;
        cudaEventRecord(C2.evD2H, user);
        cudaStreamWaitEvent(C2.d2h_stream, C2.evD2H, 0);
        const size_t n = q->N, M2 = q->M;
        const size_t goff[6] = {0, 3 * n, 3 * n + 3 * M2 * n, 3 * n + 3 * M2 * n + n, 3 * n + 3 * M2 * n + 4 * n, 3 * n + 3 * M2 * n + 8 * n};
        const size_t per[6] = {3, 3 * M2, 1, 3, 4, 3};          // means | shs | opac | scales | rots | means2D
        for (int gI = 0; gI < 6; gI++) {
            const size_t off = goff[gI] + (size_t)first * per[gI];
            cudaMemcpyAsync(q->host + off, q->dev + off, (size_t)count * per[gI] * 4, cudaMemcpyDeviceToHost, C2.d2h_stream);
        }
    };
    // no memset of the gradient buffer: the first view chunk's preprocess-backward writes every element (accumulate = 0)
    if (step_core(V, H, W, sh_degree, scale_modifier, views_host, d_views, N, M, par, d_up, C.up_ready.data(), grd,
                  d_img, num_rendered_out, s, &sink, &opts)) return 1;
    if (grads_dev) GS_CUDA_CHECK(cudaMemcpyAsync(grads_dev, d_grad, n_grad * 4, cudaMemcpyDeviceToDevice, s));
    if (images_host) GS_CUDA_CHECK(cudaMemcpyAsync(images_host, d_img, (size_t)V * 5 * npix * 4, cudaMemcpyDeviceToHost, s));
    if (grads_host) GS_CUDA_CHECK(cudaStreamSynchronize(C.d2h_stream));
    if (grads_host || images_host) GS_CUDA_CHECK(cudaStreamSynchronize(s));
    return 0;
}
}  // namespace

int32_t gs_b200_set_grad_sink(gs_b200_grad_sink sink, void* user, int32_t nchunks) {
    if (sink && (nchunks < 1 || nchunks > 64)) { gs_set_error("set_grad_sink: nchunks must be 1..64"); return 1; }
    g_user_sink.fn = sink; g_user_sink.user = user; g_user_sink.nchunks = sink ? nchunks : 1;
    return 0;
}

int32_t gs_b200_step_device(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                            const float* views_host, const float* views_dev, int32_t N, int32_t M,
                            const float* means3D, const float* shs, const float* opacities, const float* scales,
                            const float* rotations, const float* dL_dout, float* grads, float* images,
                            int64_t* num_rendered_out, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    if (V <= 0 || N <= 0 || !views_host || !views_dev || !means3D || !shs || !opacities || !scales || !rotations ||
        !dL_dout || !grads) { gs_set_error("step_device: bad argument"); return 1; }
    PackedPtrs par; par.means = (float*)means3D; par.shs = (float*)shs; par.opac = (float*)opacities;
    par.scales = (float*)scales; par.rots = (float*)rotations; par.m2d = nullptr;
    const size_t n_grad = (size_t)N * (3 + 3 * (size_t)M + 1 + 3 + 4) + (size_t)N * 3;
    (void)n_grad;   // grads need no memset: the first chunk's preprocess-backward writes every element
    const PackedPtrs grd = carve_packed(grads, N, M, true);
    return step_core(V, H, W, sh_degree, scale_modifier, views_host, views_dev, N, M, par, dL_dout, nullptr, grd, images,
                     num_rendered_out, s);
}

int32_t gs_b200_step_device_hook(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                                 const float* views_host, const float* views_dev, int32_t N, int32_t M,
                                 const float* means3D, const float* shs, const float* opacities, const float* scales,
                                 const float* rotations, float* dL_dout, float* grads, float* images, int32_t* radii,
                                 gs_b200_view_hook hook, void* hook_user, int64_t* num_rendered_out, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    if (V <= 0 || N <= 0 || !views_host || !views_dev || !means3D || !shs || !opacities || !scales || !rotations ||
        !dL_dout || !grads || !images || !hook) { gs_set_error("step_device_hook: bad argument"); return 1; }
    PackedPtrs par; par.means = (float*)means3D; par.shs = (float*)shs; par.opac = (float*)opacities;
    par.scales = (float*)scales; par.rots = (float*)rotations; par.m2d = nullptr;
    const size_t n_grad = (size_t)N * (3 + 3 * (size_t)M + 1 + 3 + 4) + (size_t)N * 3;
    (void)n_grad;   // grads need no memset: the first chunk's preprocess-backward writes every element
    const PackedPtrs grd = carve_packed(grads, N, M, true);
    StepOpts o; o.hook = hook; o.hook_user = hook_user; o.radii_out = radii;
    return step_core(V, H, W, sh_degree, scale_modifier, views_host, views_dev, N, M, par, dL_dout, nullptr, grd, images,
                     num_rendered_out, s, nullptr, &o);
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
    if (!image || !ref_image || !ref_mask || !dL_dimage || !loss_out) { gs_set_error("image_loss: NULL argument"); return 1; }
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
    cudaStream_t s = (cudaStream_t)stream_;
    if (V <= 0 || N <= 0 || !views_host || !views_dev || !means3D || !shs || !opacities || !scales || !rotations ||
        !ref_images || !ref_masks || !dL_dout || !grads || !images || !losses) { gs_set_error("step_device_train: bad argument"); return 1; }
    if (lambda_ssim > 0.f && (H <= 160 || W <= 160)) { gs_set_error("step_device_train: MS-SSIM needs image sides > 160"); return 1; }
    PackedPtrs par; par.means = (float*)means3D; par.shs = (float*)shs; par.opac = (float*)opacities;
    par.scales = (float*)scales; par.rots = (float*)rotations; par.m2d = nullptr;
    const size_t n_grad = (size_t)N * (3 + 3 * (size_t)M + 1 + 3 + 4) + (size_t)N * 3;
    (void)n_grad;   // grads need no memset: the first chunk's preprocess-backward writes every element
    const PackedPtrs grd = carve_packed(grads, N, M, true);
    TrainLossCtx ctx{H, W, ref_images, ref_masks, lambda_ssim, lambda_alpha, loss_scale, dL_dout, images, losses};
    StepOpts o; o.hook = train_loss_hook; o.hook_user = &ctx; o.radii_out = radii;
    return step_core(V, H, W, sh_degree, scale_modifier, views_host, views_dev, N, M, par, dL_dout, nullptr, grd, images,
                     num_rendered_out, s, nullptr, &o);
}

int32_t gs_b200_render_views(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                             const float* views_host, const float* views_dev, int32_t N, int32_t M,
                             const float* means3D, const float* shs, const float* colors_precomp, const float* opacities,
                             const float* scales, const float* rotations, float* images, int32_t* radii,
                             int64_t* num_rendered_out, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    if (V <= 0 || N <= 0 || !views_host || !views_dev || !means3D || !opacities || !scales || !rotations || !images) {
        gs_set_error("render_views: bad argument"); return 1; }
    if ((shs == nullptr) == (colors_precomp == nullptr)) { gs_set_error("Please provide excatly one of either SHs or precomputed colors!"); return 1; }
    PackedPtrs par; par.means = (float*)means3D; par.shs = (float*)shs; par.colors = (float*)colors_precomp; par.opac = (float*)opacities;
    par.scales = (float*)scales; par.rots = (float*)rotations; par.m2d = nullptr;
    PackedPtrs grd{};
    StepOpts o; o.forward_only = true; o.radii_out = radii;
    return step_core(V, H, W, sh_degree, scale_modifier, views_host, views_dev, N, M, par, nullptr, nullptr, grd, images,
                     num_rendered_out, s, nullptr, &o);
}

int32_t gs_b200_step_host(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                          const float* views_host, int32_t N, int32_t M, const float* means3D_host,
                          const float* shs_host, const float* opacities_host, const float* scales_host,
                          const float* rotations_host, const float* dL_dout_host, float* grads_host,
                          float* images_host, int64_t* num_rendered_out, void* stream_) {
    return step_host_impl(V, H, W, sh_degree, scale_modifier, views_host, N, M, means3D_host, shs_host,
                          opacities_host, scales_host, rotations_host, dL_dout_host, grads_host, nullptr,
                          images_host, num_rendered_out, stream_);
}

int32_t gs_b200_step_host_dev_grads(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                          const float* views_host, int32_t N, int32_t M, const float* means3D_host,
                          const float* shs_host, const float* opacities_host, const float* scales_host,
                          const float* rotations_host, const float* dL_dout_host, float* grads_dev,
                          float* images_host, int64_t* num_rendered_out, void* stream_) {
    return step_host_impl(V, H, W, sh_degree, scale_modifier, views_host, N, M, means3D_host, shs_host,
                          opacities_host, scales_host, rotations_host, dL_dout_host, nullptr, grads_dev,
                          images_host, num_rendered_out, stream_);
}

// ---- optimisation-step kernels (gs_train.cu) -------------------------------------------------------------

int32_t gs_b200_activate(int32_t N, const float* raw_opacities, const float* raw_scales, const float* raw_rotations,
                         float* opacities, float* scales, float* rotations, void* stream_) {
    if (N > 0 && (!raw_opacities || !raw_scales || !raw_rotations || !opacities || !scales || !rotations)) { gs_set_error("activate: NULL"); return 1; }
    return gs_launch_activate(N, raw_opacities, raw_scales, raw_rotations, opacities, scales, rotations, (cudaStream_t)stream_);
}
int32_t gs_b200_adam_step(int32_t N, int32_t M, const float* lrs6_host, float beta1, float beta2, float eps, int32_t step,
                          float grad_scale, const float* grads_packed, float* params_packed, float* exp_avg,
                          float* exp_avg_sq, void* stream_) {
    if (!lrs6_host || step < 1 || (N > 0 && (!grads_packed || !params_packed || !exp_avg || !exp_avg_sq))) { gs_set_error("adam_step: bad argument"); return 1; }
    return gs_launch_adam(N, M, lrs6_host, beta1, beta2, eps, step, grad_scale, grads_packed, params_packed, exp_avg, exp_avg_sq, (cudaStream_t)stream_);
}
int32_t gs_b200_densify_stats(int32_t N, const float* dL_dmeans2D, const int32_t* radii, float* xyz_gradient_accum,
                              float* denom, float* max_radii2D, void* stream_) {
    if (N > 0 && (!dL_dmeans2D || !radii || !xyz_gradient_accum || !denom || !max_radii2D)) { gs_set_error("densify_stats: NULL"); return 1; }
    return gs_launch_densify_stats(N, dL_dmeans2D, radii, xyz_gradient_accum, denom, max_radii2D, (cudaStream_t)stream_);
}

}  // extern "C"
