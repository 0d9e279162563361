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

// The multi-view step's view chunks: nchunks balanced chunks of <= VB views (VB <= 16, one batched preprocess, binning
// and preprocess backward each); chunk k holds views [k VB, min(V, (k + 1) VB)).
struct StepChunks {
    int nchunks, VB;
    explicit StepChunks(int V) {
        const int maxv = std::min(gs_preprocess_multi_max_views(), GS_MAX_SEGS);
        nchunks = (V + maxv - 1) / maxv;
        VB = nchunks > 0 ? (V + nchunks - 1) / nchunks : 0;
    }
};

// Preprocess backward of step chunk k (views [v0, v0 + nv)): the first chunk writes the gradients, later ones add to
// them.  Run over `nparts` Gaussian ranges whose starts are multiples of the kernel's 128-Gaussian CTA; after(first,
// count) follows each range's launch (a gradient sink starts the range's transfer there).
template <class After>
int step_backward_chunk(int k, int nparts, const float* views_chunk, int nv, int W, int H, int sh_degree,
                        float scale_modifier, int N, int M, const float* means, const float* shs, const float* scales,
                        const float* rots, const int32_t* radii, const SplatGrad* sg, float* gmeans, float* gm2d,
                        float* gshs, float* gopac, float* gscales, float* grots, cudaStream_t s, After after) {
    const int per = (((N + nparts - 1) / nparts) + 127) / 128 * 128;
    for (int first = 0; first < N; first += per) {
        const int count = std::min(per, N - first);
        { StageTimer t(8, s);
        if (gs_launch_preprocess_backward_multi(views_chunk, nv, W, H, sh_degree, scale_modifier, N, M, means, shs, scales,
                                                rots, radii, sg, gmeans, gm2d, gshs, gopac, gscales, grots, k > 0 ? 1 : 0,
                                                first, count, s)) return 1; }
        after(first, count);
    }
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

// ---- single-view forward, split at the one host round-trip (number of (tile,splat) pairs) -----------------
// Phase A: preprocess -> binning phase A (one view) -> async D2H of the pair count.
// Phase B (needs P on the host to size the binning buffers): binning phase B -> composite.
struct FwdCtx {
    ViewArgs va; int N = 0, M = 0, dbg = 0;
    Allocator A;
    gs_b200_state* state = nullptr;
    SplatRec* recs = nullptr;
    BinA bin;
    uint4* spans = nullptr;                        // tile culling: per-row tile spans (NULL = full squares)
    unsigned long long* host_total = nullptr;      // pinned
    float *out_color = nullptr, *out_depth = nullptr, *out_alpha = nullptr;
    cudaStream_t s = nullptr;
    FwdCtx(gs_b200_alloc_fn fn, void* user, cudaStream_t st) : A{fn, user, st}, s(st) {}
};

static int fwd_phase_a(FwdCtx& c, const gs_b200_view* view, int32_t N, int32_t M, const float* means3D,
                       const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                       const float* rotations, const float* cov3D_precomp, float* out_color, float* out_depth,
                       float* out_alpha, int32_t* radii, gs_b200_state* state, unsigned long long* host_total) {
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

    c.recs = (SplatRec*)A.get(GS_B200_BUF_GEOM, (size_t)N * sizeof(SplatRec), &state->owned[GS_B200_BUF_GEOM]);
    if (A.failed) return 1;
    state->geom = c.recs;
    *host_total = 0;
    if (N > 0) {
        const bool own_spans = g_tile_culling.load() == 2;
        const size_t sc_bytes = Carver::need(N, 4) * 3 + Carver::need(1, 8) + bin_a_bytes(1, N) + (own_spans ? Carver::need(N, 16) : 0);
        void* sc = A.get(GS_B200_BUF_SCRATCH, sc_bytes);
        if (A.failed) return 1;
        Carver cv(sc);
        c.spans = own_spans ? cv.take<uint4>(N) : nullptr;
        BinA& b = c.bin;
        b.tiles = cv.take<uint32_t>(N);
        b.dkeys = cv.take<uint32_t>(N);
        b.ids = cv.take<uint32_t>(N);
        uint32_t* min_key = (uint32_t*)cv.take<unsigned long long>(1);
        carve_bin_a(cv, b, 1, N);
        b.minkeys = min_key; b.dbg = c.dbg;
        GS_CUDA_CHECK(cudaMemsetAsync(min_key, 0xFF, 4, s));
        { StageTimer t(0, s);
        if (gs_launch_preprocess(va, N, M, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                                 c.recs, radii, b.tiles, b.dkeys, b.ids, min_key, c.spans, s)) return 1; }
        STAGE_CHECK(c.dbg, s, "preprocess");
        if (bin_a(b, host_total, s)) return 1;
    }
    return 0;
}

// caller has made sure the D2H of phase A completed (stream or event sync).  Binning half: emit -> tile sort -> ranges.
static int fwd_phase_b_bin(FwdCtx& c) {
    cudaStream_t s = c.s;
    const ViewArgs& va = c.va;
    gs_b200_state* state = c.state;
    Allocator& A = c.A;
    ViewSpans vs;
    if (view_spans(1, c.host_total, vs)) return 1;
    const int64_t P = vs.base[1];
    state->num_rendered = P;
    const size_t bin_bytes = Carver::need(P, 4) * 2;
    void* bin = A.get(GS_B200_BUF_BINNING, bin_bytes, &state->owned[GS_B200_BUF_BINNING]);
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
        if (bin_b(c.bin, vs, va.tiles_x, va.tiles_y, c.recs, c.spans, o, state->ranges, s)) return 1;
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

int32_t gs_b200_debug_preprocess_backward(const gs_b200_view* view, int32_t N, int32_t M, const float* means3D,
                                          const float* shs, const float* colors_precomp, const float* opacities,
                                          const float* scales, const float* rotations, const float* cov3D_precomp,
                                          const int32_t* radii, const double* splat_grads, float* dL_dmeans3D,
                                          float* dL_dmeans2D, float* dL_dshs, float* dL_dcolors, float* dL_dopacities,
                                          float* dL_dscales, float* dL_drotations, float* dL_dcov3D, int32_t accumulate,
                                          void* stream_) {
    ViewArgs va;
    if (make_view_args(view, va)) return 1;
    if (check_inputs(N, M, view->sh_degree, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp)) return 1;
    if (N > 0 && (!radii || !splat_grads)) { gs_set_error("debug_preprocess_backward: NULL radii/splat_grads"); return 1; }
    return gs_launch_preprocess_backward(va, N, M, means3D, shs, colors_precomp, opacities, scales, rotations,
                                         cov3D_precomp, radii, (const SplatGrad*)splat_grads, dL_dmeans3D, dL_dmeans2D,
                                         dL_dshs, dL_dcolors, dL_dopacities, dL_dscales, dL_drotations, dL_dcov3D,
                                         accumulate, (cudaStream_t)stream_);
}

int32_t gs_b200_step_view_chunks(int32_t V, int32_t* bounds) {
    if (V <= 0 || !bounds) { gs_set_error("step_view_chunks: bad argument"); return -1; }
    const StepChunks ch(V);
    for (int k = 0; k < ch.nchunks; k++) bounds[k] = k * ch.VB;
    bounds[ch.nchunks] = V;
    return ch.nchunks;
}

// The preprocess backward of the multi-view step, as step_core runs it: the same chunks (StepChunks) and the same
// per-chunk launches (step_backward_chunk), the last chunk over `nparts` Gaussian ranges as with a gradient sink.
int32_t gs_b200_debug_preprocess_backward_multi(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                                                const float* views_dev, int32_t N, int32_t M, const float* means3D,
                                                const float* shs, const float* scales, const float* rotations,
                                                const int32_t* radii, const double* splat_grads, float* grads_dev,
                                                int32_t nparts, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    if (V <= 0 || N <= 0 || M < (sh_degree + 1) * (sh_degree + 1) || M > 16 || nparts < 1 || !views_dev || !means3D ||
        !shs || !scales || !rotations || !radii || !splat_grads || !grads_dev) {
        gs_set_error("debug_preprocess_backward_multi: bad argument"); return 1;
    }
    // the step's gradient layout: means 3N | shs 3NM | opacities N | scales 3N | rotations 4N | means2D 3N
    float* gm = grads_dev; float* gsh = gm + 3 * (size_t)N; float* gop = gsh + 3 * (size_t)N * M;
    float* gsc = gop + N; float* grt = gsc + 3 * (size_t)N; float* g2 = grt + 4 * (size_t)N;
    const SplatGrad* sg = (const SplatGrad*)splat_grads;
    const StepChunks ch(V);
    for (int k = 0; k < ch.nchunks; k++) {
        const int v0 = k * ch.VB, nv = std::min(ch.VB, V - v0);
        if (step_backward_chunk(k, k + 1 == ch.nchunks ? nparts : 1, views_dev + (size_t)v0 * 40, nv, W, H, sh_degree,
                                scale_modifier, N, M, means3D, shs, scales, rotations, radii + (size_t)v0 * N,
                                sg + (size_t)v0 * N, gm, g2, gsh, gop, gsc, grt, s, [](int, int) {})) return 1;
    }
    return 0;
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
    // per-chunk workspaces of the multi-view step, two sets that alternate between chunks: [VB][N] arrays of the
    // preprocess and the depth sort, the binning scratch and ranges, and the chunk's pair lists
    Region ws_recs[2], ws_sg[2], ws_u32[2], ws_spans[2], ws_bin[2], ws_pairs[2];
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
struct UserSink { gs_b200_grad_sink fn = nullptr; void* user = nullptr; int nchunks = 1; };
thread_local UserSink g_user_sink;

struct PackedPtrs { float *means, *shs, *opac, *scales, *rots, *m2d; float* colors = nullptr; /* [N,3] instead of shs: forward-only */ };
PackedPtrs carve_packed(float* base, size_t N, size_t M, bool with_m2d) {
    PackedPtrs p;
    p.means = base; p.shs = p.means + N * 3; p.opac = p.shs + N * 3 * M; p.scales = p.opac + N;
    p.rots = p.scales + N * 3; p.m2d = with_m2d ? p.rots + N * 4 : nullptr;
    return p;
}

// Workspace of one view chunk of the multi-view step: [VB][N] preprocess outputs and depth sort, binning scratch and
// [VB][tiles][2] ranges, in five grow-only regions.
struct ChunkWS { SplatRec* recs; SplatGrad* sg; int32_t* radii; uint32_t *minkeys, *ranges; uint4* spans; BinA bin; };
int chunk_ws_setup(ChunkWS& w, Region& r_recs, Region& r_sg, Region& r_u32, Region& r_spans, Region& r_bin, int VB, int N,
                   int ntiles, bool tight, cudaStream_t s) {
    const size_t nvb = (size_t)VB * N;
    if (Slot::ensure(r_recs, nvb * sizeof(SplatRec), s) || Slot::ensure(r_sg, nvb * sizeof(SplatGrad), s) ||
        Slot::ensure(r_u32, nvb * 4 * 4 + 256 * 4, s) ||
        Slot::ensure(r_bin, bin_a_bytes(VB, N) + Carver::need((size_t)VB * ntiles * 2, 4), s)) return 1;
    if (tight && Slot::ensure(r_spans, nvb * sizeof(uint4), s)) return 1;
    uint32_t* u32 = (uint32_t*)r_u32.p;
    w.recs = (SplatRec*)r_recs.p; w.sg = (SplatGrad*)r_sg.p; w.radii = (int32_t*)u32;
    w.minkeys = u32 + 4 * nvb;        // [VB] stride 2 words
    w.spans = tight ? (uint4*)r_spans.p : nullptr;
    w.bin.tiles = u32 + nvb; w.bin.dkeys = u32 + 2 * nvb; w.bin.ids = u32 + 3 * nvb;
    w.bin.minkeys = w.minkeys; w.bin.minkey_stride = 2;
    Carver cb(r_bin.p);
    w.ranges = cb.take<uint32_t>((size_t)VB * ntiles * 2);
    carve_bin_a(cb, w.bin, VB, N);
    return 0;
}
// First half of a chunk's projection and binning (views_chunk: its nv views): preprocess, depth sort, scan, and the
// D2H of the views' pair counts to host_totals.  geom_only: colours follow from gs_launch_sh_colour_multi.
int chunk_bin_a(ChunkWS& w, const float* views_chunk, int nv, int W, int H, int sh_degree, float scale_modifier, int N,
                int M, const PackedPtrs& par, int geom_only, unsigned long long* host_totals, cudaStream_t s) {
    GS_CUDA_CHECK(cudaMemsetAsync(w.minkeys, 0xFF, 256 * 4, s));
    { StageTimer t(0, s);
    if (gs_launch_preprocess_multi(views_chunk, nv, W, H, sh_degree, scale_modifier, N, M, par.means, par.shs, par.colors,
                                   par.opac, par.scales, par.rots, w.recs, w.radii, w.bin.tiles, w.bin.dkeys, w.bin.ids,
                                   w.minkeys, w.spans, s, geom_only)) return 1; }
    w.bin.nv = nv;
    return bin_a(w.bin, host_totals, s);
}
size_t chunk_pairs_bytes(int nv, int64_t P) { return Carver::need(P, 4) * 2 + bin_b_scratch_bytes(nv, P); }
// Second half, once the host has the chunk's pair bases vs (view_spans): the pair lists o carved from `pairs`
// (chunk_pairs_bytes), ranges, emit, tile sort.
int chunk_bin_b(ChunkWS& w, const ViewSpans& vs, void* pairs, BinB& o, int tiles_x, int tiles_y, cudaStream_t s) {
    const int64_t P = vs.base[vs.n];
    Carver cp(pairs);
    o.point_list = cp.take<uint32_t>(P); o.tile_keys = cp.take<uint32_t>(P);
    carve_bin_b_scratch(cp, o, vs.n, P);
    GS_CUDA_CHECK(cudaMemsetAsync(w.ranges, 0, (size_t)vs.n * tiles_x * tiles_y * 2 * 4, s));
    return bin_b(w.bin, vs, tiles_x, tiles_y, w.recs, w.spans, o, w.ranges, s);
}

// Device-resident core.  views_host gives tanfov per view (host side), views_dev the matrices.
// Views are handled in chunks of <= VB.  Per chunk, on the aux stream: ONE multi-view preprocess pass over the
// Gaussians (parameters read once), then the batched binning of all its views (segmented depth sort, gather-scan,
// one host wait for the pair counts, emit, segmented tile sort, ranges).  Then per view, on the slot streams:
// composite forward -> view hook -> SplatGrad zeroing -> composite backward.  Then ONE multi-view
// preprocess-backward pass (parameters read once, gradients written once).
// grad_sink (optional): called after each Gaussian range [first, first+count) of the FINAL preprocess-backward has
// been enqueued on `user`, so a host-buffer caller can start the D2H of that range while the next one computes.
struct GradSink { void (*fn)(void* ctx, int first, int count, cudaStream_t user); void* ctx; int nchunks; };
// view hook (optional): called on the host after view v's forward has been enqueued on its slot stream and before
// its backward is; the callee enqueues, on that stream, whatever turns images[v] into dL_dout[v] (the loss).
// forward_only: no backward at all (render entry).  radii_out (optional): [V][N] per-view radii.
// shs_ready (optional, host-buffer step): the SH block is still being uploaded when the step starts -- `user` is ordered
// after the geometry parameters only.  Projection and binning of each chunk run first (colour-free), the colours are
// filled in when the event fires (sh_colour_multi on the aux stream), then the composites follow.
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
    const int tiles_x = (W + GS_TILE - 1) / GS_TILE, tiles_y = (H + GS_TILE - 1) / GS_TILE, ntiles = tiles_x * tiles_y;
    // View chunks: one batched preprocess + binning / preprocess-backward per chunk of <= 16 views, on the aux stream:
    //   aux stream:   pre+bin(0) | pre+bin(1) ......... bwd(0) | pre+bin(2) ...... bwd(1) | ... | bwd(last)
    //   slot streams:             views of chunk 0 ............. views of chunk 1 .......
    // pre+bin(k+1) is enqueued when chunk k's views start (its second half, after the host has read the pair counts,
    // once they have all been enqueued), bwd(k) after that; two workspace sets alternate and the aux stream's own
    // order (bwd(k-1) before pre(k+1)) protects their reuse.
    const StepChunks chunks(V);
    const int nchunks = chunks.nchunks, VB = chunks.VB;
    const bool tight = g_tile_culling.load() >= 1;
    const bool late = O.shs_ready && par.shs && !par.colors;
    if (O.shs_ready && !late) GS_CUDA_CHECK(cudaStreamWaitEvent(user, O.shs_ready, 0));
    ChunkWS ws[2];
    const int nsets = nchunks > 1 ? 2 : 1;
    for (int i = 0; i < nsets; i++)
        if (chunk_ws_setup(ws[i], C.ws_recs[i], C.ws_sg[i], C.ws_u32[i], C.ws_spans[i], C.ws_bin[i], VB, N, ntiles, tight,
                           user)) return 1;
    cudaStream_t aux = C.aux_stream;
    // everything is ordered after the caller's stream
    GS_CUDA_CHECK(cudaEventRecord(C.evFork, user));
    GS_CUDA_CHECK(cudaStreamWaitEvent(aux, C.evFork, 0));

    int64_t rendered = 0;
    ViewSpans vsp[2];
    BinB pairs[2];
    // first half of chunk k's projection and binning on the aux stream: preprocess, depth sort, scan, pair counts D2H
    auto enqueue_pre = [&](int k) -> int {
        const int v0 = k * VB, nv = std::min(VB, V - v0);
        if (chunk_bin_a(ws[k & (nsets - 1)], views_dev + (size_t)v0 * 40, nv, W, H, sh_degree, scale_modifier, N, M, par,
                        late ? 1 : 0, C.host_totals[k & 1], aux)) return 1;
        GS_CUDA_CHECK(cudaEventRecord(C.evBinA[k & 1], aux));
        return 0;
    };
    // second half, once the chunk's pair counts are on the host: pair buffers, emit, tile sort, ranges (+ colours)
    auto enqueue_bin = [&](int k) -> int {
        const int v0 = k * VB, nv = std::min(VB, V - v0);
        const int q = k & (nsets - 1);
        ChunkWS& w = ws[q];
        GS_CUDA_CHECK(cudaEventSynchronize(C.evBinA[k & 1]));
        ViewSpans& vs = vsp[k & 1];
        if (view_spans(nv, C.host_totals[k & 1], vs)) return 1;
        const int64_t P = vs.base[nv];
        rendered += P;
        // grow-only: the pair lists of all the chunk's views live until its last composite backward
        if (Slot::ensure(C.ws_pairs[q], chunk_pairs_bytes(nv, P), aux)) return 1;
        if (chunk_bin_b(w, vs, C.ws_pairs[q].p, pairs[k & 1], tiles_x, tiles_y, aux)) return 1;
        if (late) {
            GS_CUDA_CHECK(cudaStreamWaitEvent(aux, O.shs_ready, 0));
            if (gs_launch_sh_colour_multi(views_dev + (size_t)v0 * 40, nv, sh_degree, N, M, par.means, par.shs, w.radii, w.recs, aux)) return 1;
        }
        GS_CUDA_CHECK(cudaEventRecord(C.evBin[k & 1], aux));
        return 0;
    };

    int rc = enqueue_pre(0);
    if (!rc) rc = enqueue_bin(0);
    for (int k = 0; k < nchunks && !rc; k++) {
        const int v0 = k * VB, nv = std::min(VB, V - v0);
        const ChunkWS& w = ws[k & (nsets - 1)];
        const ViewSpans& vs = vsp[k & 1];
        const BinB& o = pairs[k & 1];
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
            if ((rc = make_view_args(&vw, va))) break;
            float* img = images_dev ? images_dev + (size_t)v * 5 * npix : (float*)S.image.p;
            Carver cn(S.nc.p);
            uint32_t* n_contrib = cn.take<uint32_t>(npix);
            float* final_T = cn.take<float>(npix);
            const size_t off = (size_t)j * N;
            const SplatRec* recs = w.recs + off;
            const uint32_t* point_list = o.point_list + vs.base[j];
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
            if (vs.base[j + 1] > vs.base[j]) {
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
        const bool last_chunk = k + 1 == nchunks;
        const int nparts = (sink && last_chunk && sink->nchunks > 1) ? sink->nchunks : 1;
        rc = step_backward_chunk(k, nparts, views_dev + (size_t)v0 * 40, nv, W, H, sh_degree, scale_modifier, N, M,
                                 par.means, par.shs, par.scales, par.rots, w.radii, w.sg, grd.means, grd.m2d, grd.shs,
                                 grd.opac, grd.scales, grd.rots, aux, [&](int first, int count) {
                                     if (sink && last_chunk) sink->fn(sink->ctx, first, count, aux);
                                 });
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

// ---- test entries of the binning stage ----------------------------------------------------------------------

int32_t gs_b200_debug_sort_segmented(uint32_t* keys, uint32_t* keys_alt, uint32_t* vals, uint32_t* vals_alt,
                                     const int64_t* seg_off, int32_t nseg, int32_t begin_bit, int32_t end_bit,
                                     const uint32_t* key_bias, int32_t bias_stride, int32_t* result_in_alt, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    if (!seg_off || nseg < 1 || nseg > GS_MAX_SEGS || !result_in_alt) { gs_set_error("debug_sort_segmented: bad argument"); return 1; }
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

// The multi-view step's projection and binning, as step_core runs them (StepChunks, chunk_ws_setup, chunk_bin_a,
// view_spans, chunk_bin_b), on `stream` alone, with every intermediate list copied out.
int32_t gs_b200_debug_bin_views(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                                const float* views_dev, int32_t N, int32_t M, const float* means3D, const float* shs,
                                const float* opacities, const float* scales, const float* rotations, int32_t tight,
                                int32_t* radii, uint32_t* tiles_touched, uint32_t* spans, uint32_t* sorted_dkeys,
                                uint32_t* sorted_ids, uint32_t* offsets, int64_t* totals, uint32_t* ranges,
                                uint32_t* point_list, uint32_t* tile_keys, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    if (V <= 0 || N <= 0 || M < (sh_degree + 1) * (sh_degree + 1) || M > 16 || !views_dev || !means3D || !shs ||
        !opacities || !scales || !rotations || !radii || !tiles_touched || (tight && !spans) || !sorted_dkeys ||
        !sorted_ids || !offsets || !totals || (point_list && (!tile_keys || !ranges))) {
        gs_set_error("debug_bin_views: bad argument"); return 1;
    }
    struct Regions {
        Region r[6];
        ~Regions() { for (Region& x : r) if (x.p) cudaFree(x.p); }
    } R;
    const int tiles_x = (W + GS_TILE - 1) / GS_TILE, tiles_y = (H + GS_TILE - 1) / GS_TILE, ntiles = tiles_x * tiles_y;
    const StepChunks ch(V);
    ChunkWS w;
    if (chunk_ws_setup(w, R.r[0], R.r[1], R.r[2], R.r[3], R.r[4], ch.VB, N, ntiles, tight != 0, s)) return 1;
    PackedPtrs par; par.means = (float*)means3D; par.shs = (float*)shs; par.opac = (float*)opacities;
    par.scales = (float*)scales; par.rots = (float*)rotations; par.m2d = nullptr;
    unsigned long long host_totals[GS_MAX_SEGS];
    int64_t pair0 = 0;        // the chunk's first pair in point_list / tile_keys
    for (int k = 0; k < ch.nchunks; k++) {
        const int v0 = k * ch.VB, nv = std::min(ch.VB, V - v0);
        const size_t o = (size_t)v0 * N, n = (size_t)nv * N;
        if (chunk_bin_a(w, views_dev + (size_t)v0 * 40, nv, W, H, sh_degree, scale_modifier, N, M, par, 0, host_totals, s)) return 1;
        GS_CUDA_CHECK(cudaMemcpyAsync(radii + o, w.radii, n * 4, cudaMemcpyDeviceToDevice, s));
        GS_CUDA_CHECK(cudaMemcpyAsync(tiles_touched + o, w.bin.tiles, n * 4, cudaMemcpyDeviceToDevice, s));
        if (tight) GS_CUDA_CHECK(cudaMemcpyAsync(spans + 4 * o, w.spans, n * 16, cudaMemcpyDeviceToDevice, s));
        GS_CUDA_CHECK(cudaMemcpyAsync(sorted_dkeys + o, w.bin.sorted_dkeys, n * 4, cudaMemcpyDeviceToDevice, s));
        GS_CUDA_CHECK(cudaMemcpyAsync(sorted_ids + o, w.bin.sorted_ids, n * 4, cudaMemcpyDeviceToDevice, s));
        GS_CUDA_CHECK(cudaMemcpyAsync(offsets + o, w.bin.offsets, n * 4, cudaMemcpyDeviceToDevice, s));
        GS_CUDA_CHECK(cudaStreamSynchronize(s));
        for (int j = 0; j < nv; j++) totals[v0 + j] = (int64_t)host_totals[j];
        ViewSpans vs;
        if (view_spans(nv, host_totals, vs)) return 1;
        if (!point_list) continue;      // first call of two: the caller sizes the pair lists from `totals`
        const int64_t P = vs.base[nv];
        if (Slot::ensure(R.r[5], chunk_pairs_bytes(nv, P), s)) return 1;
        // a pair slot the emit leaves unwritten keeps this value through the sort
        GS_CUDA_CHECK(cudaMemsetAsync(R.r[5].p, 0xFF, chunk_pairs_bytes(nv, P), s));
        BinB b;
        if (chunk_bin_b(w, vs, R.r[5].p, b, tiles_x, tiles_y, s)) return 1;
        GS_CUDA_CHECK(cudaMemcpyAsync(ranges + (size_t)v0 * ntiles * 2, w.ranges, (size_t)nv * ntiles * 8, cudaMemcpyDeviceToDevice, s));
        if (P > 0) {
            GS_CUDA_CHECK(cudaMemcpyAsync(point_list + pair0, b.point_list, (size_t)P * 4, cudaMemcpyDeviceToDevice, s));
            GS_CUDA_CHECK(cudaMemcpyAsync(tile_keys + pair0, b.tile_keys, (size_t)P * 4, cudaMemcpyDeviceToDevice, s));
        }
        pair0 += P;
        GS_CUDA_CHECK(cudaStreamSynchronize(s));
    }
    return 0;
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

}  // extern "C"
