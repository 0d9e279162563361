// Shared definitions for the sm_90a (H100) Gaussian-splatting kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

// SMs of an H100 SXM: capped and persistent grids are sized as small multiples of it.
#define GS_NUM_SMS 132

#define GS_TILE 16
#define GS_TILE_PIX 256

// Real SH constants — shared_utils/sh_utils.py:26-54 of the reference.
#define SH_C0 0.28209479177387814f
#define SH_C1 0.4886025119029199f
#define SH_C2_0 1.0925484305920792f
#define SH_C2_1 -1.0925484305920792f
#define SH_C2_2 0.31539156525252005f
#define SH_C2_3 -1.0925484305920792f
#define SH_C2_4 0.5462742152960396f
#define SH_C3_0 -0.5900435899266435f
#define SH_C3_1 2.890611442640554f
#define SH_C3_2 -0.4570457994644658f
#define SH_C3_3 0.3731763325901154f
#define SH_C3_4 -0.4570457994644658f
#define SH_C3_5 1.445305721320277f
#define SH_C3_6 -0.5900435899266435f

// Per-Gaussian splat record, 48 B = 3 x 128-bit, written by preprocess and
// gathered (3 x LDG.128) by the composite kernels.
struct __align__(16) SplatRec {
    float4 g;   // px, py, depth, radius(int bits)
    float4 c;   // conic pre-scaled to log2 units: -0.5*log2e*A, -log2e*B, -0.5*log2e*C ; opacity
    float4 k;   // r, g, b, tiles_touched(uint bits)
};

// Per-Gaussian gradient accumulator filled by the composite backward (atomics).  Every tile adds its fp32 partial sums
// in whatever order the CTAs finish.  In fp32 that order changes cancelling sums (the rotation gradient of an isotropic
// splat is all cancellation) by up to an ulp of the largest partial, i.e. by more than the sum itself; the fp64 sums
// here keep the order-dependent error ~2^-29 below that, so the fp32 values read back (sg_f4) differ between runs only
// where a sum lands that close to an fp32 rounding boundary -- not a guarantee, in practice bit-identical.
struct __align__(16) SplatGrad {
    // raw moment sums over the pixels a splat was blended into, w = dL/dG * G, d = mean2D - pixel:
    double4 g;   // sum w*dx, sum w*dy, dL/ddepth, -
    double4 c;   // sum w*dx*dx, sum w*dx*dy, sum w*dy*dy, dL/dopacity
    double4 k;   // dL/dr, dL/dg, dL/db, -
};

__device__ __forceinline__ float4 sg_f4(const double4 d) {
    return make_float4((float)d.x, (float)d.y, (float)d.z, (float)d.w);
}

struct ViewConst {
    float view[16];
    float proj[16];
    float campos[3];
    float bg[3];
    float tanfovx, tanfovy, focal_x, focal_y, scale_modifier;
    int W, H, tiles_x, tiles_y, sh_degree;
};

__device__ __forceinline__ void load_view(ViewConst& vc, const float* view, const float* proj,
                                          const float* campos, const float* bg) {
#pragma unroll
    for (int i = 0; i < 16; i++) { vc.view[i] = __ldg(view + i); vc.proj[i] = __ldg(proj + i); }
#pragma unroll
    for (int i = 0; i < 3; i++) { vc.campos[i] = __ldg(campos + i); vc.bg[i] = __ldg(bg + i); }
}

struct ViewArgs {       // passed by value to kernels
    const float* view; const float* proj; const float* campos; const float* bg;
    float tanfovx, tanfovy, focal_x, focal_y, scale_modifier;
    int W, H, tiles_x, tiles_y, sh_degree;
};

__device__ __forceinline__ void get_rect(float px, float py, int radius, int tiles_x, int tiles_y,
                                         int& x0, int& y0, int& x1, int& y1) {
    float r = (float)radius;
    x0 = min(tiles_x, max(0, (int)((px - r) / (float)GS_TILE)));
    y0 = min(tiles_y, max(0, (int)((py - r) / (float)GS_TILE)));
    x1 = min(tiles_x, max(0, (int)((px + r + (float)(GS_TILE - 1)) / (float)GS_TILE)));
    y1 = min(tiles_y, max(0, (int)((py + r + (float)(GS_TILE - 1)) / (float)GS_TILE)));
}


// ---- staging of per-Gaussian rows ([cnt][row] contiguous in global memory) ----
// Shared layout is [cnt][rowp] with rowp = row|1 (odd stride -> a thread walking
// its own row and a warp walking 32 rows are both bank-conflict free; 3M = 48
// unpadded would be a 16-way conflict).  Global side is 128-bit coalesced.
__device__ __forceinline__ int gs_rowp(int row) { return row | 1; }

__device__ __forceinline__ void gs_stage_rows_in(float* __restrict__ s, const float* __restrict__ g, int cnt, int row,
                                                 int tid, int nthreads) {
    const int rowp = gs_rowp(row);
    const int tot = cnt * row;
    const int nvec = ((reinterpret_cast<size_t>(g) & 15) == 0) ? (tot >> 2) : 0;
    const float4* g4 = reinterpret_cast<const float4*>(g);
    for (int i = tid; i < nvec; i += nthreads) {
        const float4 v = __ldg(g4 + i);
        int r = (4 * i) / row, c = 4 * i - r * row;
        s[r * rowp + c] = v.x; if (++c == row) { c = 0; r++; }
        s[r * rowp + c] = v.y; if (++c == row) { c = 0; r++; }
        s[r * rowp + c] = v.z; if (++c == row) { c = 0; r++; }
        s[r * rowp + c] = v.w;
    }
    for (int i = (nvec << 2) + tid; i < tot; i += nthreads) {
        const int r = i / row, c = i - r * row;
        s[r * rowp + c] = __ldg(g + i);
    }
}

__device__ __forceinline__ void gs_stage_rows_out(const float* __restrict__ s, float* __restrict__ g, int cnt, int row,
                                                  int tid, int nthreads, int accumulate) {
    const int rowp = gs_rowp(row);
    const int tot = cnt * row;
    const int nvec = ((reinterpret_cast<size_t>(g) & 15) == 0) ? (tot >> 2) : 0;
    float4* g4 = reinterpret_cast<float4*>(g);
    for (int i = tid; i < nvec; i += nthreads) {
        int r = (4 * i) / row, c = 4 * i - r * row;
        float4 v;
        v.x = s[r * rowp + c]; if (++c == row) { c = 0; r++; }
        v.y = s[r * rowp + c]; if (++c == row) { c = 0; r++; }
        v.z = s[r * rowp + c]; if (++c == row) { c = 0; r++; }
        v.w = s[r * rowp + c];
        if (accumulate) { const float4 o = g4[i]; v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w; }
        g4[i] = v;
    }
    for (int i = (nvec << 2) + tid; i < tot; i += nthreads) {
        const int r = i / row, c = i - r * row;
        const float v = s[r * rowp + c];
        g[i] = accumulate ? g[i] + v : v;
    }
}

#define GS_CUDA_CHECK(expr)                                                          \
    do {                                                                             \
        cudaError_t _e = (expr);                                                     \
        if (_e != cudaSuccess) {                                                     \
            gs_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return 1;                                                                \
        }                                                                            \
    } while (0)

void gs_set_error(const char* fmt, ...);
void gs_count_launches(int n);     // instrumentation: kernels launched by this library

// ---- launchers implemented in the .cu files --------------------------------
int gs_launch_preprocess(const ViewArgs& va, int N, int M, const float* means3D, const float* shs,
                         const float* colors_precomp, const float* opacities, const float* scales,
                         const float* rotations, const float* cov3D_precomp, SplatRec* recs, int32_t* radii,
                         uint32_t* tiles_touched, uint32_t* depth_keys, uint32_t* ids, uint32_t* min_key,
                         uint4* spans /* NULL = the package's full 3-sigma square */, cudaStream_t s);

int gs_launch_preprocess_backward(const ViewArgs& va, int N, int M, const float* means3D, const float* shs,
                                  const float* colors_precomp, const float* opacities, const float* scales,
                                  const float* rotations, const float* cov3D_precomp, const int32_t* radii,
                                  const SplatGrad* sg, float* dmeans3D, float* dmeans2D, float* dshs,
                                  float* dcolors, float* dopac, float* dscales, float* drots, float* dcov3D,
                                  int accumulate, cudaStream_t s);

int gs_preprocess_multi_max_views();
int gs_launch_preprocess_multi(const float* views_dev, int V, int W, int H, int sh_degree, float scale_modifier, int N,
                               int M, const float* means3D, const float* shs, const float* colors_precomp,
                               const float* opacities, const float* scales, const float* rotations, SplatRec* recs,
                               int32_t* radii, uint32_t* tiles_touched, uint32_t* depth_keys, uint32_t* ids,
                               uint32_t* min_keys, uint4* spans, cudaStream_t s, int geom_only = 0);
// colours of the visible (view, Gaussian) records after a geom_only pass (host-buffer step: SH block arrives late)
int gs_launch_sh_colour_multi(const float* views_dev, int V, int sh_degree, int N, int M, const float* means3D,
                              const float* shs, const int32_t* radii, SplatRec* recs, cudaStream_t s);
int gs_launch_preprocess_backward_multi(const float* views_dev, int V, int W, int H, int sh_degree,
                                        float scale_modifier, int N, int M, const float* means3D, const float* shs,
                                        const float* scales, const float* rotations, const int32_t* radii,
                                        const SplatGrad* sg, float* dmeans3D, float* dmeans2D, float* dshs,
                                        float* dopac, float* dscales, float* drots, int accumulate, int first, int count,
                                        cudaStream_t s);

// image loss + gradient of one view (gs_loss.cu); scratch >= gs_image_loss_scratch_bytes(H, W)
size_t gs_image_loss_scratch_bytes(int H, int W);
int gs_launch_image_loss(int H, int W, const float* img, const float* ref, const float* mask, float lambda_ssim,
                         float lambda_alpha, float scale, float* dL, float* loss_out, void* scratch, cudaStream_t s);

int gs_launch_activate(int, const float*, const float*, const float*, float*, float*, float*, cudaStream_t);
int gs_launch_adam(int, int, const float*, float, float, float, int, float, const float*, float*, float*, float*, cudaStream_t);
int gs_launch_densify_stats(int, const float*, const int32_t*, float*, float*, float*, cudaStream_t);

size_t gs_sort_scratch_bytes(int64_t n);
int gs_sort_pairs_u32(uint32_t* keys, uint32_t* keys_alt, uint32_t* vals, uint32_t* vals_alt, int64_t n,
                      int begin_bit, int end_bit, void* scratch, int* result_in_alt, cudaStream_t s);

int gs_sort_pairs_u32_biased(uint32_t* keys, uint32_t* keys_alt, uint32_t* vals, uint32_t* vals_alt, int64_t n,
                             int begin_bit, int end_bit, void* scratch, int* result_in_alt,
                             const uint32_t* key_bias, cudaStream_t s);

size_t gs_scan_scratch_bytes(int64_t n);
// offsets[i] = exclusive prefix of tiles[ids[i]] (ids may be NULL -> identity); total[0] = sum.
int gs_scan_gather_u32(const uint32_t* tiles, const uint32_t* ids, uint32_t* offsets, unsigned long long* total,
                       int64_t n, void* scratch, cudaStream_t s);

int gs_launch_emit(const SplatRec* recs, const uint4* spans, const uint32_t* sorted_ids, const uint32_t* offsets, int N,
                   int tiles_x, int tiles_y, uint32_t* tile_keys, uint32_t* vals, cudaStream_t s);
int gs_launch_ranges(const uint32_t* sorted_tile_keys, int64_t P, uint32_t* ranges, cudaStream_t s);

int gs_launch_render_forward(const ViewArgs& va, const SplatRec* recs, const uint32_t* point_list,
                             const uint32_t* ranges, float* out_color, float* out_depth, float* out_alpha,
                             uint32_t* n_contrib, float* final_T, cudaStream_t s);
int gs_launch_render_backward(const ViewArgs& va, const SplatRec* recs, const uint32_t* point_list,
                              const uint32_t* ranges, const uint32_t* n_contrib, const float* final_T,
                              const float* dL_dcolor, const float* dL_ddepth, const float* dL_dalpha,
                              SplatGrad* sg, cudaStream_t s);
int gs_launch_sorted_keys(const SplatRec* recs, const uint32_t* point_list, const uint32_t* tile_keys, int64_t P,
                          uint64_t* keys_out, cudaStream_t s);
int gs_launch_knn(const float* points, int N, float* out, cudaStream_t s);
