/*
 * gs_b200.h — C ABI of the H100-native 3D Gaussian-splatting rasterizer.
 *
 * Drop-in boundary for the path ComfyUI-3D-Pack reaches through the third-party
 * Python package `diff_gaussian_rasterization` (ashawkey fork), whose two
 * torch ops `rasterize_gaussians` / `rasterize_gaussians_backward` are what
 *   MVs_Algorithms/GaussianSplatting/main_3DGS_renderer.py:840-936   (render)
 *   MVs_Algorithms/GaussianSplatting/main_3DGS.py:205               (loss.backward)
 *   Gen_3D_Modules/LGM/core/gs.py:57-84, TriplaneGaussian/models/renderer.py:209-304,
 *   Gen_3D_Modules/TRELLIS/trellis/renderers/gaussian_render.py:62-137
 * end up calling.  The reference binds that package by Python import name;
 * this header is the C-level surface a binding (ctypes / pybind / cgo) links.
 * Plain pointers and sizes only — no torch types.  All pointers are DEVICE
 * pointers on the current CUDA device unless a function name ends in `_host`.
 * Every function returns 0 on success, non-zero on error (message via
 * gs_b200_last_error()).  Work is enqueued on `stream` (a cudaStream_t passed
 * as void*; NULL = legacy default stream).
 */
#ifndef GS_B200_H
#define GS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GS_B200_ABI_VERSION 1
#define GS_B200_TILE 16

/* ---- view / settings ------------------------------------------------------
 * Mirrors GaussianRasterizationSettings, the 12-field NamedTuple built at
 * main_3DGS_renderer.py:849-862.  bg/viewmatrix/projmatrix/campos stay device
 * pointers exactly as the reference passes CUDA tensors (no host sync).
 *   viewmatrix = w2c^T   row-major 4x4   (camera_utils.py:205)
 *   projmatrix = w2c^T @ P^T row-major    (camera_utils.py:213)
 */
typedef struct gs_b200_view {
    int32_t image_height;
    int32_t image_width;
    float tanfovx;
    float tanfovy;
    const float* bg;          /* [3]  */
    float scale_modifier;
    const float* viewmatrix;  /* [16] */
    const float* projmatrix;  /* [16] */
    int32_t sh_degree;
    const float* campos;      /* [3]  */
    int32_t prefiltered;      /* accepted, ignored (reference passes False) */
    int32_t debug;            /* accepted; non-zero adds a stream sync + error check per stage */
} gs_b200_view;

/* ---- allocator callback ----------------------------------------------------
 * Replaces the std::function<char*(size_t)> resize callbacks of the package's
 * RasterizeGaussiansCUDA: the caller owns every buffer (SURVEY §8b ownership).
 * tag says what the buffer is for; the callback returns >=256-byte aligned
 * device memory valid on `stream`.  If `alloc` is NULL the library uses
 * cudaMallocAsync on the stream and the caller releases saved state with
 * gs_b200_state_free().
 */
enum { GS_B200_BUF_GEOM = 0, GS_B200_BUF_BINNING = 1, GS_B200_BUF_IMAGE = 2, GS_B200_BUF_SCRATCH = 3 };
typedef void* (*gs_b200_alloc_fn)(void* user, int32_t tag, size_t bytes);

/* ---- state kept between forward and backward -------------------------------
 * (geomBuffer / binningBuffer / imgBuffer of the package.)  Filled by
 * gs_b200_rasterize_forward; pointers live in buffers obtained through the
 * callback, so freeing those buffers frees the state.
 */
typedef struct gs_b200_state {
    void* geom;              /* N x 48 B splat records {px,py,depth,radius | conic a,b,c,opacity | r,g,b,tiles} */
    uint32_t* point_list;    /* [P] Gaussian index per (tile,splat) pair, sorted by (tile, depth, index) */
    uint32_t* tile_keys;     /* [P] tile id per sorted pair */
    uint32_t* ranges;        /* [tiles][2] start,end into point_list */
    uint32_t* n_contrib;     /* [H*W] 1-based position of the last blended splat */
    float* final_T;          /* [H*W] transmittance after the last blended splat */
    int64_t num_rendered;    /* P */
    int32_t num_gaussians;   /* N */
    int32_t tiles_x, tiles_y;
    void* owned[4];          /* non-NULL only when the internal allocator was used */
} gs_b200_state;

int32_t gs_b200_abi_version(void);
const char* gs_b200_last_error(void);

/* Tile culling (no reference counterpart; an optimisation the caller can switch off).  The package's binning lists
 * every tile of each splat's 3-sigma bounding square (duplicateWithKeys); with culling on, tiles in which the
 * splat cannot reach alpha >= 1/255 at any pixel are left out of the list.  Rendered images are bit-identical and
 * gradients equal up to summation order; only point_list / ranges / n_contrib (list positions) differ from the
 * package's.  mode 0: off everywhere; 1 (default): gs_b200_step_* entries only; 2: also rasterize_forward.
 * Initial value can be set with the environment variable GS_B200_TILE_CULLING. */
int32_t gs_b200_set_tile_culling(int32_t mode);
int32_t gs_b200_get_tile_culling(void);

/* Measurement query (no reference counterpart): CTAs per SM of the composite backward kernel as the CUDA
 * occupancy calculator reports it for the current device, with the kernel's launch attributes applied, and the
 * kernel's dynamic shared memory per CTA in bytes. */
int32_t gs_b200_composite_bwd_occupancy(int32_t* ctas_per_sm, int32_t* smem_bytes);

/* Forward — replaces `_C.rasterize_gaussians` as called from
 * GaussianRasterizer.forward (main_3DGS_renderer.py:927-936).
 *   M        number of SH coefficients per channel in `shs` ([N,M,3]); ignored when colors_precomp != NULL
 *   exactly one of shs / colors_precomp, exactly one of (scales,rotations) / cov3D_precomp
 * Outputs (caller-allocated): out_color[3,H,W], out_depth[1,H,W], out_alpha[1,H,W], radii[N] int32.
 */
int32_t gs_b200_rasterize_forward(
    const gs_b200_view* view, int32_t N, int32_t M,
    const float* means3D, const float* shs, const float* colors_precomp, const float* opacities,
    const float* scales, const float* rotations, const float* cov3D_precomp,
    float* out_color, float* out_depth, float* out_alpha, int32_t* radii,
    gs_b200_alloc_fn alloc, void* alloc_user, gs_b200_state* state, void* stream);

/* Backward — replaces `_C.rasterize_gaussians_backward` (triggered by
 * loss.backward(), main_3DGS.py:205).  Gradient outputs are caller-allocated
 * and OVERWRITTEN (accumulate==0) or ADDED TO (accumulate!=0; used by the
 * multi-view optimisation step, which sums views in place):
 *   dL_dmeans3D[N,3] dL_dmeans2D[N,3] (= NDC-space screen gradient, z=0; consumed at main_3DGS_renderer.py:767-769)
 *   dL_dshs[N,M,3] | dL_dcolors[N,3]   dL_dopacities[N,1]
 *   dL_dscales[N,3], dL_drotations[N,4] | dL_dcov3D[N,6]
 * NULL gradient pointers for the unused alternative of each exclusive pair.
 */
int32_t gs_b200_rasterize_backward(
    const gs_b200_view* view, int32_t N, int32_t M,
    const float* means3D, const float* shs, const float* colors_precomp, const float* opacities,
    const float* scales, const float* rotations, const float* cov3D_precomp,
    const int32_t* radii, const gs_b200_state* state,
    const float* dL_dcolor, const float* dL_ddepth, const float* dL_dalpha,
    float* dL_dmeans3D, float* dL_dmeans2D, float* dL_dshs, float* dL_dcolors, float* dL_dopacities,
    float* dL_dscales, float* dL_drotations, float* dL_dcov3D, int32_t accumulate,
    gs_b200_alloc_fn alloc, void* alloc_user, void* stream);

/* Release state buffers obtained with the internal allocator (alloc == NULL). */
int32_t gs_b200_state_free(gs_b200_state* state, void* stream);

/* Parity/debug: reconstruct the 64-bit sorted keys (tile<<32 | float_bits(depth))
 * the package's binning stage would hold, for bit-exact comparison. keys_out[P]. */
int32_t gs_b200_debug_sorted_keys(const gs_b200_state* state, uint64_t* keys_out, void* stream);

/* Tests: the per-Gaussian preprocess backward alone, fed with per-splat sums the caller chooses instead of the
 * composite's.  splat_grads: [V][N][12] double, per splat (sum w dx, sum w dy, dL/ddepth, 0, sum w dx dx,
 * sum w dx dy, sum w dy dy, dL/dopacity, dL/dr, dL/dg, dL/db, 0) with w = dL/dG * G; radii [V][N] as the forward
 * wrote them.  The one-view form is the backward of gs_b200_rasterize_backward (V = 1, same arguments).  The multi-view
 * form runs the backward of the gs_b200_step_* entries through the same code they use: views_dev [V][40] and grads_dev
 * laid out as theirs, the views in the step's chunks (gs_b200_step_view_chunks; the first chunk writes, later ones
 * add), the last chunk over `nparts` Gaussian ranges as with a gradient sink of `nparts` chunks. */
int32_t gs_b200_debug_preprocess_backward(
    const gs_b200_view* view, int32_t N, int32_t M,
    const float* means3D, const float* shs, const float* colors_precomp, const float* opacities,
    const float* scales, const float* rotations, const float* cov3D_precomp,
    const int32_t* radii, const double* splat_grads,
    float* dL_dmeans3D, float* dL_dmeans2D, float* dL_dshs, float* dL_dcolors, float* dL_dopacities,
    float* dL_dscales, float* dL_drotations, float* dL_dcov3D, int32_t accumulate, void* stream);
int32_t gs_b200_debug_preprocess_backward_multi(
    int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier, const float* views_dev,
    int32_t N, int32_t M, const float* means3D, const float* shs, const float* scales, const float* rotations,
    const int32_t* radii, const double* splat_grads, float* grads_dev, int32_t nparts, void* stream);
/* Tests of the binning stage.
 * debug_sort_segmented: the segmented onesweep sort of the binning, nseg (1..16) segments [seg_off[i], seg_off[i+1])
 * of ping-pong key/value arrays (seg_off on the host), on bits [begin_bit, end_bit); key_bias (device, may be NULL):
 * segment i's keys are sorted as key - key_bias[i * bias_stride] (mod 2^32).  *result_in_alt = 1 when the result is
 * in keys_alt / vals_alt.
 * debug_bin_views: the projection and binning of the gs_b200_step_* entries, through the same code: views_dev [V][40]
 * and the parameters as theirs, the views in the step's chunks, tile culling on (tight = 1) or off.  Outputs, [V][N]:
 * radii, tiles_touched, spans (uint32 x 4 per Gaussian, tight only), the depth-sorted keys and Gaussian ids, the
 * exclusive scan offsets; totals[V] (host) the pairs of each view.  Call it first with point_list = NULL to learn the
 * totals; a second call with point_list / tile_keys [sum of totals] (view after view) and ranges [V][tiles][2] also
 * returns the lists.  The pair buffers are filled with 0xFFFFFFFF before the emit, so an unwritten slot shows. */
int32_t gs_b200_debug_sort_segmented(uint32_t* keys, uint32_t* keys_alt, uint32_t* vals, uint32_t* vals_alt,
                                     const int64_t* seg_off, int32_t nseg, int32_t begin_bit, int32_t end_bit,
                                     const uint32_t* key_bias, int32_t bias_stride, int32_t* result_in_alt, void* stream);
int32_t gs_b200_debug_bin_views(int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier,
                                const float* views_dev, int32_t N, int32_t M, const float* means3D, const float* shs,
                                const float* opacities, const float* scales, const float* rotations, int32_t tight,
                                int32_t* radii, uint32_t* tiles_touched, uint32_t* spans, uint32_t* sorted_dkeys,
                                uint32_t* sorted_ids, uint32_t* offsets, int64_t* totals, uint32_t* ranges,
                                uint32_t* point_list, uint32_t* tile_keys, void* stream);
/* The view chunks of the multi-view step for V views: bounds[k] is the first view of chunk k, bounds[nchunks] = V
 * (bounds holds at least V + 1 entries).  Returns nchunks, or -1 on a bad argument.  Host only. */
int32_t gs_b200_step_view_chunks(int32_t V, int32_t* bounds);

/* CUB-free onesweep LSD radix sort of (u32 key, u32 value) pairs on bits
 * [begin_bit,end_bit) — the replacement for cub::DeviceRadixSort::SortPairs in
 * the package's binning stage.  keys/vals are ping-pong pairs of n elements;
 * *result_in_alt receives 1 when the sorted data ended in keys_alt/vals_alt.
 * scratch must hold gs_b200_sort_scratch_bytes(n) bytes. vals may be NULL (keys only). */
size_t gs_b200_sort_scratch_bytes(int64_t n);
int32_t gs_b200_sort_pairs_u32(uint32_t* keys, uint32_t* keys_alt, uint32_t* vals, uint32_t* vals_alt,
                               int64_t n, int32_t begin_bit, int32_t end_bit, void* scratch,
                               int32_t* result_in_alt, void* stream);

/* distCUDA2 replacement (simple_knn._C.distCUDA2, main_3DGS_renderer.py:408,419):
 * mean squared distance to the 3 nearest neighbours. points[N,3] -> out[N]. */
int32_t gs_b200_knn_mean_dist2(const float* points, int32_t N, float* out, void* stream);

/* ---- torch_scatter replacement (scatter_sum / scatter_add, scatter_mean, scatter_max) ---------------------------
 * src, index and out are strided views over one shape of `ndim` dimensions (shape_host: src's shape; out has the
 * same shape with dim_size at `dim`).  Each tensor comes with its element strides (host arrays of ndim int64); the
 * index is int64 and has already been broadcast to src's shape, with stride 0 where it repeats.  out[.., index[e], ..]
 * collects src[e]:
 *   SUM (fp32)  out = (out or +0) + src in ascending position along `dim`, one fp32 add each (a fixed left fold)
 *   SUM (int)   exact integer sums (int32 / int64 wrap)
 *   MEAN (fp32) the fp32 sum, then one division by the number of index entries that hit the slot (at least 1)
 *   MAX         an element replaces the running value only when strictly greater (NaN never does; among equal values
 *               the smallest position wins); the initial value is out's (has_out) or the dtype's lowest, which becomes
 *               0 where nothing won.  argmax: contiguous int64 [out shape], the winner's position along `dim`, or
 *               src's size there where nothing won.
 * has_out = 0: out's prior content is ignored.  Every index value must lie in [0, dim_size): the caller checks it
 * first with gs_b200_scatter_index_range, which writes [min, max] of the index to range_out (2 device int64);
 * values outside are skipped by the kernels, never written.  Sizes: fewer than 2^31 src and out elements, fewer than
 * 2^30 index elements after dropping repeats.  No fp32 atomics: the results have the same bits on every run.
 * scratch: gs_b200_scatter_scratch_bytes(...) bytes (0 = invalid arguments, see gs_b200_last_error).
 * Backward (fp32): grad_src (contiguous [shape]) = grad_out gathered through the index (SUM), divided by the slot's
 * count (MEAN, counts read from the forward's scratch, fwd_scratch), or at the argmax positions only, zero elsewhere
 * (MAX).  MEAN also writes grad_out / count to grad_out_mean (contiguous [out shape]) when it is not NULL. */
#define GS_B200_SCATTER_MAX_DIMS 8
enum { GS_B200_SCATTER_SUM = 0, GS_B200_SCATTER_MEAN = 1, GS_B200_SCATTER_MAX = 2 };
enum { GS_B200_SCATTER_F32 = 0, GS_B200_SCATTER_I32 = 1, GS_B200_SCATTER_I64 = 2 };
int32_t gs_b200_scatter_index_range(int32_t ndim, const int64_t* shape_host, int32_t dim, const int64_t* index,
                                    const int64_t* index_strides_host, int64_t* range_out, void* stream);
size_t gs_b200_scatter_scratch_bytes(int32_t op, int32_t dtype, int32_t ndim, const int64_t* shape_host, int32_t dim,
                                     const int64_t* index_strides_host, int64_t dim_size);
int32_t gs_b200_scatter_forward(int32_t op, int32_t dtype, int32_t ndim, const int64_t* shape_host, int32_t dim,
                                int64_t dim_size, const void* src, const int64_t* src_strides_host, const int64_t* index,
                                const int64_t* index_strides_host, void* out, const int64_t* out_strides_host,
                                int32_t has_out, int64_t* argmax, void* scratch, void* stream);
int32_t gs_b200_scatter_backward(int32_t op, int32_t ndim, const int64_t* shape_host, int32_t dim, int64_t dim_size,
                                 const int64_t* index, const int64_t* index_strides_host, const float* grad_out,
                                 const int64_t* grad_out_strides_host, const int64_t* argmax, const void* fwd_scratch,
                                 float* grad_src, float* grad_out_mean, void* stream);

/* ---- pointnet2_ops replacement (furthest_point_sample, gather / grouping_operation, ball_query, three_nn,
 * three_interpolate) --------------------------------------------------------------------------------------------------
 * Every pointer is a contiguous device array: coordinates fp32 [.., 3], features fp32 [B, C, ..], indices int32.
 * Squared distances are ((dx*dx + dy*dy) + dz*dz) in fp32, one rounding per operation (no FMA contraction).
 *   furthest_point_sample  xyz [B,N,3] -> idx_out [B,npoint].  idx_out[.,0] = 0; running distances start at 1e10;
 *       step s sets temp[k] = fminf(temp[k], d2(k, last)) and picks the largest temp, the smallest index on ties.
 *       A point with (x*x + y*y) + z*z <= 1e-3 (fp32, compared as double) is never updated nor picked; when no point
 *       can be picked the pick is 0, so npoint > N is defined.  N > GS_B200_PN2_FPS_ONCHIP_MAX needs `temp`, B*N
 *       floats of scratch (otherwise it may be NULL).
 *   ball_query  xyz [B,N,3], new_xyz [B,npoint,3] -> idx_out [B,npoint,nsample]: the first nsample k, ascending, with
 *       d2 < radius*radius (fp32); slots past the last hit repeat the first hit, and a query without a hit is all 0.
 *   three_nn  unknown [B,n,3], known [B,m,3] -> dist [B,n,3], idx [B,n,3]: the three smallest (d2, k) in lexicographic
 *       order among k with d2 < +inf (NaN never enters), dist = sqrtf(d2) correctly rounded; unfilled slots (+inf, 0).
 *   gather  features [B,C,N], idx [B,M] -> out [B,C,M]: out[b,c,j] = features[b,c,idx[b,j]], 0 where idx lies outside
 *       [0,N).  gather_operation (M = npoint) and grouping_operation (M = npoint*nsample) share it.
 *   three_interpolate  features [B,C,m], idx [B,n,3], weight [B,n,3] -> out [B,C,n] =
 *       (w0*f0 + w1*f1) + w2*f2, with f = 0 for an idx outside [0,m).
 * Backward (fp32): grad_features [B, C, N + 1], where slot N collects the entries whose idx lies outside [0,N) and is
 * discarded by the caller.  Each slot is +0 plus its contributions in ascending position (j for gather, 3i + k for
 * three_interpolate, whose contribution is grad_out[b,c,i] * weight[b,i,k] rounded once) through
 * gs_b200_scatter_forward's fold: no fp32 atomics, no host read, the same bits on every run.  scratch:
 * gs_b200_pn2_backward_scratch_bytes(B, C, N, M, three) bytes (M = the gather's M, or n with three = 1;
 * 0 = invalid arguments).  Fewer than 2^31 elements per tensor and 2^30 index entries (B*M, B*n*3). */
#define GS_B200_PN2_FPS_ONCHIP_MAX 16384
int32_t gs_b200_pn2_furthest_point_sample(int32_t B, int32_t N, int32_t npoint, const float* xyz, int32_t* idx_out,
                                          float* temp, void* stream);
int32_t gs_b200_pn2_ball_query(int32_t B, int32_t N, int32_t npoint, int32_t nsample, float radius, const float* xyz,
                               const float* new_xyz, int32_t* idx_out, void* stream);
int32_t gs_b200_pn2_three_nn(int32_t B, int32_t n, int32_t m, const float* unknown, const float* known, float* dist,
                             int32_t* idx, void* stream);
int32_t gs_b200_pn2_gather(int32_t B, int32_t C, int32_t N, int32_t M, const float* features, const int32_t* idx,
                           float* out, void* stream);
int32_t gs_b200_pn2_three_interpolate(int32_t B, int32_t C, int32_t m, int32_t n, const float* features,
                                      const int32_t* idx, const float* weight, float* out, void* stream);
size_t gs_b200_pn2_backward_scratch_bytes(int32_t B, int32_t C, int32_t N, int64_t M, int32_t three);
int32_t gs_b200_pn2_gather_backward(int32_t B, int32_t C, int32_t N, int64_t M, const float* grad_out,
                                    const int32_t* idx, float* grad_features, void* scratch, void* stream);
int32_t gs_b200_pn2_three_interpolate_backward(int32_t B, int32_t C, int32_t m, int32_t n, const float* grad_out,
                                               const int32_t* idx, const float* weight, float* grad_features,
                                               void* scratch, void* stream);

/* ---- spconv replacement (spconv.pytorch.SubMConv3d, kernel size 1 or 3, stride 1, dilation 1) ------------------------
 * Rows: indices int32 [N, 4] = (b, x, y, z) in any order (16-byte aligned), features [N, Cin], out [N, Cout] in the same
 * row order; spatial shape [X, Y, Z], batch size B.  weight [Cout, k, k, k, Cin] (spconv 2.x's KRSC layout), bias [Cout]
 * or NULL.  With r = (k - 1) / 2 and offset o = (o0, o1, o2) in {-r..r}^3 (linear index ((o0+r)*k + o1+r)*k + o2+r):
 *   out[i, :] = bias + sum over o of W[:, o + r, :] . in[j, :]
 * where j is the row at (b, x+o0, y+o1, z+o2); a neighbour that is absent, outside [0,X)x[0,Y)x[0,Z) or in another batch
 * item contributes nothing (cross-correlation: on a fully occupied grid this is F.conv3d(dense, W.permute(0,4,1,2,3),
 * padding=r) with the spatial axes in index-column order).  Duplicate coordinates: every lookup resolves to the smallest
 * row among them.  A row with b outside [0,B) or a coordinate outside the grid is nobody's neighbour and has none.
 * k = 1 is a per-row GEMM without a map: every row reads its own features.
 * Neighbour map (k = 3), built on the device with no host read:
 *   nbr int32 [N, 27]: the neighbour's row, -1 when absent.  mask uint32 [N]: bit o set when nbr[i, o] >= 0; bit 31 set
 *   when row i repeats the coordinate of a smaller row.  sorted_keys / sorted_rows uint32 [N]: the rows' keys
 *   ((b*X + x)*Y + y)*Z + z (0xffffffff for an invalid row) in stable ascending order and their rows (bit 31 marks an
 *   invalid row); dgrad reads them.  B*X*Y*Z must not exceed 2^32.  scratch: gs_b200_spconv_map_scratch_bytes(N).
 * dtype GS_B200_SPCONV_F16: fp16 features / weight / bias / out, fp16 x fp16 products summed in fp32 on tensor cores,
 *   bias added in fp32, one rounding to fp16.  GS_B200_SPCONV_F32: fp32 FFMA (not TF32), one fmaf chain per output
 *   over (offset ascending, input channel ascending), then + bias.
 * Backward (same dtype as the forward):
 *   dgrad  grad_features [N, Cin] = the forward loop run with W^T and mirrored offsets over the same map (the map of an
 *          odd-k submanifold conv is symmetric); each coordinate's gradient reaching its smallest row is first summed
 *          over the coordinate's duplicate rows (fp32, ascending row, one rounding), and the duplicates get 0.
 *   wgrad  grad_weight [Cout, k, k, k, Cin] = sum over rows i of grad_out[i] (x) in[nbr[i, o]], and grad_bias [Cout] =
 *          sum of grad_out rows (either may be NULL): fp32 partials over fixed row chunks chosen from the shape alone,
 *          added in ascending chunk order, one rounding to the dtype.
 *   scratch: gs_b200_spconv_backward_scratch_bytes(...) bytes, for either call (0 = invalid arguments).
 * No fp32 atomics anywhere: every output and gradient has the same bits on every run.  N <= GS_B200_SPCONV_MAX_ROWS,
 * fewer than 2^31 elements in features, out and weight. */
enum { GS_B200_SPCONV_F32 = 0, GS_B200_SPCONV_F16 = 1 };
#define GS_B200_SPCONV_MAX_ROWS 1073741823
size_t gs_b200_spconv_map_scratch_bytes(int64_t N);
int32_t gs_b200_spconv_build_map(int64_t N, int32_t B, int32_t X, int32_t Y, int32_t Z, const int32_t* indices,
                                 int32_t* nbr, uint32_t* mask, uint32_t* sorted_keys, uint32_t* sorted_rows,
                                 void* scratch, void* stream);
int32_t gs_b200_spconv_forward(int32_t dtype, int64_t N, int32_t Cin, int32_t Cout, int32_t k, const void* features,
                               const int32_t* nbr, const uint32_t* mask, const void* weight, const void* bias,
                               void* out, void* stream);
size_t gs_b200_spconv_backward_scratch_bytes(int32_t dtype, int64_t N, int32_t Cin, int32_t Cout, int32_t k);
int32_t gs_b200_spconv_dgrad(int32_t dtype, int64_t N, int32_t Cin, int32_t Cout, int32_t k, const void* grad_out,
                             const int32_t* nbr, const uint32_t* mask, const uint32_t* sorted_keys,
                             const uint32_t* sorted_rows, const void* weight, void* grad_features, void* scratch,
                             void* stream);
int32_t gs_b200_spconv_wgrad(int32_t dtype, int64_t N, int32_t Cin, int32_t Cout, int32_t k, const void* features,
                             const void* grad_out, const int32_t* nbr, void* grad_weight, void* grad_bias,
                             void* scratch, void* stream);

/* Multi-view optimisation step with DEVICE-resident buffers: V x (forward + backward), gradients
 * summed over views into `grads` (zeroed first), packed as
 *   means3D[N,3] | shs[N,M,3] | opacities[N] | scales[N,3] | rotations[N,4] | means2D[N,3]
 * (the buffer a data-parallel caller all-reduces).  Views are software-pipelined over two internal
 * streams with persistent workspaces; all work is ordered after `stream` and `stream` continues after it.
 *   views_host / views_dev: the same V x 40 floats (layout below) in host and device memory
 *   dL_dout: device V x [5,H,W]; images: optional device V x [5,H,W] output (NULL = not kept) */
int32_t gs_b200_step_device(
    int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier, const float* views_host,
    const float* views_dev, int32_t N, int32_t M, const float* means3D, const float* shs, const float* opacities,
    const float* scales, const float* rotations, const float* dL_dout, float* grads, float* images,
    int64_t* num_rendered_out, void* stream);

/* Multi-view optimisation step with HOST buffers (the e2e entry: H2D of the
 * Gaussians, V x (forward + backward) with gradients summed over views on the
 * device, D2H of the summed gradients).  Host pointers should be pinned.
 *   views_host: V consecutive records of 40 floats:
 *      [0..15] viewmatrix, [16..31] projmatrix, [32..34] campos, [35..37] bg, [38] tanfovx, [39] tanfovy
 *   dL_dout_host: V x [5,H,W] (3 colour planes, depth, alpha) upstream gradients
 *   grads_host:   [N,(3+3M+1+3+4)] packed per parameter group in the order
 *                 means3D | shs | opacities | scales | rotations  (each contiguous), then means2D [N,3]
 *   images_host:  optional V x [5,H,W] rendered (colour, depth, alpha); may be NULL
 * Upload order: views, geometry parameters, SH block, upstream gradients view by view.  For V <= 8 the step starts
 * as soon as the geometry is resident (projection, sorting and binning of every view need nothing else) and fills the
 * colours into the records when the SH block has landed; images are bit-identical to gs_b200_step_device.
 */
int32_t gs_b200_step_host(
    int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier, const float* views_host,
    int32_t N, int32_t M, const float* means3D_host, const float* shs_host, const float* opacities_host,
    const float* scales_host, const float* rotations_host, const float* dL_dout_host,
    float* grads_host, float* images_host, int64_t* num_rendered_out, void* stream);
/* Same step, but the summed gradients are left on the device: copied (D2D) into
 * grads_dev[N*(11+3M)+3N] instead of going to the host, so a multi-GPU caller can
 * all-reduce them before its own D2H.  grads_host may then be NULL. */
int32_t gs_b200_step_host_dev_grads(
    int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier, const float* views_host,
    int32_t N, int32_t M, const float* means3D_host, const float* shs_host, const float* opacities_host,
    const float* scales_host, const float* rotations_host, const float* dL_dout_host,
    float* grads_dev, float* images_host, int64_t* num_rendered_out, void* stream);

/* Same step with the LOSS inside the pipeline (the reference computes its loss between render and backward,
 * main_3DGS.py:176-205): after view v's forward has been enqueued on an internal stream, `hook(user, v, stream)` is
 * called on the host; it must enqueue ON THAT STREAM the work that reads images[v] ([5,H,W]: rgb, depth, alpha)
 * and writes dL_dout[v]; view v's backward is ordered after it.  Non-zero return aborts the step. */
typedef int32_t (*gs_b200_view_hook)(void* user, int32_t view_index, void* stream);
int32_t gs_b200_step_device_hook(
    int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier, const float* views_host,
    const float* views_dev, int32_t N, int32_t M, const float* means3D, const float* shs, const float* opacities,
    const float* scales, const float* rotations, float* dL_dout, float* grads, float* images,
    int32_t* radii /* optional V x [N] */, gs_b200_view_hook hook, void* hook_user, int64_t* num_rendered_out,
    void* stream);

/* The reference's training loss and its gradient for ONE view, on the device (GaussianSplatting3D.training,
 * main_3DGS.py:184-192; batch of one):
 *   loss = scale * [ (1-lambda_ssim) * L1(img*m, ref*m) + lambda_alpha * MSE(alpha, m)
 *                    + lambda_ssim * (1 - MS_SSIM(ref*m, img*m)) ],   img = clamp(rgb, 0, 1)
 * MS_SSIM as pytorch_msssim.MS_SSIM(data_range=1, size_average=True, channel=3) (11-tap Gaussian, 5 scales), skipped when
 * lambda_ssim == 0 as the reference does.  image: [5,H,W] (rgb | depth | alpha, what the rasterizer entries emit),
 * ref_image [3,H,W], ref_mask [1,H,W]; dL_dimage [5,H,W] (depth plane = 0); loss_out: 1 device float.
 * H and W must exceed 160 when lambda_ssim > 0 (the package's own assertion). */
int32_t gs_b200_image_loss(
    int32_t H, int32_t W, const float* image, const float* ref_image, const float* ref_mask, float lambda_ssim,
    float lambda_alpha, float scale, float* dL_dimage, float* loss_out, void* stream);

/* gs_b200_step_device with that loss evaluated inside the pipeline (per view: forward -> loss + gradient ->
 * backward), no host callback: ref_images V x [3,H,W], ref_masks V x [1,H,W]; loss_scale = 1 / (views in the
 * global batch); losses: V device floats (their sum over all ranks' views is the batch loss); dL_dout V x [5,H,W]
 * receives the upstream gradients that were used; images V x [5,H,W]; radii optional V x [N]. */
int32_t gs_b200_step_device_train(
    int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier, const float* views_host,
    const float* views_dev, int32_t N, int32_t M, const float* means3D, const float* shs, const float* opacities,
    const float* scales, const float* rotations, const float* ref_images, const float* ref_masks, float lambda_ssim,
    float lambda_alpha, float loss_scale, float* dL_dout, float* grads, float* images, int32_t* radii, float* losses,
    int64_t* num_rendered_out, void* stream);

/* Data-parallel hook (no reference counterpart; SURVEY 8e): overlap the gradient all-reduce with the tail of the step.
 * The last pass of every gs_b200_step_device* call (chain rule from per-view splat gradients to the packed parameter
 * gradients) is cut into `nchunks` Gaussian ranges; after the kernel of range [first, first+count) has been enqueued
 * on `stream`, `sink(user, first, count, stream)` is called on the host.  Rows first..first+count of every group of
 * `grads` are final once the work enqueued on `stream` so far has run, so the callee can start the all-reduce of those
 * six slices (ordered after an event on `stream`) while the next range is still being computed.
 * Per calling thread; sink == NULL removes it.  Applies to gs_b200_step_device, _hook and _train. */
typedef void (*gs_b200_grad_sink)(void* user, int32_t first, int32_t count, void* stream);
int32_t gs_b200_set_grad_sink(gs_b200_grad_sink sink, void* user, int32_t nchunks);

/* Forward only over V views that share the Gaussians (render nodes: orbit previews, LGM / TRELLIS style multi-view
 * renders — nodes.py:1130-1163, Gen_3D_Modules/LGM/core/gs.py:41-92): one pass over the parameters for all
 * views, then the per-view pipeline.  Exactly one of shs [N,M,3] / colors_precomp [N,3] (LGM passes colours,
 * core/gs.py:75-84).  images: V x [5,H,W]; radii: optional V x [N] int32 (NULL = not kept). */
int32_t gs_b200_render_views(
    int32_t V, int32_t H, int32_t W, int32_t sh_degree, float scale_modifier, const float* views_host,
    const float* views_dev, int32_t N, int32_t M, const float* means3D, const float* shs, const float* colors_precomp,
    const float* opacities, const float* scales, const float* rotations, float* images, int32_t* radii,
    int64_t* num_rendered_out, void* stream);

/* ---- optimisation step around the rasterizer (SURVEY §8f-1/2; GaussianModel, main_3DGS_renderer.py) -------------
 * Raw (pre-activation) parameters live in ONE packed buffer laid out like the gradient buffer:
 *   xyz[N,3] | shs[N,M,3] (dc = coefficient 0) | opacity[N] | scaling[N,3] | rotation[N,4]
 * gs_b200_activate: exp / sigmoid / normalize of :293-321 (means and SHs are used as they are).
 * gs_b200_adam_step: chain rule through those activations + torch.optim.Adam (betas, eps=1e-15 as :446) with the
 *   six per-group learning rates {xyz, f_dc, f_rest, opacity, scaling, rotation} (host array), `step` = 1-based
 *   Adam step (< 1 is refused), grad_scale multiplies the incoming gradient (1/world for averaged data-parallel
 *   gradients).  The betas are doubles: 1 - beta and the bias corrections are formed in double and rounded once.
 *   grads_packed holds gradients wrt the ACTIVATED values (what gs_b200_step_device produces).
 * gs_b200_densify_stats: add_densification_stats (:767-769) + max_radii2D update (main_3DGS.py:212) for radii > 0. */
int32_t gs_b200_activate(int32_t N, const float* raw_opacities, const float* raw_scales, const float* raw_rotations,
                         float* opacities, float* scales, float* rotations, void* stream);
int32_t gs_b200_adam_step(int32_t N, int32_t M, const float* lrs6_host, double beta1, double beta2, float eps, int32_t step,
                          float grad_scale, const float* grads_packed, float* params_packed, float* exp_avg,
                          float* exp_avg_sq, void* stream);
int32_t gs_b200_densify_stats(int32_t N, const float* dL_dmeans2D, const int32_t* radii, float* xyz_gradient_accum,
                              float* denom, float* max_radii2D, void* stream);

/* ---- densification as stream compaction in the packed layout (SURVEY 8f-2) -----------------------------------------
 * Replaces GaussianModel.densify_and_prune and the optimizer surgery behind it (main_3DGS_renderer.py:543-688,752-781).
 * gs_b200_densify_plan: classifies all N Gaussians (clone / split / prune rules of :641-668,752-781 on the raw
 *   parameters and the statistics of gs_b200_densify_stats) and scans the flags into destination rows.
 *   work: [8][N] u32 (flags, then offsets); counts_dev: 5 x u64 = survivors, kept clones, split parents, split parents
 *   whose children are kept, clones selected before the prune; scratch: gs_b200_densify_scratch_bytes(N).
 *   The caller reads counts_dev (the one host sync), sizes the destination for
 *   N' = survivors + kept clones + 2 x kept split parents and draws z ~ N(0,1) [2 x split parents, 3] (the draw
 *   torch.normal(mean=0, std=stds) makes in densify_and_split, :653, before scaling by std).
 * gs_b200_densify_apply: scatters parameters and both Adam moments from buffers packed for N rows into buffers packed
 *   for N' rows: survivors in order | kept clones | kept split children (first copies, then second copies); new rows
 *   get zero moments (cat_tensors_to_optimizer, :606-625); children = R(q/|q|) (exp(scaling) * z) + xyz with scaling
 *   log(exp(scaling) / 1.6).  Source and destination must not overlap. */
size_t gs_b200_densify_scratch_bytes(int32_t N);
int32_t gs_b200_densify_plan(int32_t N, const float* raw_opacity, const float* raw_scaling, const float* grad_accum,
                             const float* denom, float max_grad, float min_opacity, float extent, float percent_dense,
                             uint32_t* work, uint64_t* counts_dev, void* scratch, void* stream);
int32_t gs_b200_densify_apply(int32_t N, int32_t M, const float* src_raw, const float* src_m1, const float* src_m2,
                              const uint32_t* work, int32_t n_keep, int32_t n_clone, int32_t n_split_parents,
                              int32_t n_split_keep, const float* z, float* dst_raw, float* dst_m1, float* dst_m2, void* stream);

/* ---- instrumentation (bench.py): kernel-launch counter and per-stage CUDA-event timing ------
 * Stages: 0 preprocess, 1 depth sort, 2 scan, 3 emit, 4 tile sort, 5 ranges, 6 composite fwd,
 *         7 composite bwd, 8 preprocess bwd.  Events are recorded on the stream each stage is
 * launched on; gs_b200_profile_read synchronises those events and returns accumulated
 * milliseconds and call counts since the last gs_b200_profile_enable(1). */
#define GS_B200_NSTAGES 9
int64_t gs_b200_launch_count(void);
void gs_b200_profile_enable(int32_t on);
int32_t gs_b200_profile_read(float* ms_out, int32_t* calls_out);

#ifdef __cplusplus
}
#endif
#endif /* GS_B200_H */
