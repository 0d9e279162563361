/*
 * ngp_b200.h — C ABI of the H100-native Instant-NGP path: multiresolution hash-grid encoding, occupancy-grid
 * ray marching, packed volume-rendering weights and per-ray accumulation.
 *
 * Replaces, for MVs_Algorithms/NeRF/Instant_NGP.py (and Gen_3D_Modules/LGM/nerf_marching_cubes_converter.py),
 * the kernels of the un-vendored packages kiui.gridencoder (torch-ngp grid encoder; Instant_NGP.py:22,32-33,73,80,195)
 * and nerfacc 0.5.3 (OccGridEstimator.sampling :129-138, render_weight_from_density :147,
 * accumulate_along_rays :148-149).  Device pointers, fp32/int32/int64, row-major; 0 = ok, else
 * gs_b200_last_error(); work is enqueued on `stream`.
 */
#ifndef NGP_B200_H
#define NGP_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* ---- hash grid (level_dim C = 2) ------------------------------------------------------------------
 * x[N,3] in [-bound,bound]; emb[offsets[L], 2]; offsets = HOST array of L+1 int32 (entries per level, computed
 * as the package does); out[N, 2L].  per-level scale = 2^(l*S)*base_res - 1 in fp32 with S = (float)log2(per_level_scale)
 * taken in double (as torch-ngp does: the scale of config 3's levels 3, 6, 9, ... is an integer only that way),
 * resolution = ceil(scale)+1;
 * dense indexing while (res+1)^3 <= level size, else XOR hash with primes {1, 2654435761, 805459861}. */
int32_t ngp_b200_grid_encode_fwd(const float* x, int64_t N, const float* emb, const int32_t* offsets, int32_t L,
                                 float bound, double per_level_scale, int32_t base_resolution, float* out, void* stream);
/* d_emb is ADDED to (caller zeroes) */
int32_t ngp_b200_grid_encode_bwd(const float* x, int64_t N, const int32_t* offsets, int32_t L, float bound,
                                 double per_level_scale, int32_t base_resolution, const float* dL_dout, float* d_emb,
                                 void* stream);
/* GridEncoder.grad_total_variation: adds weight * L1-TV gradient at the cells containing x[N,3] to d_emb */
int32_t ngp_b200_grid_tv_grad(const float* x, int64_t N, const float* emb, const int32_t* offsets, int32_t L,
                              float bound, double per_level_scale, int32_t base_resolution, float weight, float* d_emb,
                              void* stream);

/* ---- occupancy-grid marching ---------------------------------------------------------------------------
 * binary[R,R,R] uint8 indexed [x][y][z]; aabb[6]; fixed step dt; t_offset[n_rays] optional (stratified) or NULL.
 * Two phases: count -> (host reads total) -> write.  counts/offsets are uint32[n_rays]. */
size_t ngp_b200_march_scratch_bytes(int64_t n_rays, int32_t R);
int32_t ngp_b200_march_count(const float* rays_o, const float* rays_d, int64_t n_rays, const uint8_t* binary, int32_t R,
                             const float* aabb_host6, float near_plane, float far_plane, float dt, const float* t_offset,
                             uint32_t* counts, uint32_t* offsets, unsigned long long* total_dev, void* scratch, void* stream);
int32_t ngp_b200_march_write(const float* rays_o, const float* rays_d, int64_t n_rays, int32_t R,
                             const float* aabb_host6, float near_plane, float far_plane, float dt, const float* t_offset,
                             const uint32_t* offsets, int64_t* ray_indices, float* t_starts, float* t_ends,
                             void* scratch, void* stream);

/* ---- packed volume rendering -----------------------------------------------------------------------------
 * ray_indices[S] int64 sorted ascending; ranges[n_rays,2] int32 (start,count) is filled by ngp_b200_ray_ranges. */
int32_t ngp_b200_ray_ranges(const int64_t* ray_indices, int64_t S, int64_t n_rays, int32_t* ranges, void* stream);
int32_t ngp_b200_weights_fwd(const float* t_starts, const float* t_ends, const float* sigmas, const int32_t* ranges,
                             int64_t n_rays, float* weights, float* trans, float* alphas, void* stream);
int32_t ngp_b200_weights_bwd(const float* t_starts, const float* t_ends, const float* sigmas, const int32_t* ranges,
                             int64_t n_rays, const float* trans, const float* alphas, const float* g_weights,
                             const float* g_trans, const float* g_alphas, float* d_sigmas, void* stream);
/* out[n_rays,C] = sum_i w_i * values_i (values NULL -> C=1, sum of weights) */
int32_t ngp_b200_accumulate_fwd(const float* weights, const float* values, int32_t C, const int32_t* ranges,
                                int64_t n_rays, float* out, void* stream);
int32_t ngp_b200_accumulate_bwd(const float* weights, const float* values, int32_t C, const int64_t* ray_indices,
                                int64_t S, const float* g_out, float* d_weights, float* d_values, void* stream);
/* ---- fused tiny MLP: y = W2 relu(W1 x), no bias (kiui.nn.MLP(dim_in, dim_out, 32, 2, bias=False), Instant_NGP.py:34-35)
 * X[N,Din], W1[H,Din], W2[Dout,H] (torch Linear weight layout), Y[N,Dout].  Supported: H=32, Din in {24,32}, Dout 1..4
 * (ngp_b200_mlp2_supported); other shapes stay on the library GEMM path in the host wrapper.
 * Backward: GX[N,Din] written (may be NULL), GW1/GW2 ADDED to (caller zeroes). */
int32_t ngp_b200_mlp2_supported(int32_t Din, int32_t H, int32_t Dout);
int32_t ngp_b200_mlp2_fwd(const float* X, int64_t N, int32_t Din, int32_t H, int32_t Dout, const float* W1, const float* W2,
                          float* Y, void* stream);
int32_t ngp_b200_mlp2_bwd(const float* X, int64_t N, int32_t Din, int32_t H, int32_t Dout, const float* W1, const float* W2,
                          const float* GY, float* GX, float* GW1, float* GW2, void* stream);

/* ---- marching cubes (PyMCubes marching_cubes(volume, iso); mesh_processer/mesh_utils.py:509, LGM
 * nerf_marching_cubes_converter.py:245) ---------------------------------------------------------------------
 * volume[X,Y,Z] fp32 C-contiguous; a corner is above iff value > iso.  Two phases: count -> (host copies totals_dev3)
 * -> write.  totals = {vertices, triangles, non-finite flag}.  verts[V,3] fp32: column c is the coordinate along array
 * axis c, in index units; tris[F,3] int32, counter-clockwise seen from the below-iso side.  Vertices are ordered by
 * (owner grid point, axis), triangles by (cell, case-table order).  A dimension < 2 gives V = F = 0.  write fails,
 * before writing anything, on a non-finite sample or when V or F reaches 2^31.  scratch >= mcubes_scratch_bytes and
 * is passed unchanged from count to write. */
size_t ngp_b200_mcubes_scratch_bytes(int32_t X, int32_t Y, int32_t Z);
int32_t ngp_b200_mcubes_count(const float* volume, int32_t X, int32_t Y, int32_t Z, float iso,
                              unsigned long long* totals_dev3, void* scratch, void* stream);
int32_t ngp_b200_mcubes_write(const float* volume, int32_t X, int32_t Y, int32_t Z, float iso,
                              const unsigned long long* totals_host3, float* verts, int32_t* tris, void* scratch,
                              void* stream);
#ifdef __cplusplus
}
#endif
#endif
