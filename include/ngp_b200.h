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
/* ---- FlexiCubes triangle-mesh extraction (FlexiCubes.__call__, MVs_Algorithms/FlexiCubes/flexicubes.py) on the
 * regular grid of Rx x Ry x Rz cubes: point (i,j,k) = (i*(Ry+1) + j)*(Rz+1) + k, x[P,3] and s[P] fp32 contiguous.
 * Raw weights beta[F,12], alpha[F,8], gamma[F] are fp32 rows with the given row strides (unit column stride), or NULL
 * for all ones; cube (i,j,k) = (i*Ry + j)*Rz + k.  count -> (host copies totals_dev4) -> write.  totals = {dual
 * vertices, L_dev entries, quads, surface cubes}.  write: verts[V,3] (V = vertices + training * quads), faces[T,3]
 * int64 (T = 2 or 4 per quad), L_dev[E].  backward needs no host read: grad_verts[V,3] and grad_ldev[E] in, and any
 * of grad_x[P,3], grad_s[P], grad_beta[F,12], grad_alpha[F,8], grad_gamma[F] (dense, contiguous; NULL = not wanted)
 * written in full, from a fixed summation order (bit-identical from run to run).  scratch >= flexicubes_scratch_bytes
 * is passed unchanged from count to write to backward; workspace >= flexicubes_backward_workspace_bytes. */
size_t ngp_b200_flexicubes_scratch_bytes(int32_t Rx, int32_t Ry, int32_t Rz);
int32_t ngp_b200_flexicubes_count(const float* s, int32_t Rx, int32_t Ry, int32_t Rz,
                                  unsigned long long* totals_dev4, void* scratch, void* stream);
int32_t ngp_b200_flexicubes_write(const float* x, const float* s, const float* beta, int64_t beta_stride,
                                  const float* alpha, int64_t alpha_stride, const float* gamma, int64_t gamma_stride,
                                  int32_t Rx, int32_t Ry, int32_t Rz, double weight_scale, int32_t training,
                                  const unsigned long long* totals_host4, float* verts, int64_t* faces, float* ldev,
                                  void* scratch, void* stream);
size_t ngp_b200_flexicubes_backward_workspace_bytes(const unsigned long long* totals_host4, int32_t training);
int32_t ngp_b200_flexicubes_backward(const float* x, const float* s, const float* beta, int64_t beta_stride,
                                     const float* alpha, int64_t alpha_stride, const float* gamma,
                                     int64_t gamma_stride, int32_t Rx, int32_t Ry, int32_t Rz, double weight_scale,
                                     int32_t training, const unsigned long long* totals_host4, const float* verts,
                                     const float* grad_verts, const float* grad_ldev, float* grad_x, float* grad_s,
                                     float* grad_beta, float* grad_alpha, float* grad_gamma, void* scratch,
                                     void* workspace, void* stream);
/* The same extraction with C >= 1 vertex attributes (the TRELLIS / Stable3DGen FlexiCubes' voxelgrid_colors): raw
 * attrs[P,C] are fp32 rows with row stride attr_row_stride >= C (unit column stride).  Each dual vertex gets
 * sum(beta * uc) / sum(beta) per channel, uc the crossing of sigmoid(attrs) at the edge's ends with the same end
 * weights as its position; training centres get the same gamma-weighted diagonal means.  write_attrs writes
 * vattrs[V,C] next to what write writes, which it writes with the same bits.  backward_attrs takes vattrs and
 * grad_vattrs[V,C] and, besides write's gradients (which now include the attributes' terms), writes grad_attrs[P,C]
 * (contiguous, zero off the surface; NULL = not wanted); workspace >= flexicubes_backward_attrs_workspace_bytes.
 * count is shared: topology does not depend on the attributes. */
int32_t ngp_b200_flexicubes_write_attrs(const float* x, const float* s, const float* beta, int64_t beta_stride,
                                        const float* alpha, int64_t alpha_stride, const float* gamma,
                                        int64_t gamma_stride, int32_t Rx, int32_t Ry, int32_t Rz, double weight_scale,
                                        int32_t training, const unsigned long long* totals_host4, float* verts,
                                        int64_t* faces, float* ldev, const float* attrs, int64_t attr_row_stride,
                                        int32_t C, float* vattrs, void* scratch, void* stream);
size_t ngp_b200_flexicubes_backward_attrs_workspace_bytes(const unsigned long long* totals_host4, int32_t training,
                                                          int32_t C);
int32_t ngp_b200_flexicubes_backward_attrs(const float* x, const float* s, const float* beta, int64_t beta_stride,
                                           const float* alpha, int64_t alpha_stride, const float* gamma,
                                           int64_t gamma_stride, int32_t Rx, int32_t Ry, int32_t Rz,
                                           double weight_scale, int32_t training,
                                           const unsigned long long* totals_host4, const float* verts,
                                           const float* grad_verts, const float* grad_ldev, float* grad_x,
                                           float* grad_s, float* grad_beta, float* grad_alpha, float* grad_gamma,
                                           const float* attrs, int64_t attr_row_stride, int32_t C,
                                           const float* vattrs, const float* grad_vattrs, float* grad_attrs,
                                           void* scratch, void* workspace, void* stream);
/* ---- differentiable dual marching cubes (the diso.DiffDMC contract of TripoSG inference_utils.py:466-472 and
 * Hunyuan3D's DMCSurfaceExtractor; parity with diso's binaries is unpinned) -------------------------------------------
 * grid[X,Y,Z] fp32 C-contiguous; deform[X,Y,Z,3] fp32 in index units, or NULL for none.  The grid is read as if
 * padded by a ring of samples iso + 1 with deform 0 (no copy is made), which closes surfaces cut by the border.
 * Point (i,j,k) sits at (i,j,k) + deform[i,j,k]; a sample is below iff value < iso in fp32.  A cube with a non-finite
 * corner is masked: no vertex, and no quad uses it.  An unmasked cube's case is fc_table.cuh's (bit c = corner c
 * below) and its dual vertices are its fc_group_of groups, with no ambiguity swap.  A crossed edge is crossed from
 * its lower end a: p_a + t (p_b - p_a), t = (iso - s_a) / (s_b - s_a); a vertex is the fp32 mean of its group's
 * crossings in ascending edge order, in unpadded index units, column c divided by dim_c - 1 if `normalize`.  One quad
 * per crossed edge whose 4 cubes are unmasked, starting at the lowest cube, with its right-hand normal pointing from
 * the edge's above end to its below end.  Triangles (quads == 0): (0,1,3),(1,2,3) iff the larger corner cosine of
 * that pair is strictly below that of (0,1,2),(0,2,3), cosines taken on the output vertices.
 * Order: vertices by (padded cube, group), quads by (lower padded point, axis), two triangles per quad in quad order.
 * count -> (host copies totals_dev3) -> write.  totals = {vertices V, quads Q, flags}: flags bit 0/1/2 = some sample
 * is below / above (> iso) / NaN; V = Q = 0 when no sample is NaN and none is below or none above.  write fails,
 * before writing anything, when V or Q reaches 2^31, and with normalize on a dimension < 2.  verts[V,3] fp32,
 * faces[Q,4] or [2Q,3] int32.  backward needs no host read and no workspace (workspace_bytes is 0): grad_verts[V,3]
 * in; grad_grid[X,Y,Z] and grad_deform[X,Y,Z,3] (NULL = not wanted) written in full, each point gathering its up to
 * 6 crossed edges, each edge summing dL/dv / n_group over its unmasked cubes, in fixed order (bit-identical from run
 * to run).  Z <= 3000.  scratch >= dmc_scratch_bytes (~4.3 MB at 513^3) is passed unchanged from count to write to
 * backward. */
size_t ngp_b200_dmc_scratch_bytes(int32_t X, int32_t Y, int32_t Z);
int32_t ngp_b200_dmc_count(const float* grid, int32_t X, int32_t Y, int32_t Z, float iso,
                           unsigned long long* totals_dev3, void* scratch, void* stream);
int32_t ngp_b200_dmc_write(const float* grid, const float* deform, int32_t X, int32_t Y, int32_t Z, float iso,
                           int32_t quads, int32_t normalize, const unsigned long long* totals_host3, float* verts,
                           int32_t* faces, const void* scratch, void* stream);
size_t ngp_b200_dmc_backward_workspace_bytes(int32_t X, int32_t Y, int32_t Z);
int32_t ngp_b200_dmc_backward(const float* grid, const float* deform, int32_t X, int32_t Y, int32_t Z, float iso,
                              int32_t normalize, const unsigned long long* totals_host3, const float* grad_verts,
                              float* grad_grid, float* grad_deform, const void* scratch, void* workspace,
                              void* stream);
#ifdef __cplusplus
}
#endif
#endif
