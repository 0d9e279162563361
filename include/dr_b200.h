/*
 * dr_b200.h — C ABI of the H100-native mesh rasterisation ops (the nvdiffrast surface ComfyUI-3D-Pack uses).
 *
 * Replaces, for the reference's call sites, the torch ops of the un-vendored package `nvdiffrast.torch`
 * (0.3.3, my-reqs.txt:74):
 *   rasterize   MVs_Algorithms/DiffRastMesh/diff_mesh_renderer.py:97, FlexiCubes/flexicubes_renderer.py:49,
 *               mesh_processer/mesh_utils.py:531
 *   interpolate diff_mesh_renderer.py:104,110,131; FlexiCubes/util.py:90-93; mesh_utils.py:534
 *   texture     diff_mesh_renderer.py:105 (filter_mode='linear')
 *   antialias   diff_mesh_renderer.py:101,138; flexicubes_renderer.py:55
 * Plain device pointers + sizes, fp32 / int32, row-major contiguous; every function returns 0 or non-zero with
 * the message in gs_b200_last_error() (shared with gs_b200.h); work is enqueued on `stream`.
 * Layouts: pos[B,V,4] clip space; tri[F,3]; rast[B,H,W,4] = (u, v, z/w, id+1), row 0 = bottom row;
 * rast_db[B,H,W,4] = (du/dX, du/dY, dv/dX, dv/dY) per pixel.
 */
#ifndef DR_B200_H
#define DR_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* scratch for rasterize: B*H*W 64-bit depth/id words + a queue for large triangles */
size_t dr_b200_rasterize_scratch_bytes(int32_t B, int32_t F, int32_t H, int32_t W);
int32_t dr_b200_rasterize_fwd(const float* pos, const int32_t* tri, int32_t B, int32_t V, int32_t F, int32_t H,
                              int32_t W, float* rast, float* rast_db, void* scratch, void* stream);
/* dL_dpos[B,V,4] is ADDED to (caller zeroes it); gradients flow through u,v only */
int32_t dr_b200_rasterize_bwd(const float* pos, const int32_t* tri, int32_t B, int32_t V, int32_t F, int32_t H,
                              int32_t W, const float* rast, const float* dL_drast, float* dL_dpos, void* stream);

/* attr[attr_B,V,A] with attr_B in {1,B}; rast_db/out_da may be NULL (diff_attrs=None) else all attributes are
 * differentiated: out_da[B,H,W,2A] = (da/dX, da/dY) per attribute */
int32_t dr_b200_interpolate_fwd(const float* attr, int32_t attr_B, const float* rast, const int32_t* tri,
                                const float* rast_db, int32_t B, int32_t V, int32_t F, int32_t H, int32_t W,
                                int32_t A, float* out, float* out_da, void* stream);
/* dL_dattr is ADDED to (caller zeroes); dL_drast[B,H,W,4] and dL_drast_db[B,H,W,4] (may be NULL) are written */
int32_t dr_b200_interpolate_bwd(const float* attr, int32_t attr_B, const float* rast, const int32_t* tri,
                                const float* rast_db, int32_t B, int32_t V, int32_t F, int32_t H, int32_t W,
                                int32_t A, const float* dL_dout, const float* dL_dout_da, float* dL_dattr,
                                float* dL_drast, float* dL_drast_db, void* stream);

/* bilinear texture lookup; tex[tex_B,Ht,Wt,C] (tex_B in {1,B}); uv[B,H,W,2]; boundary 0 = wrap, 1 = clamp */
int32_t dr_b200_texture_fwd(const float* tex, int32_t tex_B, int32_t Ht, int32_t Wt, int32_t C, const float* uv,
                            int32_t B, int32_t H, int32_t W, int32_t boundary, float* out, void* stream);
/* dL_dtex is ADDED to (caller zeroes); dL_duv written */
int32_t dr_b200_texture_bwd(const float* tex, int32_t tex_B, int32_t Ht, int32_t Wt, int32_t C, const float* uv,
                            int32_t B, int32_t H, int32_t W, int32_t boundary, const float* dL_dout,
                            float* dL_dtex, float* dL_duv, void* stream);

/* topology for antialias: opp[F,3] = opposite vertex of the other triangle across edge e (edge e joins vertices
 * e+1,e+2 of the triangle), -1 if none.  scratch: dr_b200_topology_scratch_bytes(F) */
size_t dr_b200_topology_scratch_bytes(int32_t F);
int32_t dr_b200_edge_opposites(const int32_t* tri, int32_t F, int32_t V, int32_t* opp, void* scratch, void* stream);

int32_t dr_b200_antialias_fwd(const float* color, const float* rast, const float* pos, const int32_t* tri,
                              const int32_t* opp, int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, int32_t C,
                              float* out, void* stream);
/* dL_dcolor written; dL_dpos[B,V,4] ADDED to (caller zeroes) */
int32_t dr_b200_antialias_bwd(const float* color, const float* rast, const float* pos, const int32_t* tri,
                              const int32_t* opp, int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, int32_t C,
                              const float* dL_dout, float* dL_dcolor, float* dL_dpos, void* stream);

/* ---- Hunyuan3D's texture-bake rasterizer (the `custom_rasterizer` package; INTEGRATION §3) ----------------------
 * pos[V,4] clip space; tri[F,3]; findices[H,W] int32 = face id + 1 (0 = empty); barycentric[H,W,3], perspective
 * corrected.  Bit-identical to the reference's CPU path (csrc/cr_raster.cu states the arithmetic).  depth_prior[H,W]
 * may be NULL (no prior); with it a pixel is skipped where depth < depth_prior*0.49999 + 0.5 + occlusion_truncation.
 * scratch: dr_b200_cr_scratch_bytes(F, H, W) (an 8 B/pixel z-buffer and two face queues); 0 on bad sizes.
 * H, W <= 2^24 and H*W*3 < 2^31. */
size_t dr_b200_cr_scratch_bytes(int32_t F, int32_t H, int32_t W);
int32_t dr_b200_cr_rasterize(const float* pos, int32_t V, const int32_t* tri, int32_t F, const float* depth_prior,
                             int32_t H, int32_t W, float occlusion_truncation, int32_t* findices, float* barycentric,
                             void* scratch, void* stream);
/* out[npix,C] = ((+0 + b0 col[v0]) + b1 col[v1]) + b2 col[v2] in fp32 (torch's CPU order), for the face findices - 1 + (findices == 0) (torch's
 * wrap of negative indices; a pixel whose face or vertex is out of range gives 0).  findices is int32, or fp32 when
 * findices_f32; tri is int32, or int64 when tri_i64; col[V,C]. */
int32_t dr_b200_cr_interpolate_fwd(const float* col, int32_t V, int32_t C, const void* findices, int32_t findices_f32,
                                   const float* barycentric, const void* tri, int32_t tri_i64, int32_t F,
                                   int32_t npix, float* out, void* stream);
/* grad_barycentric[npix,3] (may be NULL) = sum over c in ascending order of grad_out * col[v_k];
 * contrib[3*npix,C] = b_k * grad_out and contrib_index[3*npix] = v_k (both NULL or neither): the rows a deterministic
 * scatter sum (gs_b200_scatter_*) folds into the col gradient.  No atomics. */
int32_t dr_b200_cr_interpolate_bwd(const float* col, int32_t V, int32_t C, const void* findices, int32_t findices_f32,
                                   const float* barycentric, const void* tri, int32_t tri_i64, int32_t F,
                                   int32_t npix, const float* grad_out, float* grad_barycentric, float* contrib,
                                   int64_t* contrib_index, void* stream);

/* ---- StableFast3D's UV texture baker (slangtorch's texture_baker.slang: bake_uv, interpolate; INTEGRATION §3) ------
 * Bit-identical to the reference's own kernels (csrc/uv_bake.cu states the arithmetic).  uv[V,2] fp32 (8-byte
 * aligned), faces[F,3] int32, square textures of res x res texels, res <= 2^15.  Only the launched region, texel rows
 * [0, rows) and columns [0, cols) (clipped to res), is written; the rest of out keeps what it held.
 * rasterize: out[res,res,4] (16-byte aligned) = (u, v, w, face) of the lowest-index face whose barycentric test
 * accepts the texel, or (0, 0, 0, -1).  A face with a vertex id out of range is skipped.
 * scratch: dr_b200_uvbake_scratch_bytes(F, res) = 256 + 4 res^2 + 8 F bytes; 0 on bad sizes.  After a call its first
 * three uint32 hold the warp-queue, CTA-queue and whole-texture face counts (whole-texture faces are in the CTA queue).
 * interpolate: out[res,res,3] = the rast-weighted attr[V,3] of face (int)rast.w, 0 where that id is negative or any
 * face or vertex id is out of range; rast[res,res,4] 16-byte aligned. */
size_t dr_b200_uvbake_scratch_bytes(int32_t F, int32_t res);
int32_t dr_b200_uvbake_rasterize(const float* uv, int32_t V, const int32_t* faces, int32_t F, float* out, int32_t res,
                                 int32_t rows, int32_t cols, void* scratch, void* stream);
int32_t dr_b200_uvbake_interpolate(const float* attr, int32_t V, const int32_t* faces, int32_t F, const float* rast,
                                   float* out, int32_t res, int32_t rows, int32_t cols, void* stream);
#ifdef __cplusplus
}
#endif
#endif
