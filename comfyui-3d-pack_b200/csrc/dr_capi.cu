// C ABI of the mesh ops (include/dr_b200.h) — thin validation + launch layer.
#include "../../include/dr_b200.h"
#include "gs_common.cuh"

size_t dr_rasterize_scratch_bytes(int B, int F, int H, int W);
int dr_launch_rasterize_fwd(const float*, const int32_t*, int, int, int, int, int, float*, float*, void*, cudaStream_t);
int dr_launch_rasterize_bwd(const float*, const int32_t*, int, int, int, int, int, const float*, const float*, float*, cudaStream_t);
int dr_launch_interpolate_fwd(const float*, int, const float*, const int32_t*, const float*, int, int, int, int, int, int, float*, float*, cudaStream_t);
int dr_launch_interpolate_bwd(const float*, int, const float*, const int32_t*, const float*, int, int, int, int, int, int, const float*, const float*, float*, float*, float*, cudaStream_t);
int dr_launch_texture_fwd(const float*, int, int, int, int, const float*, int, int, int, int, float*, cudaStream_t);
int dr_launch_texture_bwd(const float*, int, int, int, int, const float*, int, int, int, int, const float*, float*, float*, cudaStream_t);
size_t dr_topology_scratch_bytes(int F);
int dr_launch_edge_opposites(const int32_t*, int, int, int32_t*, void*, cudaStream_t);
int dr_launch_antialias_fwd(const float*, const float*, const float*, const int32_t*, const int32_t*, int, int, int, int, int, int, float*, cudaStream_t);
int dr_launch_antialias_bwd(const float*, const float*, const float*, const int32_t*, const int32_t*, int, int, int, int, int, int, const float*, float*, float*, cudaStream_t);
size_t cr_scratch_bytes(int F, int H, int W);
int cr_launch_rasterize(const float*, int, const int32_t*, int, const float*, int, int, float, int32_t*, float*, void*, cudaStream_t);
int cr_launch_interpolate(const float*, int, int, const void*, int, const float*, const void*, int, int, int, const float*, float*,
                          float*, float*, long long*, cudaStream_t);
size_t ub_scratch_bytes(int F, int res);
int ub_launch_rasterize(const float*, int, const int32_t*, int, float*, int, int, int, void*, cudaStream_t);
int ub_launch_interpolate(const float*, int, const int32_t*, int, const float*, float*, int, int, int, cudaStream_t);

#define DR_REQ(cond, msg) do { if (!(cond)) { gs_set_error("%s: %s", __func__, msg); return 1; } } while (0)

extern "C" {

size_t dr_b200_rasterize_scratch_bytes(int32_t B, int32_t F, int32_t H, int32_t W) { return dr_rasterize_scratch_bytes(B, F, H, W); }

int32_t dr_b200_rasterize_fwd(const float* pos, const int32_t* tri, int32_t B, int32_t V, int32_t F, int32_t H, int32_t W,
                              float* rast, float* rast_db, void* scratch, void* stream) {
    DR_REQ(B >= 0 && V >= 0 && F >= 0 && H > 0 && W > 0, "bad sizes");
    DR_REQ(rast && rast_db && scratch && (F == 0 || (pos && tri)), "NULL pointer");
    DR_REQ(((size_t)pos & 15) == 0 && ((size_t)rast & 15) == 0 && ((size_t)rast_db & 15) == 0, "pos/rast must be 16-byte aligned");
    return dr_launch_rasterize_fwd(pos, tri, B, V, F, H, W, rast, rast_db, scratch, (cudaStream_t)stream);
}
int32_t dr_b200_rasterize_bwd(const float* pos, const int32_t* tri, int32_t B, int32_t V, int32_t F, int32_t H, int32_t W,
                              const float* rast, const float* dL_drast, float* dL_dpos, void* stream) {
    DR_REQ(pos && tri && rast && dL_drast && dL_dpos, "NULL pointer");
    return dr_launch_rasterize_bwd(pos, tri, B, V, F, H, W, rast, dL_drast, dL_dpos, (cudaStream_t)stream);
}
int32_t dr_b200_interpolate_fwd(const float* attr, int32_t attr_B, const float* rast, const int32_t* tri, const float* rast_db,
                                int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, int32_t A, float* out, float* out_da,
                                void* stream) {
    DR_REQ(attr && rast && tri && out, "NULL pointer");
    DR_REQ(attr_B == 1 || attr_B == B, "attr batch must be 1 or B");
    DR_REQ((out_da == nullptr) || (rast_db != nullptr), "out_da needs rast_db");
    return dr_launch_interpolate_fwd(attr, attr_B, rast, tri, rast_db, B, V, F, H, W, A, out, out_da, (cudaStream_t)stream);
}
int32_t dr_b200_interpolate_bwd(const float* attr, int32_t attr_B, const float* rast, const int32_t* tri, const float* rast_db,
                                int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, int32_t A, const float* dL_dout,
                                const float* dL_dout_da, float* dL_dattr, float* dL_drast, float* dL_drast_db, void* stream) {
    DR_REQ(attr && rast && tri && dL_dout && dL_dattr && dL_drast, "NULL pointer");
    DR_REQ((dL_dout_da == nullptr) || (rast_db != nullptr), "dL_dout_da needs rast_db");
    return dr_launch_interpolate_bwd(attr, attr_B, rast, tri, rast_db, B, V, F, H, W, A, dL_dout, dL_dout_da, dL_dattr, dL_drast,
                                     dL_drast_db, (cudaStream_t)stream);
}
int32_t dr_b200_texture_fwd(const float* tex, int32_t tex_B, int32_t Ht, int32_t Wt, int32_t C, const float* uv, int32_t B,
                            int32_t H, int32_t W, int32_t boundary, float* out, void* stream) {
    DR_REQ(tex && uv && out && Ht > 0 && Wt > 0 && C > 0, "bad argument");
    DR_REQ(tex_B == 1 || tex_B == B, "tex batch must be 1 or B");
    return dr_launch_texture_fwd(tex, tex_B, Ht, Wt, C, uv, B, H, W, boundary, out, (cudaStream_t)stream);
}
int32_t dr_b200_texture_bwd(const float* tex, int32_t tex_B, int32_t Ht, int32_t Wt, int32_t C, const float* uv, int32_t B,
                            int32_t H, int32_t W, int32_t boundary, const float* dL_dout, float* dL_dtex, float* dL_duv,
                            void* stream) {
    DR_REQ(tex && uv && dL_dout && dL_dtex && dL_duv, "NULL pointer");
    return dr_launch_texture_bwd(tex, tex_B, Ht, Wt, C, uv, B, H, W, boundary, dL_dout, dL_dtex, dL_duv, (cudaStream_t)stream);
}
size_t dr_b200_topology_scratch_bytes(int32_t F) { return dr_topology_scratch_bytes(F); }
int32_t dr_b200_edge_opposites(const int32_t* tri, int32_t F, int32_t V, int32_t* opp, void* scratch, void* stream) {
    DR_REQ(F == 0 || (tri && opp && scratch), "NULL pointer");
    return dr_launch_edge_opposites(tri, F, V, opp, scratch, (cudaStream_t)stream);
}
int32_t dr_b200_antialias_fwd(const float* color, const float* rast, const float* pos, const int32_t* tri, const int32_t* opp,
                              int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, int32_t C, float* out, void* stream) {
    DR_REQ(color && rast && out && (F == 0 || (pos && tri && opp)), "NULL pointer");
    return dr_launch_antialias_fwd(color, rast, pos, tri, opp, B, V, F, H, W, C, out, (cudaStream_t)stream);
}
int32_t dr_b200_antialias_bwd(const float* color, const float* rast, const float* pos, const int32_t* tri, const int32_t* opp,
                              int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, int32_t C, const float* dL_dout,
                              float* dL_dcolor, float* dL_dpos, void* stream) {
    DR_REQ(color && rast && dL_dout && dL_dcolor && (F == 0 || (pos && tri && opp && dL_dpos)), "NULL pointer");
    return dr_launch_antialias_bwd(color, rast, pos, tri, opp, B, V, F, H, W, C, dL_dout, dL_dcolor, dL_dpos, (cudaStream_t)stream);
}

size_t dr_b200_cr_scratch_bytes(int32_t F, int32_t H, int32_t W) {
    return (F < 0 || H <= 0 || W <= 0) ? 0 : cr_scratch_bytes(F, H, W);
}
int32_t dr_b200_cr_rasterize(const float* pos, int32_t V, const int32_t* tri, int32_t F, const float* depth_prior, int32_t H,
                             int32_t W, float occlusion_truncation, int32_t* findices, float* barycentric, void* scratch,
                             void* stream) {
    DR_REQ(V >= 0 && F >= 0 && H > 0 && W > 0, "bad sizes");
    DR_REQ(H <= (1 << 24) && W <= (1 << 24) && (int64_t)H * W <= INT32_MAX / 3, "image too large");
    DR_REQ(findices && barycentric && scratch && (F == 0 || (pos && tri)), "NULL pointer");
    DR_REQ(((size_t)pos & 15) == 0, "pos must be 16-byte aligned");
    return cr_launch_rasterize(pos, V, tri, F, depth_prior, H, W, occlusion_truncation, findices, barycentric, scratch,
                               (cudaStream_t)stream);
}
int32_t dr_b200_cr_interpolate_fwd(const float* col, int32_t V, int32_t C, const void* findices, int32_t findices_f32,
                                   const float* barycentric, const void* tri, int32_t tri_i64, int32_t F, int32_t npix,
                                   float* out, void* stream) {
    DR_REQ(V >= 0 && C > 0 && F >= 0 && npix >= 0 && (int64_t)npix * 3 <= INT32_MAX, "bad sizes");
    DR_REQ(npix == 0 || (findices && barycentric && out && (F == 0 || tri) && (V == 0 || col)), "NULL pointer");
    return cr_launch_interpolate(col, V, C, findices, findices_f32, barycentric, tri, tri_i64, F, npix, nullptr, out, nullptr,
                                 nullptr, nullptr, (cudaStream_t)stream);
}
int32_t dr_b200_cr_interpolate_bwd(const float* col, int32_t V, int32_t C, const void* findices, int32_t findices_f32,
                                   const float* barycentric, const void* tri, int32_t tri_i64, int32_t F, int32_t npix,
                                   const float* grad_out, float* grad_barycentric, float* contrib, int64_t* contrib_index,
                                   void* stream) {
    DR_REQ(V >= 0 && C > 0 && F >= 0 && npix >= 0 && (int64_t)npix * 3 <= INT32_MAX, "bad sizes");
    DR_REQ(npix == 0 || (findices && barycentric && grad_out && (F == 0 || tri) && (V == 0 || col)), "NULL pointer");
    DR_REQ((contrib == nullptr) == (contrib_index == nullptr), "contrib and contrib_index go together");
    return cr_launch_interpolate(col, V, C, findices, findices_f32, barycentric, tri, tri_i64, F, npix, grad_out, nullptr,
                                 grad_barycentric, contrib, (long long*)contrib_index, (cudaStream_t)stream);
}

size_t dr_b200_uvbake_scratch_bytes(int32_t F, int32_t res) {
    return (F < 0 || res <= 0 || res > (1 << 15)) ? 0 : ub_scratch_bytes(F, res);
}
int32_t dr_b200_uvbake_rasterize(const float* uv, int32_t V, const int32_t* faces, int32_t F, float* out, int32_t res,
                                 int32_t rows, int32_t cols, void* scratch, void* stream) {
    DR_REQ(V >= 0 && F >= 0 && res > 0 && res <= (1 << 15) && rows >= 0 && cols >= 0, "bad sizes");
    DR_REQ(out && scratch && (F == 0 || (uv && faces)), "NULL pointer");
    DR_REQ(((size_t)uv & 7) == 0 && ((size_t)out & 15) == 0, "uv must be 8-byte and out 16-byte aligned");
    return ub_launch_rasterize(uv, V, faces, F, out, res, rows < res ? rows : res, cols < res ? cols : res, scratch,
                               (cudaStream_t)stream);
}
int32_t dr_b200_uvbake_interpolate(const float* attr, int32_t V, const int32_t* faces, int32_t F, const float* rast,
                                   float* out, int32_t res, int32_t rows, int32_t cols, void* stream) {
    DR_REQ(V >= 0 && F >= 0 && res > 0 && res <= (1 << 15) && rows >= 0 && cols >= 0, "bad sizes");
    DR_REQ(rast && out && (F == 0 || faces) && (V == 0 || attr), "NULL pointer");
    DR_REQ(((size_t)rast & 15) == 0, "rast must be 16-byte aligned");
    return ub_launch_interpolate(attr, V, faces, F, rast, out, res, rows < res ? rows : res, cols < res ? cols : res,
                                 (cudaStream_t)stream);
}
}
