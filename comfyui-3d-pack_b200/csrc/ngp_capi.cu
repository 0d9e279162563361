// C ABI of the Instant-NGP path (include/ngp_b200.h) — validation + launch layer.
#include "../../include/ngp_b200.h"
#include "gs_common.cuh"

int ngp_grid_encode_fwd(const float*, long long, const float*, const int32_t*, int, float, double, int, float*, cudaStream_t);
int ngp_grid_encode_bwd(const float*, long long, const int32_t*, int, float, double, int, const float*, float*, cudaStream_t);
int ngp_grid_tv(const float*, long long, const float*, const int32_t*, int, float, double, int, float, float*, cudaStream_t);
size_t ngp_march_scratch_bytes(long long, int);
int ngp_march_count(const float*, const float*, long long, const uint8_t*, int, const float*, float, float, float, const float*,
                    uint32_t*, uint32_t*, unsigned long long*, void*, cudaStream_t);
int ngp_march_write(const float*, const float*, long long, int, const float*, float, float, float, const float*, const uint32_t*,
                    long long*, float*, float*, void*, cudaStream_t);
int ngp_ray_ranges(const long long*, long long, long long, int32_t*, cudaStream_t);
int ngp_weights_fwd(const float*, const float*, const float*, const int32_t*, long long, float*, float*, float*, cudaStream_t);
int ngp_weights_bwd(const float*, const float*, const int32_t*, long long, const float*, const float*, const float*, const float*,
                    const float*, float*, cudaStream_t);
int ngp_accumulate_fwd(const float*, const float*, int, const int32_t*, long long, float*, cudaStream_t);
int ngp_accumulate_bwd(const float*, const float*, int, const long long*, long long, const float*, float*, float*, cudaStream_t);

int ngp_mlp2_supported(int, int, int);
int ngp_mlp2_fwd(const float*, long long, int, int, int, const float*, const float*, float*, cudaStream_t);
int ngp_mlp2_bwd(const float*, long long, int, int, int, const float*, const float*, const float*, float*, float*, float*, cudaStream_t);

#define NGP_REQ(cond, msg) do { if (!(cond)) { gs_set_error("%s: %s", __func__, msg); return 1; } } while (0)

extern "C" {
int32_t ngp_b200_grid_encode_fwd(const float* x, int64_t N, const float* emb, const int32_t* offsets, int32_t L, float bound,
                                 double pls, int32_t base, float* out, void* stream) {
    NGP_REQ(N == 0 || (x && emb && offsets && out), "NULL pointer");
    NGP_REQ(((size_t)emb & 7) == 0 && ((size_t)out & 7) == 0, "emb/out must be 8-byte aligned");
    return ngp_grid_encode_fwd(x, N, emb, offsets, L, bound, pls, base, out, (cudaStream_t)stream);
}
int32_t ngp_b200_grid_encode_bwd(const float* x, int64_t N, const int32_t* offsets, int32_t L, float bound, double pls,
                                 int32_t base, const float* g, float* d_emb, void* stream) {
    NGP_REQ(N == 0 || (x && offsets && g && d_emb), "NULL pointer");
    return ngp_grid_encode_bwd(x, N, offsets, L, bound, pls, base, g, d_emb, (cudaStream_t)stream);
}
int32_t ngp_b200_grid_tv_grad(const float* x, int64_t N, const float* emb, const int32_t* offsets, int32_t L, float bound,
                              double pls, int32_t base, float weight, float* d_emb, void* stream) {
    NGP_REQ(N == 0 || (x && emb && offsets && d_emb), "NULL pointer");
    return ngp_grid_tv(x, N, emb, offsets, L, bound, pls, base, weight, d_emb, (cudaStream_t)stream);
}
size_t ngp_b200_march_scratch_bytes(int64_t n_rays, int32_t R) { return ngp_march_scratch_bytes(n_rays, R); }
int32_t ngp_b200_march_count(const float* ro, const float* rd, int64_t n, const uint8_t* binary, int32_t R, const float* aabb,
                             float near_plane, float far_plane, float dt, const float* t_offset, uint32_t* counts,
                             uint32_t* offsets, unsigned long long* total_dev, void* scratch, void* stream) {
    NGP_REQ(binary && aabb && counts && offsets && total_dev && scratch && (n == 0 || (ro && rd)), "NULL pointer");
    NGP_REQ(dt > 0.f && R > 0, "bad step / resolution");
    return ngp_march_count(ro, rd, n, binary, R, aabb, near_plane, far_plane, dt, t_offset, counts, offsets, total_dev, scratch,
                           (cudaStream_t)stream);
}
int32_t ngp_b200_march_write(const float* ro, const float* rd, int64_t n, int32_t R, const float* aabb, float near_plane,
                             float far_plane, float dt, const float* t_offset, const uint32_t* offsets, int64_t* ray_indices,
                             float* t_starts, float* t_ends, void* scratch, void* stream) {
    NGP_REQ(aabb && offsets && scratch && (n == 0 || (ro && rd)), "NULL pointer");
    return ngp_march_write(ro, rd, n, R, aabb, near_plane, far_plane, dt, t_offset, offsets, (long long*)ray_indices, t_starts,
                           t_ends, scratch, (cudaStream_t)stream);
}
int32_t ngp_b200_ray_ranges(const int64_t* ri, int64_t S, int64_t n_rays, int32_t* ranges, void* stream) {
    NGP_REQ(ranges && (S == 0 || ri), "NULL pointer");
    return ngp_ray_ranges((const long long*)ri, S, n_rays, ranges, (cudaStream_t)stream);
}
int32_t ngp_b200_weights_fwd(const float* ts, const float* te, const float* sig, const int32_t* ranges, int64_t n_rays, float* w,
                             float* tr, float* al, void* stream) {
    NGP_REQ(ranges, "NULL ranges");
    return ngp_weights_fwd(ts, te, sig, ranges, n_rays, w, tr, al, (cudaStream_t)stream);
}
int32_t ngp_b200_weights_bwd(const float* ts, const float* te, const float* sig, const int32_t* ranges, int64_t n_rays,
                             const float* tr, const float* al, const float* gw, const float* gt, const float* ga, float* dsig,
                             void* stream) {
    (void)sig;
    NGP_REQ(ranges, "NULL ranges");
    return ngp_weights_bwd(ts, te, ranges, n_rays, tr, al, gw, gt, ga, dsig, (cudaStream_t)stream);
}
int32_t ngp_b200_accumulate_fwd(const float* w, const float* v, int32_t C, const int32_t* ranges, int64_t n_rays, float* out,
                                void* stream) {
    NGP_REQ(ranges && out, "NULL pointer");
    return ngp_accumulate_fwd(w, v, C, ranges, n_rays, out, (cudaStream_t)stream);
}
int32_t ngp_b200_accumulate_bwd(const float* w, const float* v, int32_t C, const int64_t* ri, int64_t S, const float* g_out,
                                float* dw, float* dv, void* stream) {
    NGP_REQ(S == 0 || (w && ri && g_out && dw), "NULL pointer");
    return ngp_accumulate_bwd(w, v, C, (const long long*)ri, S, g_out, dw, dv, (cudaStream_t)stream);
}
int32_t ngp_b200_mlp2_supported(int32_t Din, int32_t H, int32_t Dout) { return ngp_mlp2_supported(Din, H, Dout); }
int32_t ngp_b200_mlp2_fwd(const float* X, int64_t N, int32_t Din, int32_t H, int32_t Dout, const float* W1, const float* W2,
                          float* Y, void* stream) {
    NGP_REQ(N == 0 || (X && W1 && W2 && Y), "NULL pointer");
    NGP_REQ(((size_t)X & 15) == 0, "X must be 16-byte aligned");
    return ngp_mlp2_fwd(X, N, Din, H, Dout, W1, W2, Y, (cudaStream_t)stream);
}
int32_t ngp_b200_mlp2_bwd(const float* X, int64_t N, int32_t Din, int32_t H, int32_t Dout, const float* W1, const float* W2,
                          const float* GY, float* GX, float* GW1, float* GW2, void* stream) {
    NGP_REQ(N == 0 || (X && W1 && W2 && GY && GW1 && GW2), "NULL pointer");
    NGP_REQ(((size_t)X & 15) == 0 && ((size_t)GX & 15) == 0, "X/GX must be 16-byte aligned");
    return ngp_mlp2_bwd(X, N, Din, H, Dout, W1, W2, GY, GX, GW1, GW2, (cudaStream_t)stream);
}
}
