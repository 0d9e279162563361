/* gs_b200_pts.h: pytorch3d's point rasterizer and TriplaneGaussian's points_projection (pts_raster.cu), sm_90a.
 * Argument errors are reported through gs_b200_last_error() (gs_b200.h).  Plain pointers, extern "C", no torch types. */
#ifndef GS_B200_PTS_H
#define GS_B200_PTS_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- pytorch3d's point rasterizer (PointsRasterizer over cameras_from_opencv_projection) and TriplaneGaussian's
 * points_projection -------------------------------------------------------------------------------------------------
 * N clouds, P packed points [P, 3] fp32; cloud n holds points first[n] .. first[n+1]-1 (first int64 [N+1] on the
 * device), or P / N points each when first is NULL.  Cameras (ncam = 1 or N; cloud n uses camera n, or camera 0):
 * R [ncam,3,3], T [ncam,3] (OpenCV world-to-camera), camera_matrix [ncam,3,3] (fx = [0][0], fy = [1][1],
 * cx = [0][2], cy = [1][2], in pixels), image_hw [ncam,2] = (h, w) as floats, or NULL for (H, W).  All fp32, contiguous.
 * Projection, fp32, one rounding per operation (no FMA contraction), row i of R as (ri0, ri1, ri2):
 *   c_i = ((ri0*x + ri1*y) + ri2*z) + T_i;   s = fminf(h, w) * 0.5;   u = (fx*c_0)/c_2 + cx;   v = (fy*c_1)/c_2 + cy
 *   x_ndc = (w*0.5 - u) / s,  y_ndc = (h*0.5 - v) / s,  z = c_2
 * so +X points left, +Y up, the shorter image side spans [-1, 1] and the longer [-w/h, w/h] (or [-h/w, h/w]).
 * A point is drawn only when z > 0 and x_ndc, y_ndc are finite: z = 0 (and NaN) never is.
 * Pixel (y, x) of the H x W image (row 0 at the top) has pytorch3d's non-square NDC centre
 *   (pix(W-1-x, W, H), pix(H-1-y, H, W)),  pix(i, S1, S2) = -o + (range*i + o)/S1,  range = S1 > S2 ? (S1*2)/S2 : 2,
 *   o = range/2 (fp32).  A point covers the pixel iff dx*dx + dy*dy < radius*radius (fp32, strict; dx = centre - x_ndc).
 * Each pixel keeps its K (1..GS_B200_PTS_MAX_K) covering points of its own cloud with the smallest (z, packed index),
 * ascending: idx int32 [N,H,W,K] (packed index, -1 where empty), zbuf fp32 (z, -1), dists fp32 (dx*dx + dy*dy, -1);
 * zbuf and dists may be NULL.  scratch: gs_b200_pts_scratch_bytes(N, P, H, W, K) (0 = invalid arguments).
 * Lift: with that idx, point p's winner is the largest linear index e = ((n*H + y)*W + x)*K + k with idx[e] = p
 *   (-1 when none) -> winner int32 [P]; out [P, C] fp32 = features[n, :, y, x] of the winner, 0 without one.
 *   features [N, C, H, W] fp32 is read in place through feature_strides_host (4 element strides in host memory).
 * Lift backward: grad_features [N, C, H, W] (contiguous) = for each pixel, +0 plus grad_out[p, c] over its slots k
 *   (ascending) whose point p it won.  No atomics on values, no host read: the same bits on every run.
 * N*H*W*K and P below 2^31. */
#define GS_B200_PTS_MAX_K 8
size_t gs_b200_pts_scratch_bytes(int32_t N, int64_t P, int32_t H, int32_t W, int32_t K);
int32_t gs_b200_pts_rasterize(int32_t N, int64_t P, int32_t H, int32_t W, int32_t K, float radius, int32_t ncam,
                              const float* points, const int64_t* first, const float* R, const float* T,
                              const float* camera_matrix, const float* image_hw, int32_t* idx, float* zbuf,
                              float* dists, void* scratch, void* stream);
int32_t gs_b200_pts_lift(int32_t N, int64_t P, int32_t H, int32_t W, int32_t K, int32_t C, const int32_t* idx,
                         const float* features, const int64_t* feature_strides_host, int32_t* winner, float* out,
                         void* stream);
int32_t gs_b200_pts_lift_backward(int32_t N, int64_t P, int32_t H, int32_t W, int32_t K, int32_t C, const int32_t* idx,
                                  const int32_t* winner, const float* grad_out, float* grad_features, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GS_B200_PTS_H */
