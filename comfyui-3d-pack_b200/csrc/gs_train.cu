// Optimisation-step kernels either side of the rasterizer (SURVEY §8f rank 1-2, rows a6/a8/a9):
//   activate_kernel      raw parameters -> what the rasterizer boundary receives
//                        (exp / sigmoid / normalize, main_3DGS_renderer.py:293-321)
//   adam_fused_kernel    chain rule through the activations + torch.optim.Adam(eps=1e-15) update
//                        (training_setup, main_3DGS_renderer.py:435-453) over the PACKED 11+3M-float layout
//                        means3D | shs | opacities | scales | rotations in one pass:
//                        reads grad, param, m, v once and writes param, m, v once (28 B per float).
//   densify_stats_kernel add_densification_stats + max_radii2D update (main_3DGS_renderer.py:767-769,
//                        main_3DGS.py:210-213) fused.
// All three are pure streaming kernels (HBM bound).
#include "../../include/gs_b200.h"
#include "gs_common.cuh"

namespace {

__global__ void __launch_bounds__(256)
activate_kernel(int N, const float* __restrict__ raw_opac, const float* __restrict__ raw_scales,
                const float* __restrict__ raw_rots, float* __restrict__ opac, float* __restrict__ scales,
                float* __restrict__ rots) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    opac[i] = 1.0f / (1.0f + expf(-raw_opac[i]));
#pragma unroll
    for (int k = 0; k < 3; k++) scales[3 * i + k] = expf(raw_scales[3 * i + k]);
    const float r0 = raw_rots[4 * i], r1 = raw_rots[4 * i + 1], r2 = raw_rots[4 * i + 2], r3 = raw_rots[4 * i + 3];
    const float inv = 1.0f / fmaxf(sqrtf(r0 * r0 + r1 * r1 + r2 * r2 + r3 * r3), 1e-12f);     // F.normalize eps
    rots[4 * i] = r0 * inv; rots[4 * i + 1] = r1 * inv; rots[4 * i + 2] = r2 * inv; rots[4 * i + 3] = r3 * inv;
}

struct AdamArgs {
    // per-group step sizes lr / (1 - b1^t); 1 - b and the bias corrections are taken in double on the host and
    // rounded once, as torch.optim.Adam does with its Python-float hyperparameters
    float st_xyz, st_dc, st_rest, st_opac, st_scale, st_rot;
    float beta1, beta2, one_m_beta1, one_m_beta2, eps, bias2_sqrt;     // bias2_sqrt = sqrt(1 - b2^t)
    float grad_scale;                               // multiplies the incoming (summed) gradient, e.g. 1/world
};

__device__ __forceinline__ void adam_one(float& p, float& m, float& v, float g, float step_size, const AdamArgs& a) {
    m = a.beta1 * m + a.one_m_beta1 * g;
    v = a.beta2 * v + a.one_m_beta2 * g * g;
    const float denom = sqrtf(v) / a.bias2_sqrt + a.eps;
    p -= step_size * (m / denom);
}

// one thread per Gaussian; grads are wrt the ACTIVATED opac/scales/rots (what the rasterizer returns)
__global__ void __launch_bounds__(256)
adam_fused_kernel(int N, int M, AdamArgs a, const float* __restrict__ g_means,
                  const float* __restrict__ g_opac, const float* __restrict__ g_scales, const float* __restrict__ g_rots,
                  float* __restrict__ p_means, float* __restrict__ p_opac,
                  float* __restrict__ p_scales, float* __restrict__ p_rots, float* __restrict__ m1, float* __restrict__ m2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const size_t n = (size_t)N;
    // offsets of the groups inside the packed moment buffers (same layout as the parameters)
    const size_t o_sh = 3 * n, o_op = o_sh + 3 * (size_t)M * n, o_sc = o_op + n, o_ro = o_sc + 3 * n;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const size_t j = 3 * (size_t)i + k;
        adam_one(p_means[j], m1[j], m2[j], a.grad_scale * g_means[j], a.st_xyz, a);
    }
    {
        const float o = 1.0f / (1.0f + expf(-p_opac[i]));
        const float g = a.grad_scale * g_opac[i] * o * (1.f - o);
        adam_one(p_opac[i], m1[o_op + i], m2[o_op + i], g, a.st_opac, a);
    }
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const size_t j = 3 * (size_t)i + k;
        const float g = a.grad_scale * g_scales[j] * expf(p_scales[j]);
        adam_one(p_scales[j], m1[o_sc + j], m2[o_sc + j], g, a.st_scale, a);
    }
    {
        float r[4], g[4];
#pragma unroll
        for (int k = 0; k < 4; k++) { r[k] = p_rots[4 * (size_t)i + k]; g[k] = a.grad_scale * g_rots[4 * (size_t)i + k]; }
        // F.normalize divides by clamp_min(|r|, 1e-12): below the clamp no gradient flows through the norm, so the
        // projection term goes and the gradient is g / 1e-12
        const float nrm = sqrtf(r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3]);
        const float inv = 1.0f / fmaxf(nrm, 1e-12f);
        const float dot = nrm < 1e-12f ? 0.f : (r[0] * g[0] + r[1] * g[1] + r[2] * g[2] + r[3] * g[3]) * inv * inv;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const size_t j = 4 * (size_t)i + k;
            adam_one(p_rots[j], m1[o_ro + j], m2[o_ro + j], (g[k] - r[k] * dot) * inv, a.st_rot, a);
        }
    }
}

// SH coefficients (81 % of the bytes at degree 3): purely elementwise, so a flat 128-bit pass over [N * 3M].
// Coefficient 0 (first 3 floats of each row) uses the dc learning rate, the rest lr_rest.  (A thread-per-Gaussian
// walk over its 3M-float row touches 32 different cache lines per warp load and ran at 0.3 TB/s.)
__global__ void __launch_bounds__(256)
adam_sh_kernel(size_t n4, int row, AdamArgs a, const float4* __restrict__ g, float4* __restrict__ p, float4* __restrict__ m1,
               float4* __restrict__ m2) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const int c0 = (int)((i * 4) % (size_t)row);
    float4 pv = p[i], mv = m1[i], vv = m2[i];
    const float4 gv = g[i];
    // a float4 may straddle a row boundary when row = 3M is not a multiple of 4 (sh_degree 0 and 2): the wrapped
    // elements are the NEXT Gaussian's dc coefficients
    auto st_of = [&](int k) { int c = c0 + k; if (c >= row) c -= row; return c < 3 ? a.st_dc : a.st_rest; };
    adam_one(pv.x, mv.x, vv.x, a.grad_scale * gv.x, st_of(0), a);
    adam_one(pv.y, mv.y, vv.y, a.grad_scale * gv.y, st_of(1), a);
    adam_one(pv.z, mv.z, vv.z, a.grad_scale * gv.z, st_of(2), a);
    adam_one(pv.w, mv.w, vv.w, a.grad_scale * gv.w, st_of(3), a);
    p[i] = pv; m1[i] = mv; m2[i] = vv;
}

// scalar tail / unaligned fallback of the SH pass
__global__ void __launch_bounds__(256)
adam_sh_scalar_kernel(size_t first, size_t n, int row, AdamArgs a, const float* __restrict__ g, float* __restrict__ p,
                      float* __restrict__ m1, float* __restrict__ m2) {
    const size_t j = first + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    adam_one(p[j], m1[j], m2[j], a.grad_scale * g[j], (int)(j % (size_t)row) < 3 ? a.st_dc : a.st_rest, a);
}

__global__ void __launch_bounds__(256)
densify_stats_kernel(int N, const float* __restrict__ g_means2D, const int32_t* __restrict__ radii,
                     float* __restrict__ grad_accum, float* __restrict__ denom, float* __restrict__ max_radii) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int r = radii[i];
    if (r <= 0) return;
    const float gx = g_means2D[3 * (size_t)i], gy = g_means2D[3 * (size_t)i + 1];
    // the norm in double: the squares neither overflow (|g| > 1.8e19) nor flush to zero (|g| < 1e-23)
    grad_accum[i] += (float)sqrt((double)gx * gx + (double)gy * gy);
    denom[i] += 1.0f;
    max_radii[i] = fmaxf(max_radii[i], (float)r);
}

}  // namespace

extern "C" {

int32_t gs_b200_activate(int32_t N, const float* raw_opac, const float* raw_scales, const float* raw_rots, float* opac,
                         float* scales, float* rots, void* stream) {
    if (N > 0 && (!raw_opac || !raw_scales || !raw_rots || !opac || !scales || !rots)) { gs_set_error("activate: NULL"); return 1; }
    const cudaStream_t s = (cudaStream_t)stream;
    if (N <= 0) return 0;
    activate_kernel<<<(N + 255) / 256, 256, 0, s>>>(N, raw_opac, raw_scales, raw_rots, opac, scales, rots);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int32_t gs_b200_adam_step(int32_t N, int32_t M, const float* lrs6, double beta1, double beta2, float eps, int32_t step,
                          float grad_scale, const float* grads_packed, float* params_packed, float* m1, float* m2,
                          void* stream) {
    if (!lrs6 || step < 1 || (N > 0 && (!grads_packed || !params_packed || !m1 || !m2))) { gs_set_error("adam_step: bad argument"); return 1; }
    const cudaStream_t s = (cudaStream_t)stream;
    if (N <= 0) return 0;
    AdamArgs a;
    const double bias1 = 1.0 - pow(beta1, (double)step);
    a.st_xyz = (float)(lrs6[0] / bias1); a.st_dc = (float)(lrs6[1] / bias1); a.st_rest = (float)(lrs6[2] / bias1);
    a.st_opac = (float)(lrs6[3] / bias1); a.st_scale = (float)(lrs6[4] / bias1); a.st_rot = (float)(lrs6[5] / bias1);
    a.beta1 = (float)beta1; a.beta2 = (float)beta2; a.one_m_beta1 = (float)(1.0 - beta1); a.one_m_beta2 = (float)(1.0 - beta2);
    a.eps = eps; a.bias2_sqrt = (float)sqrt(1.0 - pow(beta2, (double)step));
    a.grad_scale = grad_scale;
    const size_t n = (size_t)N;
    const float* g = grads_packed; float* p = params_packed;
    const size_t o_sh = 3 * n, o_op = o_sh + 3 * (size_t)M * n, o_sc = o_op + n, o_ro = o_sc + 3 * n;
    adam_fused_kernel<<<(N + 255) / 256, 256, 0, s>>>(N, M, a, g, g + o_op, g + o_sc, g + o_ro, p, p + o_op, p + o_sc, p + o_ro,
                                                      m1, m2);
    // SH block: 128-bit path when every base pointer of the block is 16-byte aligned (o_sh = 3N floats)
    const size_t n_sh = 3 * (size_t)M * n;
    const int row = 3 * M;
    const bool aligned = (((uintptr_t)(g + o_sh) | (uintptr_t)(p + o_sh) | (uintptr_t)(m1 + o_sh) | (uintptr_t)(m2 + o_sh)) & 15) == 0;
    const size_t n4 = aligned ? n_sh / 4 : 0;
    if (n4) adam_sh_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, s>>>(n4, row, a, (const float4*)(g + o_sh), (float4*)(p + o_sh),
                                                                       (float4*)(m1 + o_sh), (float4*)(m2 + o_sh));
    if (n4 * 4 < n_sh) {
        const size_t rest = n_sh - n4 * 4;
        adam_sh_scalar_kernel<<<(unsigned)((rest + 255) / 256), 256, 0, s>>>(n4 * 4, n_sh, row, a, g + o_sh, p + o_sh, m1 + o_sh, m2 + o_sh);
    }
    gs_count_launches(1 + (n4 ? 1 : 0) + (n4 * 4 < n_sh ? 1 : 0));
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int32_t gs_b200_densify_stats(int32_t N, const float* g_means2D, const int32_t* radii, float* grad_accum, float* denom,
                              float* max_radii, void* stream) {
    if (N > 0 && (!g_means2D || !radii || !grad_accum || !denom || !max_radii)) { gs_set_error("densify_stats: NULL"); return 1; }
    const cudaStream_t s = (cudaStream_t)stream;
    if (N <= 0) return 0;
    densify_stats_kernel<<<(N + 255) / 256, 256, 0, s>>>(N, g_means2D, radii, grad_accum, denom, max_radii);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

}  // extern "C"
