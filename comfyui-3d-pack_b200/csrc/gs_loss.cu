// Image loss of the optimisation step and its gradient, as CUDA kernels on the view's own stream:
//   loss = (1-ls) * L1(img*m, ref*m) + la * MSE(alpha, m) + ls * (1 - MS-SSIM(ref*m, img*m)),  img = clamp(rgb, 0, 1)
// (GaussianSplatting3D.training, main_3DGS.py:184-192; MS-SSIM = pytorch_msssim.MS_SSIM(data_range=1, channel=3):
// 11-tap Gaussian sigma 1.5, valid convolution, 5 scales, 2x2 average pooling with padding = size % 2, weights
// .0448/.2856/.3001/.2363/.1333, relu on the per-channel means, product of powers, mean over channels).
// The torch restatement in gs_b200/losses.py is the checker (tests/test_gpu_trainer.py); this file exists because at
// 1080p the ~200 small torch kernels of that graph cost more host time per view than the whole rasterizer step.
//
// Per view:  prep (mask, clamp, L1/MSE sums) -> per scale [fused row+column filter + map sums -> pool] ->
// coefficients (one thread) -> per scale, coarse to fine [fused row+column filter + map derivatives ->
// transposed column filter -> transposed row filter + combine + pooled gradient of the coarser scale] -> final.
// All planes are [3][H][W] fp32; everything is streaming / stencil work (HBM / L2 bound, < 1 GB per 1080p view).
#include "gs_common.cuh"

namespace {

constexpr int WIN = 11;
constexpr int LEVELS = 5;
struct Win { float w[WIN]; };        // 11-tap Gaussian, passed by value (no per-device constant state)
__constant__ float c_msw[LEVELS] = {0.0448f, 0.2856f, 0.3001f, 0.2363f, 0.1333f};
constexpr float SSIM_C1 = 0.01f * 0.01f, SSIM_C2 = 0.03f * 0.03f;

struct LossAcc {            // device accumulators of one view
    // the block partials meet in fp64 reds: at 1080p ~8000 fp32 atomics per sum drifted ~1e-6 relative
    double l1_sum, mse_sum;
    double sums[LEVELS][3][2];    // [level][channel]{ssim_map sum, cs_map sum}
    float coef[LEVELS][3][2];     // per-location coefficients {d loss / d ssim_map, d loss / d cs_map}
};

__device__ __forceinline__ float block_sum(float v, float* s_red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    v = (threadIdx.x < nw) ? s_red[threadIdx.x] : 0.f;
    if (warp == 0) for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    return v;    // valid in thread 0
}

// X0 = ref * m, Y0 = clamp(rgb) * m; sums of |Y0 - X0| and (alpha - m)^2
__global__ void __launch_bounds__(256)
prep_kernel(int npix, const float* __restrict__ img, const float* __restrict__ ref, const float* __restrict__ mask,
            float* __restrict__ X0, float* __restrict__ Y0, LossAcc* __restrict__ acc) {
    __shared__ float s_red[8];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float l1 = 0.f, mse = 0.f;
    if (i < npix) {
        const float m = mask[i];
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const float y = fminf(fmaxf(img[(size_t)c * npix + i], 0.f), 1.f) * m;
            const float x = ref[(size_t)c * npix + i] * m;
            X0[(size_t)c * npix + i] = x; Y0[(size_t)c * npix + i] = y;
            l1 += fabsf(y - x);
        }
        const float d = img[(size_t)4 * npix + i] - m;
        mse = d * d;
    }
    l1 = block_sum(l1, s_red);
    if (threadIdx.x == 0) atomicAdd(&acc->l1_sum, (double)l1);
    mse = block_sum(mse, s_red);
    if (threadIdx.x == 0) atomicAdd(&acc->mse_sum, (double)mse);
}

// Gaussian-window statistics of one 32x8 tile of window positions, fused row + column filter through shared memory:
// the (32+10)x(8+10) input tile of X and Y is staged once, the row filter writes its five quantities
// {x, y, x^2, y^2, xy} for 18 rows into shared memory, the column filter reads them back.  (The unfused version
// round-tripped those five planes through HBM: 250 MB per 1080p scale-0 pass, twice per view.)
constexpr int ST_W = 32, ST_H = 8, ST_IW = ST_W + WIN - 1, ST_IH = ST_H + WIN - 1;
struct Stats { float mx, my, ex2, ey2, exy; };

__device__ __forceinline__ Stats tile_stats(const Win& win, int Hs, int Ws, const float* __restrict__ X, const float* __restrict__ Y,
                                            float (*s_xy)[ST_IH][ST_IW], float (*s_r)[ST_IH][ST_W], bool& valid, int& xo, int& yo) {
    const int Wo = Ws - (WIN - 1), Ho = Hs - (WIN - 1);
    const int c = blockIdx.z, x0 = blockIdx.x * ST_W, y0 = blockIdx.y * ST_H;
    const int tid = threadIdx.x;
    const float* xc = X + (size_t)c * Hs * Ws;
    const float* yc = Y + (size_t)c * Hs * Ws;
    for (int i = tid; i < ST_IH * ST_IW; i += ST_W * ST_H) {
        const int r = i / ST_IW, q = i - r * ST_IW;
        const int gy = y0 + r, gx = x0 + q;
        const bool in = gy < Hs && gx < Ws;
        s_xy[0][r][q] = in ? xc[(size_t)gy * Ws + gx] : 0.f;
        s_xy[1][r][q] = in ? yc[(size_t)gy * Ws + gx] : 0.f;
    }
    __syncthreads();
    for (int i = tid; i < ST_IH * ST_W; i += ST_W * ST_H) {
        const int r = i / ST_W, q = i - r * ST_W;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f, a4 = 0.f;
#pragma unroll
        for (int k = 0; k < WIN; k++) {
            const float w = win.w[k], xv = s_xy[0][r][q + k], yv = s_xy[1][r][q + k];
            a0 = fmaf(w, xv, a0); a1 = fmaf(w, yv, a1); a2 = fmaf(w, xv * xv, a2); a3 = fmaf(w, yv * yv, a3); a4 = fmaf(w, xv * yv, a4);
        }
        s_r[0][r][q] = a0; s_r[1][r][q] = a1; s_r[2][r][q] = a2; s_r[3][r][q] = a3; s_r[4][r][q] = a4;
    }
    __syncthreads();
    const int lx = tid & (ST_W - 1), ly = tid / ST_W;
    xo = x0 + lx; yo = y0 + ly;
    valid = xo < Wo && yo < Ho;
    Stats s{0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < WIN; k++) {
        const float w = win.w[k];
        s.mx = fmaf(w, s_r[0][ly + k][lx], s.mx); s.my = fmaf(w, s_r[1][ly + k][lx], s.my); s.ex2 = fmaf(w, s_r[2][ly + k][lx], s.ex2);
        s.ey2 = fmaf(w, s_r[3][ly + k][lx], s.ey2); s.exy = fmaf(w, s_r[4][ly + k][lx], s.exy);
    }
    return s;
}

// SSIM / CS maps summed per channel
__global__ void __launch_bounds__(ST_W * ST_H)
stats_sums_kernel(Win win, int Hs, int Ws, const float* __restrict__ X, const float* __restrict__ Y, LossAcc* __restrict__ acc, int level) {
    __shared__ float s_xy[2][ST_IH][ST_IW];
    __shared__ float s_r[5][ST_IH][ST_W];
    __shared__ float s_red[8];
    bool valid; int xo, yo;
    const Stats s = tile_stats(win, Hs, Ws, X, Y, s_xy, s_r, valid, xo, yo);
    float ssim = 0.f, cs = 0.f;
    if (valid) {
        const float mxx = s.mx * s.mx, myy = s.my * s.my, mxy = s.mx * s.my;
        const float sx = s.ex2 - mxx, sy = s.ey2 - myy, sxy = s.exy - mxy;
        cs = (2.f * sxy + SSIM_C2) / (sx + sy + SSIM_C2);
        ssim = ((2.f * mxy + SSIM_C1) / (mxx + myy + SSIM_C1)) * cs;
    }
    const int c = blockIdx.z;
    ssim = block_sum(ssim, s_red);
    if (threadIdx.x == 0) atomicAdd(&acc->sums[level][c][0], (double)ssim);
    cs = block_sum(cs, s_red);
    if (threadIdx.x == 0) atomicAdd(&acc->sums[level][c][1], (double)cs);
}

// derivatives of (b*ssim + a*cs) wrt (mu_y, E[y^2], E[xy]) -> D[3][c][yo][xo]
__global__ void __launch_bounds__(ST_W * ST_H)
stats_maps_kernel(Win win, int Hs, int Ws, const float* __restrict__ X, const float* __restrict__ Y, const LossAcc* __restrict__ acc, int level,
                  float* __restrict__ D) {
    __shared__ float s_xy[2][ST_IH][ST_IW];
    __shared__ float s_r[5][ST_IH][ST_W];
    bool valid; int xo, yo;
    const Stats s = tile_stats(win, Hs, Ws, X, Y, s_xy, s_r, valid, xo, yo);
    if (!valid) return;
    const int Wo = Ws - (WIN - 1), Ho = Hs - (WIN - 1), c = blockIdx.z;
    const float b = acc->coef[level][c][0], a = acc->coef[level][c][1];
    const float mxx = s.mx * s.mx, myy = s.my * s.my, mxy = s.mx * s.my;
    const float sx = s.ex2 - mxx, sy = s.ey2 - myy, sxy = s.exy - mxy;
    const float Dcs = sx + sy + SSIM_C2, inv_Dcs = 1.f / Dcs;
    const float cs = (2.f * sxy + SSIM_C2) * inv_Dcs;
    const float Dl = mxx + myy + SSIM_C1, inv_Dl = 1.f / Dl;
    const float l = (2.f * mxy + SSIM_C1) * inv_Dl;
    const float dcs_dexy = 2.f * inv_Dcs, dcs_dey2 = -cs * inv_Dcs;
    const float dcs_dmy = (-2.f * s.mx + 2.f * s.my * cs) * inv_Dcs;
    const float dl_dmy = (2.f * s.mx - 2.f * s.my * l) * inv_Dl;
    const float w_cs = a + b * l;                 // d(b*l*cs + a*cs)/d cs
    const size_t plane = (size_t)3 * Ho * Wo, o = ((size_t)c * Ho + yo) * Wo + xo;
    D[o] = w_cs * dcs_dmy + b * cs * dl_dmy;
    D[plane + o] = w_cs * dcs_dey2;
    D[2 * plane + o] = w_cs * dcs_dexy;
}

// 2x2 average pooling, padding (Hs%2, Ws%2), zeros counted (count_include_pad)
__global__ void __launch_bounds__(256)
pool_kernel(int Hs, int Ws, int Hn, int Wn, const float* __restrict__ X, const float* __restrict__ Y,
            float* __restrict__ Xn, float* __restrict__ Yn) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, c = blockIdx.z;
    if (x >= Wn) return;
    const int py = Hs & 1, px = Ws & 1;
    float sx = 0.f, sy = 0.f;
#pragma unroll
    for (int dy = 0; dy < 2; dy++)
#pragma unroll
        for (int dx = 0; dx < 2; dx++) {
            const int iy = 2 * y - py + dy, ix = 2 * x - px + dx;
            if (iy >= 0 && iy < Hs && ix >= 0 && ix < Ws) {
                const size_t o = ((size_t)c * Hs + iy) * Ws + ix;
                sx += X[o]; sy += Y[o];
            }
        }
    const size_t o = ((size_t)c * Hn + y) * Wn + x;
    Xn[o] = 0.25f * sx; Yn[o] = 0.25f * sy;
}

// one thread: MS-SSIM value, loss value, per-location coefficients for the backward maps
__global__ void coef_kernel(int H, int W, float lambda_ssim, float lambda_alpha, float scale, LossAcc* __restrict__ acc,
                            float* __restrict__ loss_out, int4 dims0, int4 dims1, int dims4h, int dims4w) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const int hs[LEVELS] = {dims0.x, dims0.y, dims0.z, dims0.w, dims4h};
    const int ws[LEVELS] = {dims1.x, dims1.y, dims1.z, dims1.w, dims4w};
    const float npix = (float)H * (float)W;
    float loss = (float)((1.0 - lambda_ssim) * acc->l1_sum / (3.0 * npix) + lambda_alpha * acc->mse_sum / npix);
    for (int l = 0; l < LEVELS; l++) for (int c = 0; c < 3; c++) { acc->coef[l][c][0] = 0.f; acc->coef[l][c][1] = 0.f; }
    if (lambda_ssim > 0.f) {
        float ms = 0.f;
        for (int c = 0; c < 3; c++) {
            float v[LEVELS], P = 1.f;
            for (int l = 0; l < LEVELS; l++) {
                const float cnt = (float)(hs[l] - (WIN - 1)) * (float)(ws[l] - (WIN - 1));
                const float mean = (float)(acc->sums[l][c][l == LEVELS - 1 ? 0 : 1] / cnt);
                v[l] = fmaxf(mean, 0.f);
                P *= powf(v[l], c_msw[l]);
            }
            ms += P;
            for (int l = 0; l < LEVELS; l++) {
                const float cnt = (float)(hs[l] - (WIN - 1)) * (float)(ws[l] - (WIN - 1));
                // d loss / d mean = -scale * ls * (1/3) * w_l * P / v_l ; per location: / cnt
                const float d = (v[l] > 0.f) ? -scale * lambda_ssim * (1.f / 3.f) * c_msw[l] * P / v[l] / cnt : 0.f;
                acc->coef[l][c][l == LEVELS - 1 ? 0 : 1] = d;
            }
        }
        loss += lambda_ssim * (1.f - ms * (1.f / 3.f));
    }
    *loss_out = scale * loss;
}

// transposed column filter: E[k][c][y][xo] = sum_j w[j] D[k][c][y - j][xo]
__global__ void __launch_bounds__(256)
vfull_kernel(Win win, int Hs, int Ws, const float* __restrict__ D, float* __restrict__ E) {
    const int Wo = Ws - (WIN - 1), Ho = Hs - (WIN - 1);
    const int xo = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, c = blockIdx.z;
    if (xo >= Wo) return;
    const size_t dplane = (size_t)3 * Ho * Wo, eplane = (size_t)3 * Hs * Wo;
    float e0 = 0.f, e1 = 0.f, e2 = 0.f;
#pragma unroll
    for (int j = 0; j < WIN; j++) {
        const int yo = y - j;
        if (yo >= 0 && yo < Ho) {
            const float w = win.w[j];
            const size_t o = ((size_t)c * Ho + yo) * Wo + xo;
            e0 = fmaf(w, D[o], e0); e1 = fmaf(w, D[dplane + o], e1); e2 = fmaf(w, D[2 * dplane + o], e2);
        }
    }
    const size_t o = ((size_t)c * Hs + y) * Wo + xo;
    E[o] = e0; E[eplane + o] = e1; E[2 * eplane + o] = e2;
}

// transposed row filter + combine with x, y + pooled gradient of the next coarser scale
__global__ void __launch_bounds__(256)
hfull_combine_kernel(Win win, int Hs, int Ws, const float* __restrict__ E, const float* __restrict__ X, const float* __restrict__ Y,
                     const float* __restrict__ Gn /* coarser gradient or NULL */, int Hn, int Wn, float* __restrict__ G) {
    const int Wo = Ws - (WIN - 1);
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, c = blockIdx.z;
    if (x >= Ws) return;
    const size_t eplane = (size_t)3 * Hs * Wo;
    const float* e = E + ((size_t)c * Hs + y) * Wo;
    float g0 = 0.f, g1 = 0.f, g2 = 0.f;
#pragma unroll
    for (int j = 0; j < WIN; j++) {
        const int xo = x - j;
        if (xo >= 0 && xo < Wo) {
            const float w = win.w[j];
            g0 = fmaf(w, e[xo], g0); g1 = fmaf(w, e[eplane + xo], g1); g2 = fmaf(w, e[2 * eplane + xo], g2);
        }
    }
    const size_t o = ((size_t)c * Hs + y) * Ws + x;
    float g = g0 + 2.f * Y[o] * g1 + X[o] * g2;
    if (Gn) g += 0.25f * Gn[((size_t)c * Hn + ((y + (Hs & 1)) >> 1)) * Wn + ((x + (Ws & 1)) >> 1)];
    G[o] = g;
}

__global__ void __launch_bounds__(256)
final_kernel(int npix, const float* __restrict__ img, const float* __restrict__ mask, const float* __restrict__ X0,
             const float* __restrict__ Y0, const float* __restrict__ G0 /* may be NULL */, float lambda_ssim, float lambda_alpha,
             float scale, float* __restrict__ dL) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    const float m = mask[i];
    const float k1 = scale * (1.f - lambda_ssim) / (3.f * (float)npix);
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float v = img[(size_t)c * npix + i];
        const float d = Y0[(size_t)c * npix + i] - X0[(size_t)c * npix + i];
        float g = k1 * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
        if (G0) g += G0[(size_t)c * npix + i];
        dL[(size_t)c * npix + i] = (v >= 0.f && v <= 1.f) ? g * m : 0.f;     // clamp passes gradient on [0,1]
    }
    dL[(size_t)3 * npix + i] = 0.f;
    dL[(size_t)4 * npix + i] = scale * lambda_alpha * 2.f * (img[(size_t)4 * npix + i] - m) / (float)npix;
}

Win make_window() {
    Win win; float sum = 0.f;
    for (int i = 0; i < WIN; i++) { const float c = (float)(i - WIN / 2); win.w[i] = expf(-(c * c) / (2.f * 1.5f * 1.5f)); sum += win.w[i]; }
    for (int i = 0; i < WIN; i++) win.w[i] /= sum;
    return win;
}

struct Pyr { int h[LEVELS], w[LEVELS]; size_t off[LEVELS], total; };
Pyr make_pyr(int H, int W) {
    Pyr p; size_t o = 0;
    int h = H, w = W;
    for (int l = 0; l < LEVELS; l++) {
        p.h[l] = h; p.w[l] = w; p.off[l] = o; o += (size_t)3 * h * w;
        h = (h + (h & 1)) / 2; w = (w + (w & 1)) / 2;
    }
    p.total = o;
    return p;
}

}  // namespace

size_t gs_image_loss_scratch_bytes(int H, int W) {
    const Pyr p = make_pyr(H, W);
    const size_t npix3 = (size_t)3 * H * W;
    // X, Y, G pyramids + R (5 planes) + D (3 planes) + accumulators
    return (p.total * 3 + npix3 * 8) * sizeof(float) + 1024;
}

int gs_launch_image_loss(int H, int W, const float* img, const float* ref, const float* mask, float lambda_ssim,
                         float lambda_alpha, float scale, float* dL, float* loss_out, void* scratch, cudaStream_t s) {
    if (H <= 0 || W <= 0) { gs_set_error("image_loss: bad size"); return 1; }
    if (lambda_ssim > 0.f && (H <= (WIN - 1) * 16 || W <= (WIN - 1) * 16)) {
        gs_set_error("image_loss: image side must exceed 160 for the 4 downsamplings of MS-SSIM (%dx%d)", W, H); return 1; }
    const Win win = make_window();
    const Pyr p = make_pyr(H, W);
    const int npix = H * W;
    const size_t npix3 = (size_t)3 * npix;
    LossAcc* acc = (LossAcc*)scratch;
    float* base = (float*)((char*)scratch + 1024);
    float* PX = base; float* PY = PX + p.total; float* PG = PY + p.total;
    float* R = PG + p.total; float* D = R + npix3 * 5;
    GS_CUDA_CHECK(cudaMemsetAsync(acc, 0, sizeof(LossAcc), s));
    prep_kernel<<<(npix + 255) / 256, 256, 0, s>>>(npix, img, ref, mask, PX, PY, acc);
    int launches = 1;
    if (lambda_ssim > 0.f) {
        for (int l = 0; l < LEVELS; l++) {
            const int Hs = p.h[l], Ws = p.w[l], Wo = Ws - (WIN - 1), Ho = Hs - (WIN - 1);
            stats_sums_kernel<<<dim3((Wo + ST_W - 1) / ST_W, (Ho + ST_H - 1) / ST_H, 3), ST_W * ST_H, 0, s>>>(win, Hs, Ws, PX + p.off[l],
                                                                                                       PY + p.off[l], acc, l);
            launches += 1;
            if (l + 1 < LEVELS) {
                pool_kernel<<<dim3((p.w[l + 1] + 255) / 256, p.h[l + 1], 3), 256, 0, s>>>(Hs, Ws, p.h[l + 1], p.w[l + 1], PX + p.off[l],
                                                                                         PY + p.off[l], PX + p.off[l + 1], PY + p.off[l + 1]);
                launches++;
            }
        }
    }
    coef_kernel<<<1, 32, 0, s>>>(H, W, lambda_ssim, lambda_alpha, scale, acc, loss_out, make_int4(p.h[0], p.h[1], p.h[2], p.h[3]),
                                 make_int4(p.w[0], p.w[1], p.w[2], p.w[3]), p.h[4], p.w[4]);
    launches++;
    if (lambda_ssim > 0.f) {
        for (int l = LEVELS - 1; l >= 0; l--) {
            const int Hs = p.h[l], Ws = p.w[l], Wo = Ws - (WIN - 1), Ho = Hs - (WIN - 1);
            stats_maps_kernel<<<dim3((Wo + ST_W - 1) / ST_W, (Ho + ST_H - 1) / ST_H, 3), ST_W * ST_H, 0, s>>>(win, Hs, Ws, PX + p.off[l],
                                                                                                       PY + p.off[l], acc, l, D);
            vfull_kernel<<<dim3((Wo + 255) / 256, Hs, 3), 256, 0, s>>>(win, Hs, Ws, D, R);
            const bool has_n = l + 1 < LEVELS;
            hfull_combine_kernel<<<dim3((Ws + 255) / 256, Hs, 3), 256, 0, s>>>(win, Hs, Ws, R, PX + p.off[l], PY + p.off[l],
                                                                               has_n ? PG + p.off[l + 1] : nullptr, has_n ? p.h[l + 1] : 0,
                                                                               has_n ? p.w[l + 1] : 0, PG + p.off[l]);
            launches += 3;
        }
    }
    final_kernel<<<(npix + 255) / 256, 256, 0, s>>>(npix, img, mask, PX, PY, lambda_ssim > 0.f ? PG : nullptr, lambda_ssim,
                                                    lambda_alpha, scale, dL);
    launches++;
    gs_count_launches(launches);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
