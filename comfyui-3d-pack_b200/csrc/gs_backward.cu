// Backward of the per-Gaussian preprocess: chains the composite's per-splat
// raw moment sums (SplatGrad) to means3D, scales, rotations (or cov3D), SH
// coefficients (or colours), opacities and the screen-space means2D gradient.
//
// Replaces preprocessCUDA + computeCov2DCUDA of the backward pass of
// diff_gaussian_rasterization (SURVEY.md App. A.1.7).  All forward
// intermediates are recomputed from the inputs (nothing but `radii` is saved).
// Quirks kept (they define the reference's gradients):
//   * 1/(det^2 + 1e-7) in the conic->cov2D chain;
//   * zero gradient to t.x / t.y when the 1.3*tanfov clamp is active, while
//     t.z differentiates J with the clamped value held fixed;
//   * SH clamp mask, decided on the forward's own colour (gs_sh_colour); quaternion NOT normalised inside.
//
// Two kernels share one per-view device function:
//   preprocess_backward_kernel        one view  (the drop-in backward op)
//   preprocess_backward_multi_kernel  V views in one pass over the Gaussians (multi-view step): parameters
//       are read once, gradients written once; dL/dSigma3D is summed over views BEFORE the scale/quaternion
//       chain (Sigma3D is view independent), SH gradients accumulate in shared memory.
#include "gs_common.cuh"

namespace {

constexpr int PB_THREADS = 128;
constexpr int PB_MAXV = 16;

struct ViewB {
    const float* m; const float* p; const float* cam;
    float tanfovx, tanfovy, fx, fy;
    int W, H, deg;
};

struct GaussAcc {           // per-Gaussian accumulators over views
    float dmx = 0.f, dmy = 0.f, dmz = 0.f;
    float g2x = 0.f, g2y = 0.f;
    float dop = 0.f;
    float dcv[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float dcol[3] = {0.f, 0.f, 0.f};
};

// cov3D and (optionally) the rotation matrix / scaled scales it was built from
__device__ __forceinline__ void cov3d_fwd(const float* __restrict__ scales, const float* __restrict__ rotations,
                                          const float* __restrict__ cov3D_precomp, float mod, int idx, float c[6],
                                          float R[9], float sc[3]) {
    if (cov3D_precomp != nullptr) {
        const float* cp = cov3D_precomp + 6 * (size_t)idx;
#pragma unroll
        for (int k = 0; k < 6; k++) c[k] = cp[k];
        return;
    }
    sc[0] = mod * scales[3 * idx + 0]; sc[1] = mod * scales[3 * idx + 1]; sc[2] = mod * scales[3 * idx + 2];
    const float* q = rotations + 4 * (size_t)idx;
    const float r = q[0], qx = q[1], qy = q[2], qz = q[3];
    R[0] = 1.f - 2.f * (qy * qy + qz * qz); R[1] = 2.f * (qx * qy - r * qz); R[2] = 2.f * (qx * qz + r * qy);
    R[3] = 2.f * (qx * qy + r * qz); R[4] = 1.f - 2.f * (qx * qx + qz * qz); R[5] = 2.f * (qy * qz - r * qx);
    R[6] = 2.f * (qx * qz - r * qy); R[7] = 2.f * (qy * qz + r * qx); R[8] = 1.f - 2.f * (qx * qx + qy * qy);
    const float M00 = R[0] * sc[0], M01 = R[1] * sc[1], M02 = R[2] * sc[2];
    const float M10 = R[3] * sc[0], M11 = R[4] * sc[1], M12 = R[5] * sc[2];
    const float M20 = R[6] * sc[0], M21 = R[7] * sc[1], M22 = R[8] * sc[2];
    c[0] = M00 * M00 + M01 * M01 + M02 * M02; c[1] = M00 * M10 + M01 * M11 + M02 * M12;
    c[2] = M00 * M20 + M01 * M21 + M02 * M22; c[3] = M10 * M10 + M11 * M11 + M12 * M12;
    c[4] = M10 * M20 + M11 * M21 + M12 * M22; c[5] = M20 * M20 + M21 * M21 + M22 * M22;
}

// dL/dSigma3D (6 unique entries) -> dL/dscale, dL/dquaternion
__device__ __forceinline__ void cov3d_bwd(const float dcv[6], const float R[9], const float sc[3], float mod,
                                          const float* __restrict__ q, float dsc[3], float dq[4]) {
    const float Gxx = dcv[0], Gxy = 0.5f * dcv[1], Gxz = 0.5f * dcv[2], Gyy = dcv[3], Gyz = 0.5f * dcv[4], Gzz = dcv[5];
    float dR[9];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float M0k = R[0 + k] * sc[k], M1k = R[3 + k] * sc[k], M2k = R[6 + k] * sc[k];
        const float dM0 = 2.f * (Gxx * M0k + Gxy * M1k + Gxz * M2k);
        const float dM1 = 2.f * (Gxy * M0k + Gyy * M1k + Gyz * M2k);
        const float dM2 = 2.f * (Gxz * M0k + Gyz * M1k + Gzz * M2k);
        dsc[k] = mod * (dM0 * R[0 + k] + dM1 * R[3 + k] + dM2 * R[6 + k]);
        dR[0 + k] = dM0 * sc[k]; dR[3 + k] = dM1 * sc[k]; dR[6 + k] = dM2 * sc[k];
    }
    const float r = q[0], qx = q[1], qy = q[2], qz = q[3];
    dq[0] = 2.f * (qz * (dR[3] - dR[1]) + qy * (dR[2] - dR[6]) + qx * (dR[7] - dR[5]));
    dq[1] = 2.f * (qy * (dR[1] + dR[3]) + qz * (dR[2] + dR[6]) + r * (dR[7] - dR[5])) - 4.f * qx * (dR[4] + dR[8]);
    dq[2] = 2.f * (qx * (dR[1] + dR[3]) + r * (dR[2] - dR[6]) + qz * (dR[5] + dR[7])) - 4.f * qy * (dR[0] + dR[8]);
    dq[3] = 2.f * (r * (dR[3] - dR[1]) + qx * (dR[2] + dR[6]) + qy * (dR[5] + dR[7])) - 4.f * qz * (dR[0] + dR[4]);
}

// One view's contribution for one visible Gaussian.  sh_row: this Gaussian's SH inputs (shared memory) or null;
// dsh_row: where dL/dSH goes (ACCUM: +=, may not alias sh_row; !ACCUM: =, may alias sh_row).
template <bool ACCUM>
__device__ __forceinline__ void backward_view(const ViewB& vb, int M, float x, float y, float z, const float c[6],
                                              const float4 gg, const float4 gc4, const float4 gk,
                                              const float* sh_row, float* dsh_row, bool has_sh, GaussAcc& A) {
    const float* m = vb.m;
    const float* p = vb.p;
    const float tx = m[0] * x + m[4] * y + m[8] * z + m[12];
    const float ty = m[1] * x + m[5] * y + m[9] * z + m[13];
    const float tz = m[2] * x + m[6] * y + m[10] * z + m[14];
    const float hx = p[0] * x + p[4] * y + p[8] * z + p[12];
    const float hy = p[1] * x + p[5] * y + p[9] * z + p[13];
    const float hw = p[3] * x + p[7] * y + p[11] * z + p[15];
    const float pw = 1.0f / (hw + 0.0000001f);
    float dmx = m[2] * gg.z, dmy = m[6] * gg.z, dmz = m[10] * gg.z;       // depth
    A.dop += gc4.w;

    // ---- colour ---------------------------------------------------------
    if (has_sh) {
        const int deg = vb.deg;
        const float vx = x - vb.cam[0], vy = y - vb.cam[1], vz = z - vb.cam[2];
        // the clamp mask is decided on the forward's colour, bit for bit (the chain below keeps its own arithmetic)
        float rgb[3];
        gs_sh_colour(deg, sh_row, vx, vy, vz, rgb);
        const float inv = 1.0f / sqrtf(vx * vx + vy * vy + vz * vz);
        const float dx = vx * inv, dy = vy * inv, dz = vz * inv;
        float bas[16], bx[16], by[16], bz[16];
#pragma unroll
        for (int k = 0; k < 16; k++) { bas[k] = 0.f; bx[k] = 0.f; by[k] = 0.f; bz[k] = 0.f; }
        bas[0] = SH_C0;
        int nb = 1;
        if (deg > 0) {
            nb = 4;
            bas[1] = -SH_C1 * dy; by[1] = -SH_C1;
            bas[2] = SH_C1 * dz;  bz[2] = SH_C1;
            bas[3] = -SH_C1 * dx; bx[3] = -SH_C1;
            if (deg > 1) {
                nb = 9;
                const float xx = dx * dx, yy = dy * dy, zz = dz * dz, xy = dx * dy, yz = dy * dz, xz = dx * dz;
                bas[4] = SH_C2_0 * xy; bx[4] = SH_C2_0 * dy; by[4] = SH_C2_0 * dx;
                bas[5] = SH_C2_1 * yz; by[5] = SH_C2_1 * dz; bz[5] = SH_C2_1 * dy;
                bas[6] = SH_C2_2 * (2.f * zz - xx - yy); bx[6] = SH_C2_2 * -2.f * dx; by[6] = SH_C2_2 * -2.f * dy; bz[6] = SH_C2_2 * 4.f * dz;
                bas[7] = SH_C2_3 * xz; bx[7] = SH_C2_3 * dz; bz[7] = SH_C2_3 * dx;
                bas[8] = SH_C2_4 * (xx - yy); bx[8] = SH_C2_4 * 2.f * dx; by[8] = SH_C2_4 * -2.f * dy;
                if (deg > 2) {
                    nb = 16;
                    bas[9] = SH_C3_0 * dy * (3.f * xx - yy); bx[9] = SH_C3_0 * 6.f * xy; by[9] = SH_C3_0 * (3.f * xx - 3.f * yy);
                    bas[10] = SH_C3_1 * xy * dz; bx[10] = SH_C3_1 * yz; by[10] = SH_C3_1 * xz; bz[10] = SH_C3_1 * xy;
                    bas[11] = SH_C3_2 * dy * (4.f * zz - xx - yy); bx[11] = SH_C3_2 * -2.f * xy; by[11] = SH_C3_2 * (4.f * zz - xx - 3.f * yy); bz[11] = SH_C3_2 * 8.f * yz;
                    bas[12] = SH_C3_3 * dz * (2.f * zz - 3.f * xx - 3.f * yy); bx[12] = SH_C3_3 * -6.f * xz; by[12] = SH_C3_3 * -6.f * yz; bz[12] = SH_C3_3 * (6.f * zz - 3.f * xx - 3.f * yy);
                    bas[13] = SH_C3_4 * dx * (4.f * zz - xx - yy); bx[13] = SH_C3_4 * (4.f * zz - 3.f * xx - yy); by[13] = SH_C3_4 * -2.f * xy; bz[13] = SH_C3_4 * 8.f * xz;
                    bas[14] = SH_C3_5 * dz * (xx - yy); bx[14] = SH_C3_5 * 2.f * xz; by[14] = SH_C3_5 * -2.f * yz; bz[14] = SH_C3_5 * (xx - yy);
                    bas[15] = SH_C3_6 * dx * (xx - 3.f * yy); bx[15] = SH_C3_6 * (3.f * xx - 3.f * yy); by[15] = SH_C3_6 * -6.f * xy;
                }
            }
        }
        const float dr = (rgb[0] < 0.f) ? 0.f : gk.x, dg = (rgb[1] < 0.f) ? 0.f : gk.y, db = (rgb[2] < 0.f) ? 0.f : gk.z;
        float ddx = 0.f, ddy = 0.f, ddz = 0.f;
#pragma unroll
        for (int k = 0; k < 16; k++) {
            if (k < nb) {
                const float s = dr * sh_row[3 * k] + dg * sh_row[3 * k + 1] + db * sh_row[3 * k + 2];
                ddx += bx[k] * s; ddy += by[k] * s; ddz += bz[k] * s;
                if (ACCUM) { dsh_row[3 * k] += bas[k] * dr; dsh_row[3 * k + 1] += bas[k] * dg; dsh_row[3 * k + 2] += bas[k] * db; }
                else { dsh_row[3 * k] = bas[k] * dr; dsh_row[3 * k + 1] = bas[k] * dg; dsh_row[3 * k + 2] = bas[k] * db; }
            }
        }
        if (!ACCUM) for (int k = 3 * nb; k < 3 * M; k++) dsh_row[k] = 0.f;
        const float dot = dx * ddx + dy * ddy + dz * ddz;      // back through dir = v/|v|
        dmx += (ddx - dx * dot) * inv; dmy += (ddy - dy * dot) * inv; dmz += (ddz - dz * dot) * inv;
    } else {
        A.dcol[0] += gk.x; A.dcol[1] += gk.y; A.dcol[2] += gk.z;
    }

    // ---- cov2D / conic chain ---------------------------------------------
    const float c0 = c[0], c1 = c[1], c2 = c[2], c3 = c[3], c4 = c[4], c5 = c[5];
    const float fx = vb.fx, fy = vb.fy;
    const float limx = 1.3f * vb.tanfovx, limy = 1.3f * vb.tanfovy;
    const float txtz = tx / tz, tytz = ty / tz;
    const float cx = fminf(limx, fmaxf(-limx, txtz)) * tz;
    const float cy = fminf(limy, fmaxf(-limy, tytz)) * tz;
    const float xmul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
    const float ymul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
    const float itz = 1.0f / tz, itz2 = itz * itz, itz3 = itz2 * itz;
    const float J00 = fx * itz, J02 = -(fx * cx) * itz2, J11 = fy * itz, J12 = -(fy * cy) * itz2;
    const float T00 = J00 * m[0] + J02 * m[2], T01 = J00 * m[4] + J02 * m[6], T02 = J00 * m[8] + J02 * m[10];
    const float T10 = J11 * m[1] + J12 * m[2], T11 = J11 * m[5] + J12 * m[6], T12 = J11 * m[9] + J12 * m[10];
    const float v00 = c0 * T00 + c1 * T01 + c2 * T02, v01 = c1 * T00 + c3 * T01 + c4 * T02, v02 = c2 * T00 + c4 * T01 + c5 * T02;
    const float v10 = c0 * T10 + c1 * T11 + c2 * T12, v11 = c1 * T10 + c3 * T11 + c4 * T12, v12 = c2 * T10 + c4 * T11 + c5 * T12;
    const float ca = T00 * v00 + T01 * v01 + T02 * v02 + 0.3f;
    const float cb = T00 * v10 + T01 * v11 + T02 * v12;
    const float cc = T10 * v10 + T11 * v11 + T12 * v12 + 0.3f;
    const float denom = ca * cc - cb * cb;
    const float d2i = 1.0f / (denom * denom + 0.0000001f);
    // composite hands over raw moment sums; true partials wrt the conic (A,B,C) and the pixel mean:
    const float gA = -0.5f * gc4.x, gB = -gc4.y, gC = -0.5f * gc4.z;
    {
        const float di = (denom != 0.f) ? 1.0f / denom : 0.f;
        const float cA = cc * di, cB = -cb * di, cC = ca * di;
        const float dpx = -(cA * gg.x + cB * gg.y), dpy = -(cB * gg.x + cC * gg.y);
        const float g2x = dpx * (0.5f * (float)vb.W), g2y = dpy * (0.5f * (float)vb.H);
        A.g2x += g2x; A.g2y += g2y;
        const float mul1 = hx * pw * pw, mul2 = hy * pw * pw;
        dmx += (p[0] * pw - p[3] * mul1) * g2x + (p[1] * pw - p[3] * mul2) * g2y;
        dmy += (p[4] * pw - p[7] * mul1) * g2x + (p[5] * pw - p[7] * mul2) * g2y;
        dmz += (p[8] * pw - p[11] * mul1) * g2x + (p[9] * pw - p[11] * mul2) * g2y;
    }
    float ga = 0.f, gb = 0.f, gcc = 0.f;
    if (denom != 0.f) {
        ga = d2i * (-cc * cc * gA + cb * cc * gB - cb * cb * gC);
        gb = d2i * (2.f * cb * cc * gA - (denom + 2.f * cb * cb) * gB + 2.f * ca * cb * gC);
        gcc = d2i * (-cb * cb * gA + ca * cb * gB - ca * ca * gC);
    }
    A.dcv[0] += T00 * T00 * ga + T00 * T10 * gb + T10 * T10 * gcc;
    A.dcv[3] += T01 * T01 * ga + T01 * T11 * gb + T11 * T11 * gcc;
    A.dcv[5] += T02 * T02 * ga + T02 * T12 * gb + T12 * T12 * gcc;
    A.dcv[1] += 2.f * T00 * T01 * ga + (T00 * T11 + T01 * T10) * gb + 2.f * T10 * T11 * gcc;
    A.dcv[2] += 2.f * T00 * T02 * ga + (T00 * T12 + T02 * T10) * gb + 2.f * T10 * T12 * gcc;
    A.dcv[4] += 2.f * T01 * T02 * ga + (T01 * T12 + T02 * T11) * gb + 2.f * T11 * T12 * gcc;
    const float dT00 = 2.f * ga * v00 + gb * v10, dT01 = 2.f * ga * v01 + gb * v11, dT02 = 2.f * ga * v02 + gb * v12;
    const float dT10 = 2.f * gcc * v10 + gb * v00, dT11 = 2.f * gcc * v11 + gb * v01, dT12 = 2.f * gcc * v12 + gb * v02;
    const float dJ00 = m[0] * dT00 + m[4] * dT01 + m[8] * dT02;
    const float dJ02 = m[2] * dT00 + m[6] * dT01 + m[10] * dT02;
    const float dJ11 = m[1] * dT10 + m[5] * dT11 + m[9] * dT12;
    const float dJ12 = m[2] * dT10 + m[6] * dT11 + m[10] * dT12;
    const float dtx = xmul * (-fx * itz2) * dJ02;
    const float dty = ymul * (-fy * itz2) * dJ12;
    const float dtz = -fx * itz2 * dJ00 - fy * itz2 * dJ11 + (2.f * fx * cx) * itz3 * dJ02 + (2.f * fy * cy) * itz3 * dJ12;
    dmx += m[0] * dtx + m[1] * dty + m[2] * dtz;
    dmy += m[4] * dtx + m[5] * dty + m[6] * dtz;
    dmz += m[8] * dtx + m[9] * dty + m[10] * dtz;
    A.dmx += dmx; A.dmy += dmy; A.dmz += dmz;
}

__device__ __forceinline__ void store_grads(bool live, bool any_vis, int accumulate, int idx, const GaussAcc& A,
                                            const float dsc[3], const float dq[4], float* dmeans3D, float* dmeans2D,
                                            float* dcolors, float* dopac, float* dscales, float* drots, float* dcov3D) {
    if (!live) return;
    if (accumulate) {
        if (!any_vis) return;
        dmeans3D[3 * idx] += A.dmx; dmeans3D[3 * idx + 1] += A.dmy; dmeans3D[3 * idx + 2] += A.dmz;
        dmeans2D[3 * idx] += A.g2x; dmeans2D[3 * idx + 1] += A.g2y;
        dopac[idx] += A.dop;
        if (dscales) { for (int k = 0; k < 3; k++) dscales[3 * idx + k] += dsc[k]; for (int k = 0; k < 4; k++) drots[4 * idx + k] += dq[k]; }
        if (dcov3D) for (int k = 0; k < 6; k++) dcov3D[6 * (size_t)idx + k] += A.dcv[k];
        if (dcolors) for (int k = 0; k < 3; k++) dcolors[3 * idx + k] += A.dcol[k];
    } else {
        dmeans3D[3 * idx] = A.dmx; dmeans3D[3 * idx + 1] = A.dmy; dmeans3D[3 * idx + 2] = A.dmz;
        dmeans2D[3 * idx] = A.g2x; dmeans2D[3 * idx + 1] = A.g2y; dmeans2D[3 * idx + 2] = 0.f;
        dopac[idx] = A.dop;
        if (dscales) { for (int k = 0; k < 3; k++) dscales[3 * idx + k] = dsc[k]; for (int k = 0; k < 4; k++) drots[4 * idx + k] = dq[k]; }
        if (dcov3D) for (int k = 0; k < 6; k++) dcov3D[6 * (size_t)idx + k] = A.dcv[k];
        if (dcolors) for (int k = 0; k < 3; k++) dcolors[3 * idx + k] = A.dcol[k];
    }
}

__global__ void __launch_bounds__(PB_THREADS)
preprocess_backward_kernel(ViewArgs va, int N, int M, const float* __restrict__ means3D,
                           const float* __restrict__ shs, const float* __restrict__ colors_precomp,
                           const float* __restrict__ opacities, const float* __restrict__ scales,
                           const float* __restrict__ rotations, const float* __restrict__ cov3D_precomp,
                           const int32_t* __restrict__ radii, const SplatGrad* __restrict__ sg,
                           float* __restrict__ dmeans3D, float* __restrict__ dmeans2D, float* __restrict__ dshs,
                           float* __restrict__ dcolors, float* __restrict__ dopac, float* __restrict__ dscales,
                           float* __restrict__ drots, float* __restrict__ dcov3D, int accumulate) {
    extern __shared__ __align__(16) float s_sh[];     // [128][3M|1]: SH in, dSH out
    __shared__ float s_view[16], s_proj[16], s_cam[3];
    const int tid = threadIdx.x;
    const int base = blockIdx.x * PB_THREADS;
    if (tid < 16) { s_view[tid] = __ldg(va.view + tid); s_proj[tid] = __ldg(va.proj + tid); }
    if (tid < 3) s_cam[tid] = __ldg(va.campos + tid);
    const int row = 3 * M;
    const int rowp = gs_rowp(row);
    const int cnt = min(PB_THREADS, N - base);
    const size_t goff = (size_t)base * row;
    if (shs != nullptr) gs_stage_rows_in(s_sh, shs + goff, cnt, row, tid, PB_THREADS);
    __syncthreads();

    const int idx = base + tid;
    const bool live = idx < N;
    const bool vis = live && radii[idx] > 0;
    GaussAcc A;
    float dsc[3] = {0.f, 0.f, 0.f}, dq[4] = {0.f, 0.f, 0.f, 0.f};
    float* my_sh = s_sh + tid * rowp;
    if (vis) {
        const float x = means3D[3 * idx + 0], y = means3D[3 * idx + 1], z = means3D[3 * idx + 2];
        float c[6], R[9], sc[3];
        cov3d_fwd(scales, rotations, cov3D_precomp, va.scale_modifier, idx, c, R, sc);
        ViewB vb{s_view, s_proj, s_cam, va.tanfovx, va.tanfovy, va.focal_x, va.focal_y, va.W, va.H, va.sh_degree};
        backward_view<false>(vb, M, x, y, z, c, sg_f4(sg[idx].g), sg_f4(sg[idx].c), sg_f4(sg[idx].k), my_sh, my_sh, shs != nullptr, A);
        if (cov3D_precomp == nullptr) cov3d_bwd(A.dcv, R, sc, va.scale_modifier, rotations + 4 * (size_t)idx, dsc, dq);
    } else if (live && shs != nullptr) {
        for (int k = 0; k < row; k++) my_sh[k] = 0.f;
    }
    store_grads(live, vis, accumulate, idx, A, dsc, dq, dmeans3D, dmeans2D, dcolors, dopac, dscales, drots, dcov3D);
    if (dshs != nullptr) {
        __syncthreads();
        gs_stage_rows_out(s_sh, dshs + goff, cnt, row, tid, PB_THREADS, accumulate);
    }
}

// V views in one pass (SH + scale/rotation parameterisation only — what the optimisation step uses).
// sg, radii: [V][N].
__global__ void __launch_bounds__(PB_THREADS, 4)     // 128 registers: 4 CTAs / SM (was 168 -> 3)
preprocess_backward_multi_kernel(const float* __restrict__ views, int V, int W, int H, int sh_degree,
                                 float scale_modifier, int N, int M, const float* __restrict__ means3D,
                                 const float* __restrict__ shs, const float* __restrict__ scales,
                                 const float* __restrict__ rotations, const int32_t* __restrict__ radii,
                                 const SplatGrad* __restrict__ sg, float* __restrict__ dmeans3D,
                                 float* __restrict__ dmeans2D, float* __restrict__ dshs, float* __restrict__ dopac,
                                 float* __restrict__ dscales, float* __restrict__ drots, int accumulate, int first,
                                 int count) {
    extern __shared__ __align__(16) float s_all[];    // [128][rowp] SH in, then [128][rowp] dSH accumulators
    __shared__ float s_views[PB_MAXV * 40];
    const int tid = threadIdx.x;
    const int base = first + blockIdx.x * PB_THREADS;       // Gaussian range [first, first+count), first % 128 == 0
    const int row = 3 * M;
    const int rowp = gs_rowp(row);
    float* s_sh = s_all;
    float* s_dsh = s_all + PB_THREADS * rowp;
    for (int i = tid; i < V * 40; i += PB_THREADS) s_views[i] = __ldg(views + i);
    const int cnt = min(PB_THREADS, first + count - base);
    const size_t goff = (size_t)base * row;
    gs_stage_rows_in(s_sh, shs + goff, cnt, row, tid, PB_THREADS);
    for (int i = tid; i < PB_THREADS * rowp; i += PB_THREADS) s_dsh[i] = 0.f;
    __syncthreads();

    const int idx = base + tid;
    const bool live = idx < first + count;
    GaussAcc A;
    float dsc[3] = {0.f, 0.f, 0.f}, dq[4] = {0.f, 0.f, 0.f, 0.f};
    bool any_vis = false;
    if (live) {
        const float x = means3D[3 * idx + 0], y = means3D[3 * idx + 1], z = means3D[3 * idx + 2];
        float c[6], R[9], sc[3];
        cov3d_fwd(scales, rotations, nullptr, scale_modifier, idx, c, R, sc);
        // visibility of every view first (V independent loads in flight instead of one load -> branch -> load chain per
        // view), then the visible views in order with the NEXT view's screen-space gradients loading while the current
        // view's chain is evaluated: the kernel was long-scoreboard bound at 16 warps / SM
        uint32_t vis = 0;
#pragma unroll 4
        for (int v = 0; v < V; v++) vis |= (radii[(size_t)v * N + idx] > 0 ? 1u : 0u) << v;
        any_vis = vis != 0;
        float4 ng = make_float4(0.f, 0.f, 0.f, 0.f), nc = ng, nk = ng;
        if (vis) { const SplatGrad* q = sg + (size_t)(__ffs(vis) - 1) * N + idx; ng = sg_f4(q->g); nc = sg_f4(q->c); nk = sg_f4(q->k); }
        while (vis) {
            const int v = __ffs(vis) - 1;
            vis &= vis - 1;
            const float4 cg = ng, cc = nc, ck = nk;
            if (vis) { const SplatGrad* q = sg + (size_t)(__ffs(vis) - 1) * N + idx; ng = sg_f4(q->g); nc = sg_f4(q->c); nk = sg_f4(q->k); }
            const float* vw = s_views + v * 40;
            const float tfx = vw[38], tfy = vw[39];
            ViewB vb{vw, vw + 16, vw + 32, tfx, tfy, (float)W / (2.0f * tfx), (float)H / (2.0f * tfy), W, H, sh_degree};
            backward_view<true>(vb, M, x, y, z, c, cg, cc, ck, s_sh + tid * rowp, s_dsh + tid * rowp, true, A);
        }
        if (any_vis) cov3d_bwd(A.dcv, R, sc, scale_modifier, rotations + 4 * (size_t)idx, dsc, dq);
    }
    store_grads(live, any_vis, accumulate, idx, A, dsc, dq, dmeans3D, dmeans2D, nullptr, dopac, dscales, drots, nullptr);
    __syncthreads();
    gs_stage_rows_out(s_dsh, dshs + goff, cnt, row, tid, PB_THREADS, accumulate);
}

}  // namespace

int gs_launch_preprocess_backward(const ViewArgs& va, int N, int M, const float* means3D, const float* shs,
                                  const float* colors_precomp, const float* opacities, const float* scales,
                                  const float* rotations, const float* cov3D_precomp, const int32_t* radii,
                                  const SplatGrad* sg, float* dmeans3D, float* dmeans2D, float* dshs,
                                  float* dcolors, float* dopac, float* dscales, float* drots, float* dcov3D,
                                  int accumulate, cudaStream_t s) {
    if (N <= 0) return 0;
    size_t smem = shs ? (size_t)PB_THREADS * ((3 * M) | 1) * sizeof(float) : 0;
    if (smem > 48 * 1024)
        GS_CUDA_CHECK(cudaFuncSetAttribute(preprocess_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int blocks = (N + PB_THREADS - 1) / PB_THREADS;
    preprocess_backward_kernel<<<blocks, PB_THREADS, smem, s>>>(va, N, M, means3D, shs, colors_precomp, opacities,
                                                                scales, rotations, cov3D_precomp, radii, sg, dmeans3D,
                                                                dmeans2D, dshs, dcolors, dopac, dscales, drots, dcov3D,
                                                                accumulate);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int gs_launch_preprocess_backward_multi(const float* views_dev, int V, int W, int H, int sh_degree,
                                        float scale_modifier, int N, int M, const float* means3D, const float* shs,
                                        const float* scales, const float* rotations, const int32_t* radii,
                                        const SplatGrad* sg, float* dmeans3D, float* dmeans2D, float* dshs,
                                        float* dopac, float* dscales, float* drots, int accumulate, int first, int count,
                                        cudaStream_t s) {
    if (N <= 0 || V <= 0 || count <= 0) return 0;
    if (first % PB_THREADS) { gs_set_error("preprocess_backward_multi: range start must be a multiple of %d", PB_THREADS); return 1; }
    if (V > PB_MAXV) { gs_set_error("preprocess_backward_multi: V=%d > %d", V, PB_MAXV); return 1; }
    size_t smem = 2 * (size_t)PB_THREADS * ((3 * M) | 1) * sizeof(float);
    static bool attr_set = false;
    if (smem > 48 * 1024 && !attr_set) {
        GS_CUDA_CHECK(cudaFuncSetAttribute(preprocess_backward_multi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        GS_CUDA_CHECK(cudaFuncSetAttribute(preprocess_backward_multi_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                           (int)cudaSharedmemCarveoutMaxShared));
        attr_set = true;
    }
    int blocks = (count + PB_THREADS - 1) / PB_THREADS;
    preprocess_backward_multi_kernel<<<blocks, PB_THREADS, smem, s>>>(views_dev, V, W, H, sh_degree, scale_modifier, N, M,
                                                                      means3D, shs, scales, rotations, radii, sg, dmeans3D,
                                                                      dmeans2D, dshs, dopac, dscales, drots, accumulate, first,
                                                                      count);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
