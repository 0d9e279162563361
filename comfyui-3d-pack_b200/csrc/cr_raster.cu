// Hunyuan3D's texture-bake rasterizer (the `custom_rasterizer` package: mesh_render.py:145,165-189 in Hunyuan3D 2.0,
// MeshRender.py:373 in 2.1), with findices and barycentrics bit-identical to the reference's CPU path.
//
// Contract (INTEGRATION §3): pos[V,4] clip space, tri[F,3] int32.  Per face, in fp32:
//   x_s = (x/w*0.5 + 0.5)*(W-1) + 0.5,  y_s = (0.5 + (0.5*y)/w)*(H-1) + 0.5,  z_s = (z/w)*0.49999 + 0.5;
// candidate pixels px from (int)min x_s while (float)px < max x_s + 1, clipped to [0, W) (the same for py); a pixel
// centre (px+0.5, py+0.5) is covered when its three barycentrics (signed areas times 1/area, with 1/area and
// 1 - beta - gamma evaluated in double and rounded to float, as the reference's 1.0 literals make them) all lie in the
// closed [0, 1]; depth = (b0 z0 + b1 z1) + b2 z2, skipped when below the prior threshold; the token
// (u64)(int)(depth * 2^18) * (2^31-1) + f + 1 is min-reduced per pixel, so the nearest quantised depth wins and a tie
// goes to the lowest face id, whatever order the atomics land in.  (int) of a value outside the int range, or of NaN,
// is INT_MIN, as x86's cvttss2si gives it; such a token, like every negative one, is above the empty sentinel and
// never wins.  The resolve recomputes the winner's barycentrics at the pixel centre, divides each by its vertex's w
// and renormalises.
// Faces the reference's loop is undefined on are skipped: a vertex id out of range, a non-finite screen coordinate,
// or an x_s / y_s outside the int range.
// THIS TU IS COMPILED WITH -fmad=false: every fp32 expression above is evaluated with one rounding per operation, in
// the order written, as gcc evaluates the reference's CPU path.
#include <type_traits>

#include "gs_common.cuh"

namespace {

constexpr unsigned long long CR_MAXINT = 2147483647ull;
constexpr unsigned long long CR_EMPTY = CR_MAXINT * CR_MAXINT + (CR_MAXINT - 1);
constexpr long long CR_WARP_AREA = 256;     // boxes above this go to the warp queue
constexpr long long CR_CTA_AREA = 8192;     // ... and above this to the CTA queue

struct Face {
    float x0, y0, z0, x1, y1, z1, x2, y2, z2;
    float area, inv;                        // signed area (x2), and (float)(1.0 / area)
    int xlo, xhi, ylo, yhi;                 // candidate pixels, inclusive, clipped to the image
};

__device__ __forceinline__ void screen(const float4 v, int W, int H, float& x, float& y, float& z) {
    x = (v.x / v.w * 0.5f + 0.5f) * (float)(W - 1) + 0.5f;
    y = (0.5f + 0.5f * v.y / v.w) * (float)(H - 1) + 0.5f;
    z = v.z / v.w * 0.49999f + 0.5f;
}

__device__ __forceinline__ bool in_int_range(float v) { return v >= -2147483648.0f && v < 2147483648.0f; }

// false: the face is skipped (bad vertex id, non-finite or out-of-range screen coordinate)
__device__ __forceinline__ bool face_setup(const float4* __restrict__ V, const int32_t* __restrict__ T, int NV, int f,
                                           int W, int H, Face& s) {
    const int i0 = T[3 * f], i1 = T[3 * f + 1], i2 = T[3 * f + 2];
    if ((unsigned)i0 >= (unsigned)NV || (unsigned)i1 >= (unsigned)NV || (unsigned)i2 >= (unsigned)NV) return false;
    screen(V[i0], W, H, s.x0, s.y0, s.z0);
    screen(V[i1], W, H, s.x1, s.y1, s.z1);
    screen(V[i2], W, H, s.x2, s.y2, s.z2);
    if (!(isfinite(s.z0) && isfinite(s.z1) && isfinite(s.z2))) return false;
    if (!(in_int_range(s.x0) && in_int_range(s.x1) && in_int_range(s.x2) && in_int_range(s.y0) && in_int_range(s.y1) &&
          in_int_range(s.y2))) return false;                                   // NaN and +-inf fail here too
    const float xmin = fminf(s.x0, fminf(s.x1, s.x2)), xmax = fmaxf(s.x0, fmaxf(s.x1, s.x2));
    const float ymin = fminf(s.y0, fminf(s.y1, s.y2)), ymax = fmaxf(s.y0, fmaxf(s.y1, s.y2));
    // px < xmax + 1 (a float compare; px < 2^24 converts exactly) <=> px <= ceil(xmax + 1) - 1
    s.xlo = max(0, (int)xmin);
    s.ylo = max(0, (int)ymin);
    s.xhi = (int)fminf(ceilf(xmax + 1.0f) - 1.0f, (float)(W - 1));
    s.yhi = (int)fminf(ceilf(ymax + 1.0f) - 1.0f, (float)(H - 1));
    s.area = (s.x2 - s.x0) * (s.y1 - s.y0) - (s.x1 - s.x0) * (s.y2 - s.y0);
    s.inv = (float)(1.0 / (double)s.area);
    return true;
}

// the reference's barycentric coordinate at p; false when outside [0,1]^3 (zero area and NaN included)
__device__ __forceinline__ bool barycentric(const Face& s, float px, float py, float& a, float& b, float& c) {
    if (s.area == 0.0f) return false;
    const float beta_tri = (s.x2 - s.x0) * (py - s.y0) - (px - s.x0) * (s.y2 - s.y0);
    const float gamma_tri = (px - s.x0) * (s.y1 - s.y0) - (s.x1 - s.x0) * (py - s.y0);
    b = beta_tri * s.inv;
    c = gamma_tri * s.inv;
    a = (float)((1.0 - (double)b) - (double)c);
    return a >= 0.0f && a <= 1.0f && b >= 0.0f && b <= 1.0f && c >= 0.0f && c <= 1.0f;
}

__device__ __forceinline__ void shade(const Face& s, int f, int px, int py, int W, const float* __restrict__ D,
                                      float trunc, unsigned long long* __restrict__ zbuf) {
    float a, b, c;
    if (!barycentric(s, (float)px + 0.5f, (float)py + 0.5f, a, b, c)) return;
    const int pixel = py * W + px;
    const float depth = a * s.z0 + b * s.z1 + c * s.z2;
    const float thres = D ? D[pixel] * 0.49999f + 0.5f + trunc : 0.0f;
    if (depth < thres) return;
    const float zq = depth * 262144.0f;
    const int q = in_int_range(zq) ? __float2int_rz(zq) : INT_MIN;
    const unsigned long long token = (unsigned long long)(long long)q * CR_MAXINT + (unsigned long long)(f + 1);
    if (token < CR_EMPTY) atomicMin(zbuf + pixel, token);      // every other token loses to the sentinel
}

__global__ void __launch_bounds__(256) cr_init_kernel(unsigned long long* __restrict__ zbuf, size_t npix, uint32_t* __restrict__ counts) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 2) counts[i] = 0u;
    if (i < npix) zbuf[i] = CR_EMPTY;
}

// one thread per face: small boxes are rasterized here, larger ones queued
__global__ void __launch_bounds__(256)
cr_small_kernel(const float4* __restrict__ V, const int32_t* __restrict__ T, int NV, int NF, int H, int W, const float* __restrict__ D,
                float trunc, unsigned long long* __restrict__ zbuf, uint32_t* __restrict__ qwarp, uint32_t* __restrict__ qcta,
                uint32_t* __restrict__ counts) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= NF) return;
    Face s;
    if (!face_setup(V, T, NV, f, W, H, s) || s.xhi < s.xlo || s.yhi < s.ylo) return;
    const long long area = (long long)(s.xhi - s.xlo + 1) * (s.yhi - s.ylo + 1);
    if (area > CR_CTA_AREA) { qcta[atomicAdd(counts + 1, 1u)] = (uint32_t)f; return; }
    if (area > CR_WARP_AREA) { qwarp[atomicAdd(counts, 1u)] = (uint32_t)f; return; }
    for (int px = s.xlo; px <= s.xhi; px++)
        for (int py = s.ylo; py <= s.yhi; py++) shade(s, f, px, py, W, D, trunc, zbuf);
}

// persistent grid: each warp drains faces of the warp queue; then the CTAs share the faces of the CTA queue.  With
// fewer such faces than CTAs (screen-filling triangles) each face gets gridDim.x / n CTAs, which split its box;
// otherwise each CTA takes whole faces in turn.  The split is decided on the device from the queue's length.
__global__ void __launch_bounds__(256)
cr_large_kernel(const float4* __restrict__ V, const int32_t* __restrict__ T, int NV, int H, int W, const float* __restrict__ D,
                float trunc, unsigned long long* __restrict__ zbuf, const uint32_t* __restrict__ qwarp,
                const uint32_t* __restrict__ qcta, const uint32_t* __restrict__ counts) {
    const uint32_t nwarp = counts[0], ncta = counts[1];
    const int lane = threadIdx.x & 31;
    const uint32_t warps = gridDim.x * (blockDim.x >> 5);
    for (uint32_t q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); q < nwarp; q += warps) {
        const int f = (int)qwarp[q];
        Face s;
        face_setup(V, T, NV, f, W, H, s);
        const int bw = s.xhi - s.xlo + 1, total = bw * (s.yhi - s.ylo + 1);
        for (int i = lane; i < total; i += 32) {
            const int r = i / bw;
            shade(s, f, s.xlo + i - r * bw, s.ylo + r, W, D, trunc, zbuf);
        }
    }
    if (ncta == 0) return;
    uint32_t q0 = blockIdx.x, qstep = gridDim.x, part = 0, parts = 1;
    if (ncta <= gridDim.x) {
        parts = gridDim.x / ncta;
        q0 = blockIdx.x % ncta; part = blockIdx.x / ncta; qstep = ncta;
        if (part >= parts) return;
    }
    for (uint32_t q = q0; q < ncta; q += qstep) {
        const int f = (int)qcta[q];
        Face s;
        face_setup(V, T, NV, f, W, H, s);
        const long long bw = s.xhi - s.xlo + 1, total = bw * (s.yhi - s.ylo + 1);
        const long long stride = (long long)parts * blockDim.x;
        for (long long i = (long long)part * blockDim.x + threadIdx.x; i < total; i += stride) {
            const long long r = i / bw;
            shade(s, f, s.xlo + (int)(i - r * bw), s.ylo + (int)r, W, D, trunc, zbuf);
        }
    }
}

// per pixel: the winner's id and its perspective-corrected barycentrics at the pixel centre
__global__ void __launch_bounds__(256)
cr_resolve_kernel(const float4* __restrict__ V, const int32_t* __restrict__ T, int NV, int H, int W,
                  const unsigned long long* __restrict__ zbuf, int32_t* __restrict__ findices, float* __restrict__ bary) {
    const int pix = blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= H * W) return;
    const unsigned long long id = zbuf[pix] % CR_MAXINT;
    float r0 = 0.f, r1 = 0.f, r2 = 0.f;
    int out = 0;
    if (id != CR_MAXINT - 1) {
        out = (int)id;
        const int f = out - 1;
        const float4 p0 = V[T[3 * f]], p1 = V[T[3 * f + 1]], p2 = V[T[3 * f + 2]];
        Face s;
        screen(p0, W, H, s.x0, s.y0, s.z0);
        screen(p1, W, H, s.x1, s.y1, s.z1);
        screen(p2, W, H, s.x2, s.y2, s.z2);
        s.area = (s.x2 - s.x0) * (s.y1 - s.y0) - (s.x1 - s.x0) * (s.y2 - s.y0);
        s.inv = (float)(1.0 / (double)s.area);
        const int py = pix / W, px = pix - py * W;
        barycentric(s, (float)px + 0.5f, (float)py + 0.5f, r0, r1, r2);
        r0 = r0 / p0.w; r1 = r1 / p1.w; r2 = r2 / p2.w;
        const float w = 1.0f / (r0 + r1 + r2);
        r0 *= w; r1 *= w; r2 *= w;
    }
    findices[pix] = out;
    bary[3 * (size_t)pix] = r0;
    bary[3 * (size_t)pix + 1] = r1;
    bary[3 * (size_t)pix + 2] = r2;
}

// ---- interpolate ---------------------------------------------------------------------------------------------------
// face of a pixel as the reference's `findices - 1 + (findices == 0)` then `.long()` computes it (in fp32 for fp32 ids),
// with torch's wrap of a negative index; -1 when out of range
template <typename IdT>
__device__ __forceinline__ long long face_of(const IdT* __restrict__ fid, int pix, int NF) {
    long long f;
    if constexpr (sizeof(IdT) == 4 && !std::is_integral<IdT>::value) {
        const float x = fid[pix];
        const float g = x - 1.0f + (x == 0.0f ? 1.0f : 0.0f);
        if (!(g > -9.2e18f && g < 9.2e18f)) return -1;
        f = (long long)g;
    } else {
        const long long x = fid[pix];
        f = x - 1 + (x == 0);
    }
    if (f < 0) f += NF;
    return (f >= 0 && f < NF) ? f : -1;
}

template <typename TriT>
__device__ __forceinline__ bool verts_of(const TriT* __restrict__ T, long long f, int NV, long long v[3]) {
    if (f < 0) return false;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        long long x = (long long)T[3 * f + k];
        if (x < 0) x += NV;
        if (x < 0 || x >= NV) return false;
        v[k] = x;
    }
    return true;
}

template <typename IdT, typename TriT>
__global__ void __launch_bounds__(256)
cr_interp_fwd_kernel(const float* __restrict__ col, int NV, int C, const IdT* __restrict__ fid, const float* __restrict__ bary,
                     const TriT* __restrict__ T, int NF, int npix, float* __restrict__ out) {
    const int pix = blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= npix) return;
    long long v[3];
    float* o = out + (size_t)pix * C;
    if (!verts_of(T, face_of(fid, pix, NF), NV, v)) {
        for (int c = 0; c < C; c++) o[c] = 0.0f;
        return;
    }
    const float b0 = bary[3 * (size_t)pix], b1 = bary[3 * (size_t)pix + 1], b2 = bary[3 * (size_t)pix + 2];
    const float *c0 = col + v[0] * C, *c1 = col + v[1] * C, *c2 = col + v[2] * C;
    // torch's CPU sum over the three corners: ((+0 + t0) + t1) + t2, so a sum of -0 terms is +0 there too
    for (int c = 0; c < C; c++) o[c] = 0.0f + b0 * c0[c] + b1 * c1[c] + b2 * c2[c];
}

// d bary[p,k] = sum_c g[p,c] col[v_k,c] (ascending c);  contrib[3p+k, c] = bary[p,k] g[p,c] for the deterministic
// scatter into d col, with its vertex in cidx (0 and a zero row for a pixel with an invalid face)
template <typename IdT, typename TriT>
__global__ void __launch_bounds__(256)
cr_interp_bwd_kernel(const float* __restrict__ col, int NV, int C, const IdT* __restrict__ fid, const float* __restrict__ bary,
                     const TriT* __restrict__ T, int NF, int npix, const float* __restrict__ g, float* __restrict__ dbary,
                     float* __restrict__ contrib, long long* __restrict__ cidx) {
    const int pix = blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= npix) return;
    long long v[3];
    const bool ok = verts_of(T, face_of(fid, pix, NF), NV, v);
    const float* gp = g + (size_t)pix * C;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const size_t row = 3 * (size_t)pix + k;
        if (dbary) {
            float acc = 0.0f;
            if (ok)
                for (int c = 0; c < C; c++) acc = acc + gp[c] * col[v[k] * C + c];
            dbary[row] = acc;
        }
        if (contrib) {
            const float b = bary[row];
            for (int c = 0; c < C; c++) contrib[row * C + c] = ok ? b * gp[c] : 0.0f;
            cidx[row] = ok ? v[k] : 0;
        }
    }
}

template <typename IdT, typename TriT>
void interp_launch(const float* col, int NV, int C, const void* fid, const float* bary, const void* tri, int NF, int npix,
                   const float* g, float* out, float* dbary, float* contrib, long long* cidx, cudaStream_t s) {
    const unsigned blocks = (unsigned)((npix + 255) / 256);
    if (g == nullptr)
        cr_interp_fwd_kernel<IdT, TriT><<<blocks, 256, 0, s>>>(col, NV, C, (const IdT*)fid, bary, (const TriT*)tri, NF, npix, out);
    else
        cr_interp_bwd_kernel<IdT, TriT><<<blocks, 256, 0, s>>>(col, NV, C, (const IdT*)fid, bary, (const TriT*)tri, NF, npix, g,
                                                               dbary, contrib, cidx);
}

}  // namespace

size_t cr_scratch_bytes(int F, int H, int W) { return (size_t)H * W * 8 + 256 + (size_t)F * 8; }

int cr_launch_rasterize(const float* V, int NV, const int32_t* T, int NF, const float* D, int H, int W, float trunc,
                        int32_t* findices, float* bary, void* scratch, cudaStream_t s) {
    const size_t npix = (size_t)H * W;
    unsigned long long* zbuf = (unsigned long long*)scratch;
    uint32_t* counts = (uint32_t*)((char*)scratch + npix * 8);
    uint32_t* qwarp = (uint32_t*)((char*)scratch + npix * 8 + 256);
    uint32_t* qcta = qwarp + NF;
    cr_init_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, s>>>(zbuf, npix, counts);
    if (NF > 0) {
        cr_small_kernel<<<(unsigned)((NF + 255) / 256), 256, 0, s>>>((const float4*)V, T, NV, NF, H, W, D, trunc, zbuf, qwarp, qcta, counts);
        cr_large_kernel<<<GS_NUM_SMS * 8, 256, 0, s>>>((const float4*)V, T, NV, H, W, D, trunc, zbuf, qwarp, qcta, counts);
        gs_count_launches(2);
    }
    cr_resolve_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, s>>>((const float4*)V, T, NV, H, W, zbuf, findices, bary);
    gs_count_launches(2);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int cr_launch_interpolate(const float* col, int NV, int C, const void* fid, int fid_f32, const float* bary, const void* tri,
                          int tri_i64, int NF, int npix, const float* g, float* out, float* dbary, float* contrib,
                          long long* cidx, cudaStream_t s) {
    if (npix == 0) return 0;
    if (fid_f32) {
        if (tri_i64) interp_launch<float, long long>(col, NV, C, fid, bary, tri, NF, npix, g, out, dbary, contrib, cidx, s);
        else interp_launch<float, int32_t>(col, NV, C, fid, bary, tri, NF, npix, g, out, dbary, contrib, cidx, s);
    } else {
        if (tri_i64) interp_launch<int32_t, long long>(col, NV, C, fid, bary, tri, NF, npix, g, out, dbary, contrib, cidx, s);
        else interp_launch<int32_t, int32_t>(col, NV, C, fid, bary, tri, NF, npix, g, out, dbary, contrib, cidx, s);
    }
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
