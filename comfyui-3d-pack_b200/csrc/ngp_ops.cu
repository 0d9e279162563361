// Instant-NGP path kernels: multiresolution hash-grid encode (+ backward, + TV gradient), occupancy-grid
// ray marching, packed volume-rendering weights and per-ray accumulation.
//
// Replace kiui.gridencoder (torch-ngp) and nerfacc for Instant_NGP.py:101-156,195 (SURVEY.md App. A.3-A.4).
// Bounds: encode / scatter are random gathers / reds into the two hash tables (<= 2 x 12 levels x 4 MiB, close
// to the 50 MB L2 of an H100); marching is ALU-bound on a 32 KB bit grid held in shared memory;
// weights / accumulate stream the packed samples once.
// fp32 operation order of everything that decides an INTEGER output (corner indices, the packed sample list)
// is pinned with __fmul_rn/__fadd_rn/__fdiv_rn to match oracle/ngp_oracle.py bit for bit.
#include "gs_common.cuh"

namespace {

constexpr uint32_t PRIME1 = 2654435761u, PRIME2 = 805459861u;
constexpr int NGP_MAX_LEVELS = 32;

struct GridMeta { float scale[NGP_MAX_LEVELS]; int res[NGP_MAX_LEVELS]; int off[NGP_MAX_LEVELS + 1]; int L; float bound; };

__device__ __forceinline__ uint32_t grid_index(uint32_t gx, uint32_t gy, uint32_t gz, int res, uint32_t hsize) {
    const unsigned long long r1 = (unsigned long long)(res + 1);
    if (r1 * r1 * r1 <= (unsigned long long)hsize) return (gx + gy * (uint32_t)r1 + gz * (uint32_t)(r1 * r1)) % hsize;
    return (gx ^ (gy * PRIME1) ^ (gz * PRIME2)) % hsize;
}

__device__ __forceinline__ void cell_of(const float* __restrict__ x, long long n, const GridMeta& gm, int l, uint32_t pg[3],
                                        float fr[3]) {
    const float two_b = __fmul_rn(2.0f, gm.bound);
#pragma unroll
    for (int d = 0; d < 3; d++) {
        const float x01 = __fdiv_rn(__fadd_rn(x[3 * n + d], gm.bound), two_b);
        const float pos = __fadd_rn(__fmul_rn(x01, gm.scale[l]), 0.5f);
        const float fl = floorf(pos);
        fr[d] = pos - fl;
        pg[d] = (uint32_t)(int)fl;
    }
}

// thread = (sample n, level l); adjacent threads = adjacent levels of one sample -> coalesced [N, 2L] rows
__global__ void __launch_bounds__(256)
grid_encode_fwd_kernel(const float* __restrict__ x, long long N, const float2* __restrict__ emb, GridMeta gm,
                       float2* __restrict__ out) {
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= N * gm.L) return;
    const long long n = gid / gm.L; const int l = (int)(gid - n * gm.L);
    uint32_t pg[3]; float fr[3];
    cell_of(x, n, gm, l, pg, fr);
    const uint32_t hsize = (uint32_t)(gm.off[l + 1] - gm.off[l]);
    const float2* table = emb + gm.off[l];
    float2 acc = make_float2(0.f, 0.f);
    // (pairing the two x-neighbours into one 128-bit load, as the backward does for its reds, was measured neutral:
    // 5.76 -> 5.92 ms on ray-ordered samples, 7.30 -> 6.38 ms on random ones; the gather is L1-wavefront bound)
#pragma unroll
    for (int c = 0; c < 8; c++) {
        const uint32_t bx = c & 1, by = (c >> 1) & 1, bz = (c >> 2) & 1;
        const float w = (bx ? fr[0] : 1.f - fr[0]) * (by ? fr[1] : 1.f - fr[1]) * (bz ? fr[2] : 1.f - fr[2]);
        const float2 v = __ldg(table + grid_index(pg[0] + bx, pg[1] + by, pg[2] + bz, gm.res[l], hsize));
        acc.x += w * v.x; acc.y += w * v.y;
    }
    out[gid] = acc;
}

// V4: the two x-neighbours of a corner pair sit in ONE 16-byte-aligned float4 whenever their indices differ only in
// bit 0 (always for even cell x in the hashed levels: (x+1)^h == (x^h)^1 and the table size is a power of two; for
// even linear indices in the dense levels) -> one red.global.add.v4.f32 instead of two .v2 (L2 atomic units are
// the bound of this kernel: profiles/r1_ngp_kernels.txt).
// one x-neighbour corner pair (values a = corner x, b = corner x+1) -> one .v4 red or two .v2 reds
template <bool V4>
__device__ __forceinline__ void red_pair(float2* __restrict__ table, uint32_t i0, uint32_t i1, float2 a, float2 b) {
    if (V4 && (i0 ^ i1) == 1u) {
        const bool lo0 = (i0 & 1u) == 0u;                  // which of the two is the even (lower) entry
        const float2 lo = lo0 ? a : b, hi = lo0 ? b : a;
        atomicAdd(reinterpret_cast<float4*>(table + (i0 & ~1u)), make_float4(lo.x, lo.y, hi.x, hi.y));
    } else {
        atomicAdd(table + i0, a);                          // red.global.add.v2.f32
        atomicAdd(table + i1, b);
    }
}

// levels [l0, L): thread = (sample, level), adjacent threads = adjacent levels of one sample
template <bool V4>
__global__ void __launch_bounds__(256)
grid_encode_bwd_kernel(const float* __restrict__ x, long long N, GridMeta gm, int l0, const float2* __restrict__ g_out,
                       float2* __restrict__ d_emb) {
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int nl = gm.L - l0;
    if (gid >= N * nl) return;
    const long long n = gid / nl; const int l = l0 + (int)(gid - n * nl);
    const float2 g = g_out[n * gm.L + l];
    if (g.x == 0.f && g.y == 0.f) return;
    uint32_t pg[3]; float fr[3];
    cell_of(x, n, gm, l, pg, fr);
    const uint32_t hsize = (uint32_t)(gm.off[l + 1] - gm.off[l]);
    float2* table = d_emb + gm.off[l];
#pragma unroll
    for (int c = 0; c < 4; c++) {
        const uint32_t by = c & 1, bz = (c >> 1) & 1;
        const float wyz = (by ? fr[1] : 1.f - fr[1]) * (bz ? fr[2] : 1.f - fr[2]);
        const float w0 = (1.f - fr[0]) * wyz, w1 = fr[0] * wyz;
        const uint32_t i0 = grid_index(pg[0], pg[1] + by, pg[2] + bz, gm.res[l], hsize);
        const uint32_t i1 = grid_index(pg[0] + 1, pg[1] + by, pg[2] + bz, gm.res[l], hsize);
        red_pair<V4>(table, i0, i1, make_float2(w0 * g.x, w0 * g.y), make_float2(w1 * g.x, w1 * g.y));
    }
}

// Coarse levels [0, l0) (cell much larger than the marching step): consecutive samples of a ray fall into the SAME cell
// for long runs (25 samples at resolution 16 with dt = 5e-3), i.e. hit the same 8 table entries.  Here a warp takes
// 32 consecutive samples of ONE level, sums the 16 corner contributions over each run of equal cells with a segmented
// shuffle reduction, and only the head lane of a run issues the reds: the kernel is bound by L2 atomic operations
// (profiles/r1_ngp_kernels.txt), the shuffles ride in otherwise idle issue slots.
template <bool V4>
__global__ void __launch_bounds__(256)
grid_encode_bwd_runs_kernel(const float* __restrict__ x, long long N, GridMeta gm, const float2* __restrict__ g_out,
                            float2* __restrict__ d_emb) {
    const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int l = blockIdx.y, lane = threadIdx.x & 31;
    const bool live = n < N;
    float2 g = make_float2(0.f, 0.f);
    uint32_t pg[3] = {0u, 0u, 0u}; float fr[3] = {0.f, 0.f, 0.f};
    if (live) { g = g_out[n * gm.L + l]; cell_of(x, n, gm, l, pg, fr); }
    const uint32_t key = live ? (pg[0] | (pg[1] << 10) | (pg[2] << 20)) : 0xFFFFFFFFu;      // res + 1 <= 1024 here
    float vx[8], vy[8];
#pragma unroll
    for (int c = 0; c < 8; c++) {
        const uint32_t bx = c & 1, by = (c >> 1) & 1, bz = (c >> 2) & 1;
        const float w = (bx ? fr[0] : 1.f - fr[0]) * ((by ? fr[1] : 1.f - fr[1]) * (bz ? fr[2] : 1.f - fr[2]));
        vx[c] = w * g.x; vy[c] = w * g.y;
    }
    const uint32_t prev = __shfl_up_sync(0xFFFFFFFFu, key, 1);
    const bool head = (lane == 0) || (key != prev);
    const uint32_t heads = __ballot_sync(0xFFFFFFFFu, head);
    const int run = __popc(heads & (0xFFFFFFFFu >> (31 - lane)));
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const int orun = __shfl_down_sync(0xFFFFFFFFu, run, off);
        const bool take = (lane + off < 32) && (orun == run);
#pragma unroll
        for (int c = 0; c < 8; c++) {
            const float ox = __shfl_down_sync(0xFFFFFFFFu, vx[c], off), oy = __shfl_down_sync(0xFFFFFFFFu, vy[c], off);
            if (take) { vx[c] += ox; vy[c] += oy; }
        }
    }
    if (!head || !live) return;
    bool any = false;
#pragma unroll
    for (int c = 0; c < 8; c++) any = any || (vx[c] != 0.f) || (vy[c] != 0.f);
    if (!any) return;
    const uint32_t hsize = (uint32_t)(gm.off[l + 1] - gm.off[l]);
    float2* table = d_emb + gm.off[l];
#pragma unroll
    for (int c = 0; c < 4; c++) {
        const uint32_t by = c & 1, bz = (c >> 1) & 1;
        const uint32_t i0 = grid_index(pg[0], pg[1] + by, pg[2] + bz, gm.res[l], hsize);
        const uint32_t i1 = grid_index(pg[0] + 1, pg[1] + by, pg[2] + bz, gm.res[l], hsize);
        red_pair<V4>(table, i0, i1, make_float2(vx[2 * c], vy[2 * c]), make_float2(vx[2 * c + 1], vy[2 * c + 1]));
    }
}

__device__ __forceinline__ float sgn(float v) { return (v > 0.f) ? 1.f : ((v < 0.f) ? -1.f : 0.f); }

__global__ void __launch_bounds__(256)
grid_tv_kernel(const float* __restrict__ x, long long N, const float2* __restrict__ emb, GridMeta gm, float weight,
               float2* __restrict__ d_emb) {
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= N * gm.L) return;
    const long long n = gid / gm.L; const int l = (int)(gid - n * gm.L);
    uint32_t pg[3]; float fr[3];
    cell_of(x, n, gm, l, pg, fr);
    const int res = gm.res[l];
    const uint32_t hsize = (uint32_t)(gm.off[l + 1] - gm.off[l]);
    const float2* table = emb + gm.off[l];
    const uint32_t ci = grid_index(pg[0], pg[1], pg[2], res, hsize);
    const float2 cur = __ldg(table + ci);
    float2 acc = make_float2(0.f, 0.f);
#pragma unroll
    for (int d = 0; d < 3; d++) {
#pragma unroll
        for (int s = -1; s <= 1; s += 2) {
            const int q = (int)pg[d] + s;
            if (q < 0 || q > res) continue;
            uint32_t g3[3] = {pg[0], pg[1], pg[2]};
            g3[d] = (uint32_t)q;
            const float2 nb = __ldg(table + grid_index(g3[0], g3[1], g3[2], res, hsize));
            acc.x += sgn(cur.x - nb.x); acc.y += sgn(cur.y - nb.y);
        }
    }
    atomicAdd(d_emb + gm.off[l] + ci, make_float2(weight * acc.x, weight * acc.y));
}

// ------------------------------------------------------------------------------------------------ marching
__global__ void __launch_bounds__(256) pack_bits_kernel(const uint8_t* __restrict__ binary, int n, uint32_t* __restrict__ bits) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;           // one 32-bit word per thread
    if (i * 32 >= n) return;
    uint32_t w = 0;
    for (int b = 0; b < 32; b++) { const int j = i * 32 + b; if (j < n && binary[j]) w |= 1u << b; }
    bits[i] = w;
}

struct MarchArgs { float lo[3], hi[3], near_plane, far_plane, dt; int R; };

template <bool WRITE>
__global__ void __launch_bounds__(256)
march_kernel(const float* __restrict__ rays_o, const float* __restrict__ rays_d, long long n_rays,
             const uint32_t* __restrict__ bits, MarchArgs ma, const float* __restrict__ t_offset,
             uint32_t* __restrict__ counts, const uint32_t* __restrict__ offsets, long long* __restrict__ ray_indices,
             float* __restrict__ t_starts, float* __restrict__ t_ends) {
    extern __shared__ uint32_t s_bits[];
    const int nwords = (ma.R * ma.R * ma.R + 31) / 32;
    for (int i = threadIdx.x; i < nwords; i += blockDim.x) s_bits[i] = bits[i];
    __syncthreads();
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rays) return;
    const float o[3] = {rays_o[3 * r], rays_o[3 * r + 1], rays_o[3 * r + 2]};
    const float d[3] = {rays_d[3 * r], rays_d[3 * r + 1], rays_d[3 * r + 2]};
    float tmin = -3.0e38f, tmax = 3.0e38f;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const float inv = __fdiv_rn(1.0f, d[a]);
        const float t0 = __fmul_rn(__fsub_rn(ma.lo[a], o[a]), inv), t1 = __fmul_rn(__fsub_rn(ma.hi[a], o[a]), inv);
        tmin = fmaxf(tmin, fminf(t0, t1)); tmax = fminf(tmax, fmaxf(t0, t1));
    }
    float t_enter = fmaxf(tmin, ma.near_plane);
    const float t_exit = fminf(tmax, ma.far_plane);
    if (t_offset) t_enter = __fadd_rn(t_enter, t_offset[r]);
    uint32_t cnt = 0;
    uint32_t wpos = WRITE ? offsets[r] : 0;
    if (t_exit > t_enter) {
        const float Rf = (float)ma.R;
        const float ext[3] = {__fsub_rn(ma.hi[0], ma.lo[0]), __fsub_rn(ma.hi[1], ma.lo[1]), __fsub_rn(ma.hi[2], ma.lo[2])};
        for (int k = 0;; k++) {
            const float ts = __fadd_rn(t_enter, __fmul_rn((float)k, ma.dt));
            const float te = __fadd_rn(t_enter, __fmul_rn(__fadd_rn((float)k, 1.0f), ma.dt));
            const float tm = __fmul_rn(__fadd_rn(ts, te), 0.5f);
            if (!(tm < t_exit)) break;
            int c3[3]; bool inb = true;
#pragma unroll
            for (int a = 0; a < 3; a++) {
                const float p = __fadd_rn(o[a], __fmul_rn(d[a], tm));
                const float f = floorf(__fmul_rn(__fdiv_rn(__fsub_rn(p, ma.lo[a]), ext[a]), Rf));
                inb = inb && (f >= 0.f) && (f < Rf);
                c3[a] = (int)f;
            }
            if (!inb) continue;
            const int cell = (c3[0] * ma.R + c3[1]) * ma.R + c3[2];        // binary[x][y][z]
            if (!((s_bits[cell >> 5] >> (cell & 31)) & 1u)) continue;
            if (WRITE) { ray_indices[wpos] = r; t_starts[wpos] = ts; t_ends[wpos] = te; wpos++; }
            cnt++;
        }
    }
    if (!WRITE) counts[r] = cnt;
}

// ------------------------------------------------------------------------------------------------ packed rendering
__global__ void __launch_bounds__(256)
ray_ranges_kernel(const long long* __restrict__ ri, long long S, int32_t* __restrict__ ranges) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= S) return;
    const long long r = ri[i];
    if (i == 0 || ri[i - 1] != r) ranges[2 * r] = (int32_t)i;       // counts: second kernel (needs every start written)
}
__global__ void __launch_bounds__(256)
ray_counts_kernel(const long long* __restrict__ ri, long long S, int32_t* __restrict__ ranges) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= S) return;
    const long long r = ri[i];
    if (i == S - 1 || ri[i + 1] != r) ranges[2 * r + 1] = (int32_t)(i + 1) - ranges[2 * r];
}

__global__ void __launch_bounds__(128)
weights_fwd_kernel(const float* __restrict__ ts, const float* __restrict__ te, const float* __restrict__ sig,
                   const int32_t* __restrict__ ranges, long long n_rays, float* __restrict__ w, float* __restrict__ tr,
                   float* __restrict__ al) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rays) return;
    const int s = ranges[2 * r], c = ranges[2 * r + 1];
    float T = 1.f;
    for (int i = s; i < s + c; i++) {
        const float a = 1.f - __expf(-sig[i] * (te[i] - ts[i]));
        w[i] = T * a; tr[i] = T; al[i] = a;
        T *= 1.f - a;
    }
}

__global__ void __launch_bounds__(128)
weights_bwd_kernel(const float* __restrict__ ts, const float* __restrict__ te, const int32_t* __restrict__ ranges,
                   long long n_rays, const float* __restrict__ tr, const float* __restrict__ al,
                   const float* __restrict__ gw, const float* __restrict__ gt, const float* __restrict__ ga,
                   float* __restrict__ dsig) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rays) return;
    const int s = ranges[2 * r], c = ranges[2 * r + 1];
    float G = 0.f;                                           // dL/dT_{i+1}
    for (int i = s + c - 1; i >= s; i--) {
        const float T = tr[i], a = al[i];
        const float gwi = gw ? gw[i] : 0.f, gti = gt ? gt[i] : 0.f, gai = ga ? ga[i] : 0.f;
        const float dalpha = gwi * T + gai - G * T;
        G = gti + gwi * a + G * (1.f - a);
        dsig[i] = dalpha * (1.f - a) * (te[i] - ts[i]);
    }
}

__global__ void __launch_bounds__(128)
accumulate_fwd_kernel(const float* __restrict__ w, const float* __restrict__ v, int C, const int32_t* __restrict__ ranges,
                      long long n_rays, float* __restrict__ out) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rays) return;
    const int s = ranges[2 * r], c = ranges[2 * r + 1];
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int i = s; i < s + c; i++) {
        const float wi = w[i];
        if (v == nullptr) acc[0] += wi;
        else for (int k = 0; k < C; k++) acc[k] += wi * v[(size_t)i * C + k];
    }
    for (int k = 0; k < C; k++) out[r * C + k] = acc[k];
}

__global__ void __launch_bounds__(256)
accumulate_bwd_kernel(const float* __restrict__ w, const float* __restrict__ v, int C, const long long* __restrict__ ri,
                      long long S, const float* __restrict__ g_out, float* __restrict__ dw, float* __restrict__ dv) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= S) return;
    const long long r = ri[i];
    float g = 0.f;
    if (v == nullptr) g = g_out[r];
    else for (int k = 0; k < C; k++) { const float go = g_out[r * C + k]; g += go * v[i * C + k]; if (dv) dv[i * C + k] = w[i] * go; }
    dw[i] = g;
}

int make_meta(GridMeta& gm, const int32_t* offsets_host, int L, float bound, float pls, int base) {
    if (L <= 0 || L > NGP_MAX_LEVELS) { gs_set_error("grid: num_levels must be 1..%d", NGP_MAX_LEVELS); return 1; }
    gm.L = L; gm.bound = bound;
    const float S = log2f(pls);
    for (int l = 0; l < L; l++) {
        gm.scale[l] = exp2f((float)l * S) * (float)base - 1.0f;
        gm.res[l] = (int)ceilf(gm.scale[l]) + 1;
        gm.off[l] = offsets_host[l];
    }
    gm.off[L] = offsets_host[L];
    return 0;
}

}  // namespace

#define NGP_GRID(n) (unsigned)(((n) + 255) / 256), 256

int ngp_grid_encode_fwd(const float* x, long long N, const float* emb, const int32_t* offsets_host, int L, float bound,
                        float pls, int base, float* out, cudaStream_t s) {
    if (N <= 0) return 0;
    GridMeta gm; if (make_meta(gm, offsets_host, L, bound, pls, base)) return 1;
    grid_encode_fwd_kernel<<<NGP_GRID(N * L), 0, s>>>(x, N, (const float2*)emb, gm, (float2*)out);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
int ngp_grid_encode_bwd(const float* x, long long N, const int32_t* offsets_host, int L, float bound, float pls, int base,
                        const float* g_out, float* d_emb, cudaStream_t s) {
    if (N <= 0) return 0;
    GridMeta gm; if (make_meta(gm, offsets_host, L, bound, pls, base)) return 1;
    static const bool v4env = []() { const char* e = getenv("NGP_B200_RED_V4"); return !(e && e[0] == '0'); }();
    static const bool runs = []() { const char* e = getenv("NGP_B200_BWD_RUNS"); return !(e && e[0] == '0'); }();
    const bool v4 = v4env && ((uintptr_t)d_emb & 15) == 0;
    // coarse levels (resolution <= 128: runs of >= ~3 samples per cell at the reference's 5e-3 step) go through the
    // run-reducing kernel; they are the first levels since resolutions grow with the level index
    int l0 = 0;
    if (runs) while (l0 < L && gm.res[l0] <= 128 && l0 < 8) l0++;
    if (l0 > 0) {
        const dim3 grid((unsigned)((N + 255) / 256), (unsigned)l0);
        if (v4) grid_encode_bwd_runs_kernel<true><<<grid, 256, 0, s>>>(x, N, gm, (const float2*)g_out, (float2*)d_emb);
        else grid_encode_bwd_runs_kernel<false><<<grid, 256, 0, s>>>(x, N, gm, (const float2*)g_out, (float2*)d_emb);
    }
    if (l0 < L) {
        if (v4) grid_encode_bwd_kernel<true><<<NGP_GRID(N * (L - l0)), 0, s>>>(x, N, gm, l0, (const float2*)g_out, (float2*)d_emb);
        else grid_encode_bwd_kernel<false><<<NGP_GRID(N * (L - l0)), 0, s>>>(x, N, gm, l0, (const float2*)g_out, (float2*)d_emb);
    }
    gs_count_launches((l0 > 0) + (l0 < L));
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
int ngp_grid_tv(const float* x, long long N, const float* emb, const int32_t* offsets_host, int L, float bound, float pls,
                int base, float weight, float* d_emb, cudaStream_t s) {
    if (N <= 0) return 0;
    GridMeta gm; if (make_meta(gm, offsets_host, L, bound, pls, base)) return 1;
    grid_tv_kernel<<<NGP_GRID(N * L), 0, s>>>(x, N, (const float2*)emb, gm, weight, (float2*)d_emb);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

size_t ngp_march_scratch_bytes(long long n_rays, int R) {
    return (((size_t)R * R * R + 31) / 32) * 4 + 256 + gs_scan_scratch_bytes(n_rays);
}

static MarchArgs make_march(const float* aabb, float near_plane, float far_plane, float dt, int R) {
    MarchArgs ma;
    for (int a = 0; a < 3; a++) { ma.lo[a] = aabb[a]; ma.hi[a] = aabb[3 + a]; }
    ma.near_plane = near_plane; ma.far_plane = far_plane; ma.dt = dt; ma.R = R;
    return ma;
}

int ngp_march_count(const float* rays_o, const float* rays_d, long long n_rays, const uint8_t* binary, int R,
                    const float* aabb, float near_plane, float far_plane, float dt, const float* t_offset, uint32_t* counts,
                    uint32_t* offsets, unsigned long long* total_dev, void* scratch, cudaStream_t s) {
    const int ncell = R * R * R, nwords = (ncell + 31) / 32;
    if ((size_t)nwords * 4 > 200 * 1024) { gs_set_error("march: occupancy grid %d^3 does not fit shared memory", R); return 1; }
    uint32_t* bits = (uint32_t*)scratch;
    void* scan_scratch = (char*)scratch + (((size_t)nwords * 4 + 255) & ~(size_t)255);
    pack_bits_kernel<<<NGP_GRID(nwords), 0, s>>>(binary, ncell, bits);
    if (n_rays > 0) {
        const size_t smem = (size_t)nwords * 4;
        if (smem > 48 * 1024) GS_CUDA_CHECK(cudaFuncSetAttribute(march_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        march_kernel<false><<<NGP_GRID(n_rays), smem, s>>>(rays_o, rays_d, n_rays, bits, make_march(aabb, near_plane, far_plane, dt, R),
                                                           t_offset, counts, nullptr, nullptr, nullptr, nullptr);
    }
    gs_count_launches(2);
    if (gs_scan_gather_u32(counts, nullptr, offsets, total_dev, n_rays, scan_scratch, s)) return 1;
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int ngp_march_write(const float* rays_o, const float* rays_d, long long n_rays, int R, const float* aabb, float near_plane,
                    float far_plane, float dt, const float* t_offset, const uint32_t* offsets, long long* ray_indices,
                    float* t_starts, float* t_ends, void* scratch, cudaStream_t s) {
    if (n_rays <= 0) return 0;
    const int nwords = (R * R * R + 31) / 32;
    const size_t smem = (size_t)nwords * 4;
    if (smem > 48 * 1024) GS_CUDA_CHECK(cudaFuncSetAttribute(march_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    march_kernel<true><<<NGP_GRID(n_rays), smem, s>>>(rays_o, rays_d, n_rays, (const uint32_t*)scratch,
                                                      make_march(aabb, near_plane, far_plane, dt, R), t_offset, nullptr, offsets,
                                                      ray_indices, t_starts, t_ends);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int ngp_ray_ranges(const long long* ri, long long S, long long n_rays, int32_t* ranges, cudaStream_t s) {
    GS_CUDA_CHECK(cudaMemsetAsync(ranges, 0, (size_t)n_rays * 8, s));
    if (S <= 0) return 0;
    ray_ranges_kernel<<<NGP_GRID(S), 0, s>>>(ri, S, ranges);
    ray_counts_kernel<<<NGP_GRID(S), 0, s>>>(ri, S, ranges);
    gs_count_launches(2);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
int ngp_weights_fwd(const float* ts, const float* te, const float* sig, const int32_t* ranges, long long n_rays, float* w,
                    float* tr, float* al, cudaStream_t s) {
    if (n_rays <= 0) return 0;
    weights_fwd_kernel<<<(unsigned)((n_rays + 127) / 128), 128, 0, s>>>(ts, te, sig, ranges, n_rays, w, tr, al);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
int ngp_weights_bwd(const float* ts, const float* te, const int32_t* ranges, long long n_rays, const float* tr, const float* al,
                    const float* gw, const float* gt, const float* ga, float* dsig, cudaStream_t s) {
    if (n_rays <= 0) return 0;
    weights_bwd_kernel<<<(unsigned)((n_rays + 127) / 128), 128, 0, s>>>(ts, te, ranges, n_rays, tr, al, gw, gt, ga, dsig);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
int ngp_accumulate_fwd(const float* w, const float* v, int C, const int32_t* ranges, long long n_rays, float* out, cudaStream_t s) {
    if (n_rays <= 0) return 0;
    if (C < 1 || C > 4) { gs_set_error("accumulate: 1..4 channels supported, got %d", C); return 1; }
    accumulate_fwd_kernel<<<(unsigned)((n_rays + 127) / 128), 128, 0, s>>>(w, v, C, ranges, n_rays, out);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
int ngp_accumulate_bwd(const float* w, const float* v, int C, const long long* ri, long long S, const float* g_out, float* dw,
                       float* dv, cudaStream_t s) {
    if (S <= 0) return 0;
    accumulate_bwd_kernel<<<NGP_GRID(S), 0, s>>>(w, v, C, ri, S, g_out, dw, dv);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
