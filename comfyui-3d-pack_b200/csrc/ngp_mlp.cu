// Fused two-layer MLP (Linear -> ReLU -> Linear, no bias) for the tiny per-sample networks of the Instant-NGP
// path: kiui.nn.MLP(dim_in, dim_out, 32, 2, bias=False) at Instant_NGP.py:34-35,73,80.
//
// With ~50 M samples per 1080p frame the [N,32] hidden activations are 6.6 GB each; a library-GEMM MLP writes
// and re-reads them several times per step.  Here one thread owns one sample: the input row is read once
// (128 B), the hidden layer lives in registers, weights are broadcast from shared memory (LDS.128), only the
// [N,dim_out] result is written.  The backward recomputes the hidden layer instead of loading it, produces
// dL/dx in the same pass, and reduces the weight gradients per CTA in shared memory (persistent CTAs, one set of
// global atomics per CTA at the end).  fp32 SIMT on purpose: the reference runs these MLPs in fp32 and the cost is
// ~3 kFMA/sample — far below the hash-grid gather/scatter around it, so tensor cores would not move the step time.
#include "gs_common.cuh"

namespace {

constexpr int MT = 128;            // threads per CTA == samples per tile

struct MlpDims { int Din, H, Dout; };

// shared layout: W1t[Din][H] (input-major: the k-loop reads 4 hidden weights per LDS.128), W1[H][Din], W2[Dout][H]
__device__ __forceinline__ void load_weights(const float* __restrict__ W1, const float* __restrict__ W2, MlpDims d,
                                             float* sW1t, float* sW1, float* sW2) {
    for (int i = threadIdx.x; i < d.H * d.Din; i += blockDim.x) {
        const int k = i / d.Din, j = i - k * d.Din;
        const float w = __ldg(W1 + i);
        sW1[i] = w; sW1t[j * d.H + k] = w;
    }
    for (int i = threadIdx.x; i < d.Dout * d.H; i += blockDim.x) sW2[i] = __ldg(W2 + i);
}

// cooperative, fully coalesced load of a tile of MT rows [MT][DIN] into padded shared memory [MT][DIN+1]
template <int DIN>
__device__ __forceinline__ void load_tile(const float* __restrict__ X, long long n0, long long N, float* sX) {
    const long long rows = (N - n0 < MT) ? (N - n0) : MT;
    const int tot = (int)rows * DIN;
    const float4* src = reinterpret_cast<const float4*>(X + n0 * DIN);
    for (int i = threadIdx.x; i < (tot >> 2); i += MT) {
        const float4 v = __ldg(src + i);
        const int e = 4 * i, r = e / DIN, c = e - r * DIN;            // DIN % 4 == 0: a float4 never straddles rows
        float* d = sX + r * (DIN + 1) + c;
        d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
    }
    for (int i = tot + threadIdx.x; i < MT * DIN; i += MT) { const int r = i / DIN, c = i - r * DIN; sX[r * (DIN + 1) + c] = 0.f; }
}

// h = W1 x, x read from this thread's shared-memory row
template <int DIN, int H>
__device__ __forceinline__ void hidden_of(const float* sXrow, const float* sW1t, float (&h)[H]) {
#pragma unroll
    for (int k = 0; k < H; k++) h[k] = 0.f;
#pragma unroll
    for (int j = 0; j < DIN; j++) {
        const float xj = sXrow[j];
#pragma unroll
        for (int k = 0; k < H; k += 4) {
            const float4 w = *reinterpret_cast<const float4*>(sW1t + j * H + k);
            h[k] = fmaf(w.x, xj, h[k]); h[k + 1] = fmaf(w.y, xj, h[k + 1]);
            h[k + 2] = fmaf(w.z, xj, h[k + 2]); h[k + 3] = fmaf(w.w, xj, h[k + 3]);
        }
    }
}

template <int DIN, int H, int DOUT>
__global__ void __launch_bounds__(MT, 4)
mlp2_fwd_kernel(const float* __restrict__ X, long long N, const float* __restrict__ W1, const float* __restrict__ W2,
                float* __restrict__ Y) {
    extern __shared__ __align__(16) float smem[];
    float* sW1t = smem; float* sW1 = sW1t + DIN * H; float* sW2 = sW1 + DIN * H;
    float* sX = sW2 + 4 * H;                       // [MT][DIN+1]
    MlpDims d{DIN, H, DOUT};
    load_weights(W1, W2, d, sW1t, sW1, sW2);
    const long long n0 = (long long)blockIdx.x * MT;                 // one tile per CTA
    load_tile<DIN>(X, n0, N, sX);
    __syncthreads();
    const long long n = n0 + threadIdx.x;
    if (n >= N) return;
    float h[H];
    hidden_of<DIN, H>(sX + threadIdx.x * (DIN + 1), sW1t, h);
#pragma unroll
    for (int o = 0; o < DOUT; o++) {
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < H; k += 4) {
            const float4 w = *reinterpret_cast<const float4*>(sW2 + o * H + k);
            acc = fmaf(w.x, fmaxf(h[k], 0.f), acc); acc = fmaf(w.y, fmaxf(h[k + 1], 0.f), acc);
            acc = fmaf(w.z, fmaxf(h[k + 2], 0.f), acc); acc = fmaf(w.w, fmaxf(h[k + 3], 0.f), acc);
        }
        Y[n * DOUT + o] = acc;
    }
}

template <int DIN, int H, int DOUT>
__global__ void __launch_bounds__(MT, 3)
mlp2_bwd_kernel(const float* __restrict__ X, long long N, const float* __restrict__ W1, const float* __restrict__ W2,
                const float* __restrict__ GY, float* __restrict__ GX, float* __restrict__ GW1, float* __restrict__ GW2) {
    extern __shared__ __align__(16) float smem[];
    float* sW1t = smem; float* sW1 = sW1t + DIN * H; float* sW2 = sW1 + DIN * H;
    float* sX = sW2 + 4 * H;                       // [MT][DIN+1]
    float* sGH = sX + MT * (DIN + 1);              // [MT][H+1]
    float* sA = sGH + MT * (H + 1);                // [MT][H+1]   relu(h)
    float* sGY = sA + MT * (H + 1);                // [MT][4]
    MlpDims d{DIN, H, DOUT};
    load_weights(W1, W2, d, sW1t, sW1, sW2);
    constexpr int PER = (DIN * H) / MT;            // gW1 outputs per thread (6 or 8), contiguous in j for one k
    static_assert((DIN * H) % MT == 0 && DIN % PER == 0, "weight-gradient partition");
    float acc1[PER];
#pragma unroll
    for (int i = 0; i < PER; i++) acc1[i] = 0.f;
    float acc2 = 0.f;                              // gW2: one output per thread (t < DOUT*H <= MT)
    __syncthreads();
    const long long tiles = (N + MT - 1) / MT;
    float* myX = sX + threadIdx.x * (DIN + 1);
    float* myGH = sGH + threadIdx.x * (H + 1);
    float* myA = sA + threadIdx.x * (H + 1);
    for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const long long n = tile * MT + threadIdx.x;
        const bool live = n < N;
        load_tile<DIN>(X, tile * MT, N, sX);       // rows past N are zero-filled
        __syncthreads();
        float h[H];                                // becomes gh in place
        hidden_of<DIN, H>(myX, sW1t, h);
        float gy[DOUT];
#pragma unroll
        for (int o = 0; o < DOUT; o++) { gy[o] = live ? GY[n * DOUT + o] : 0.f; sGY[threadIdx.x * 4 + o] = gy[o]; }
#pragma unroll
        for (int k = 0; k < H; k++) {
            float g = 0.f;
#pragma unroll
            for (int o = 0; o < DOUT; o++) g = fmaf(sW2[o * H + k], gy[o], g);
            myA[k] = fmaxf(h[k], 0.f);
            h[k] = (h[k] > 0.f) ? g : 0.f;
            myGH[k] = h[k];
        }
        if (live && GX != nullptr) {
            // dL/dx[j] = sum_k W1[k][j] gh[k], 8 columns at a time to bound live registers
#pragma unroll
            for (int j0 = 0; j0 < DIN; j0 += 8) {
                float gx[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int k = 0; k < H; k++) {
                    const float g = h[k];
                    const float4 wa = *reinterpret_cast<const float4*>(sW1 + k * DIN + j0);
                    const float4 wb = *reinterpret_cast<const float4*>(sW1 + k * DIN + j0 + 4);
                    gx[0] = fmaf(wa.x, g, gx[0]); gx[1] = fmaf(wa.y, g, gx[1]); gx[2] = fmaf(wa.z, g, gx[2]); gx[3] = fmaf(wa.w, g, gx[3]);
                    gx[4] = fmaf(wb.x, g, gx[4]); gx[5] = fmaf(wb.y, g, gx[5]); gx[6] = fmaf(wb.z, g, gx[6]); gx[7] = fmaf(wb.w, g, gx[7]);
                }
                *reinterpret_cast<float4*>(GX + n * DIN + j0) = make_float4(gx[0], gx[1], gx[2], gx[3]);
                *reinterpret_cast<float4*>(GX + n * DIN + j0 + 4) = make_float4(gx[4], gx[5], gx[6], gx[7]);
            }
        }
        __syncthreads();
        // weight gradients over the tile: thread t owns outputs [t*PER, t*PER+PER) of the flattened [H][DIN] matrix
        {
            const int first = threadIdx.x * PER;
            const int k = first / DIN, j0 = first - k * DIN;
            for (int s = 0; s < MT; s++) {
                const float g = sGH[s * (H + 1) + k];
#pragma unroll
                for (int i = 0; i < PER; i++) acc1[i] = fmaf(g, sX[s * (DIN + 1) + j0 + i], acc1[i]);
            }
            if (threadIdx.x < DOUT * H) {
                const int o = threadIdx.x / H, kk = threadIdx.x - o * H;
                for (int s = 0; s < MT; s++) acc2 = fmaf(sGY[s * 4 + o], sA[s * (H + 1) + kk], acc2);
            }
        }
        __syncthreads();
    }
    {
        const int first = threadIdx.x * PER;
#pragma unroll
        for (int i = 0; i < PER; i++) atomicAdd(GW1 + first + i, acc1[i]);
        if (threadIdx.x < DOUT * H) atomicAdd(GW2 + threadIdx.x, acc2);
    }
}

template <int DIN, int H, int DOUT>
int launch_fwd(const float* X, long long N, const float* W1, const float* W2, float* Y, cudaStream_t s) {
    const size_t smem = (size_t)(2 * DIN * H + 4 * H + MT * (DIN + 1)) * 4;
    const long long tiles_ = (N + MT - 1) / MT;
    mlp2_fwd_kernel<DIN, H, DOUT><<<(unsigned)tiles_, MT, smem, s>>>(X, N, W1, W2, Y);
    return 0;
}
template <int DIN, int H, int DOUT>
int launch_bwd(const float* X, long long N, const float* W1, const float* W2, const float* GY, float* GX, float* GW1,
               float* GW2, cudaStream_t s) {
    const size_t smem = (size_t)(2 * DIN * H + 4 * H + MT * (DIN + 1) + 2 * MT * (H + 1) + MT * 4) * 4;
    static bool set = false;
    if (!set) { cudaFuncSetAttribute(mlp2_bwd_kernel<DIN, H, DOUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); set = true; }
    const long long tiles_ = (N + MT - 1) / MT; const int grid = (int)(tiles_ < GS_NUM_SMS * 3 ? tiles_ : GS_NUM_SMS * 3);
    mlp2_bwd_kernel<DIN, H, DOUT><<<grid, MT, smem, s>>>(X, N, W1, W2, GY, GX, GW1, GW2);
    return 0;
}

#define MLP_DISPATCH(FN, ...)                                                              \
    do {                                                                                   \
        if (Din == 24) { switch (Dout) { case 1: FN<24, 32, 1>(__VA_ARGS__); break; case 2: FN<24, 32, 2>(__VA_ARGS__); break; \
                                         case 3: FN<24, 32, 3>(__VA_ARGS__); break; default: FN<24, 32, 4>(__VA_ARGS__); } }  \
        else { switch (Dout) { case 1: FN<32, 32, 1>(__VA_ARGS__); break; case 2: FN<32, 32, 2>(__VA_ARGS__); break;           \
                               case 3: FN<32, 32, 3>(__VA_ARGS__); break; default: FN<32, 32, 4>(__VA_ARGS__); } }            \
    } while (0)

}  // namespace

int ngp_mlp2_supported(int Din, int H, int Dout) {
    return (H == 32 && (Din == 24 || Din == 32) && Dout >= 1 && Dout <= 4) ? 1 : 0;
}

int ngp_mlp2_fwd(const float* X, long long N, int Din, int H, int Dout, const float* W1, const float* W2, float* Y, cudaStream_t s) {
    if (N <= 0) return 0;
    if (!ngp_mlp2_supported(Din, H, Dout)) { gs_set_error("mlp2: unsupported dims %d-%d-%d", Din, H, Dout); return 1; }
    MLP_DISPATCH(launch_fwd, X, N, W1, W2, Y, s);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int ngp_mlp2_bwd(const float* X, long long N, int Din, int H, int Dout, const float* W1, const float* W2, const float* GY,
                 float* GX, float* GW1, float* GW2, cudaStream_t s) {
    if (N <= 0) return 0;
    if (!ngp_mlp2_supported(Din, H, Dout)) { gs_set_error("mlp2: unsupported dims %d-%d-%d", Din, H, Dout); return 1; }
    MLP_DISPATCH(launch_bwd, X, N, W1, W2, GY, GX, GW1, GW2, s);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
