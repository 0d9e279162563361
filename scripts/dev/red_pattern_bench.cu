// Times the two shapes of the composite backward's fp64 gradient reds on their own (built and run by
// red_pattern_bench.py).  A 96 MB array of 96 B records (SplatGrad's size and alignment) receives `visits` sets of ten
// fp64 reds, at the value offsets SplatGrad uses, into records picked by a seeded random permutation of `ids` ids:
//   records: lanes = records, ten red instructions per 32 visits (combine_stage before the coalesced combine);
//   values:  lanes = (record r in 0..2, value k in 0..9), one red instruction per 3 visits, lanes 30 and 31 idle.
// Both shapes add the same values to the same words; the program checks that the arrays they leave are identical.
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

struct __align__(32) Rec { double v[12]; };
constexpr int NVAL = 10;

__device__ __forceinline__ int off(int k) { return k < 3 ? k : k + 1; }          // SplatGrad skips doubles 3 and 11
__device__ __forceinline__ double val(int k) { return (double)(k + 1) * 0x1p-20; }  // exact in any order

__global__ void red_records(Rec* __restrict__ a, const uint32_t* __restrict__ perm, int ids, long long visits) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < visits; t += stride) {
        double* d = a[perm[t % ids]].v;
#pragma unroll
        for (int k = 0; k < NVAL; k++) atomicAdd(d + off(k), val(k));
    }
}

__global__ void red_values(Rec* __restrict__ a, const uint32_t* __restrict__ perm, int ids, long long visits) {
    const int lane = threadIdx.x & 31, r = lane % 3, k = lane / 3;
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long b = warp * 3; b < visits; b += nwarps * 3) {
        const long long t = b + r;
        if (k < NVAL && t < visits) atomicAdd(a[perm[t % ids]].v + off(k), val(k));
    }
}

int main(int argc, char** argv) {
    const int ids = argc > 1 ? atoi(argv[1]) : 1000000;
    const long long visits = argc > 2 ? atoll(argv[2]) : 4800000;       // x 10 values = 48 M reds per launch
    const int launches = argc > 3 ? atoi(argv[3]) : 20;
    const int reps = argc > 4 ? atoi(argv[4]) : 3;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    std::vector<uint32_t> perm(ids);
    for (int i = 0; i < ids; i++) perm[i] = (uint32_t)i;
    std::shuffle(perm.begin(), perm.end(), std::mt19937(1234));
    Rec* a; uint32_t* dperm;
    const size_t bytes = (size_t)ids * sizeof(Rec);
    CK(cudaMalloc(&a, bytes));
    CK(cudaMalloc(&dperm, (size_t)ids * 4));
    CK(cudaMemcpy(dperm, perm.data(), (size_t)ids * 4, cudaMemcpyHostToDevice));
    const int grid = prop.multiProcessorCount * 8, block = 256;
    auto launch = [&](int shape) {
        if (shape == 0) red_records<<<grid, block>>>(a, dperm, ids, visits);
        else red_values<<<grid, block>>>(a, dperm, ids, visits);
    };
    // same result from both shapes (one launch each into a zeroed array)
    std::vector<double> h0(bytes / 8), h1(bytes / 8);
    for (int shape = 0; shape < 2; shape++) {
        CK(cudaMemset(a, 0, bytes));
        launch(shape);
        CK(cudaGetLastError());
        CK(cudaMemcpy(shape ? h1.data() : h0.data(), a, bytes, cudaMemcpyDeviceToHost));
    }
    const bool same = memcmp(h0.data(), h1.data(), bytes) == 0;
    for (int shape = 0; shape < 2; shape++) for (int i = 0; i < 3; i++) launch(shape);      // warm-up
    CK(cudaDeviceSynchronize());
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    printf("{\"device\": \"%s\", \"sms\": %d, \"ids\": %d, \"array_mb\": %.1f, \"reds_per_launch\": %lld, \"launches\": %d, "
           "\"same_result\": %s}\n", prop.name, prop.multiProcessorCount, ids, bytes / 1e6, visits * NVAL, launches,
           same ? "true" : "false");
    for (int rep = 0; rep < reps; rep++) {
        for (int shape = 0; shape < 2; shape++) {           // alternating
            CK(cudaEventRecord(e0));
            for (int i = 0; i < launches; i++) launch(shape);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            float ms;
            CK(cudaEventElapsedTime(&ms, e0, e1));
            printf("{\"rep\": %d, \"shape\": \"%s\", \"ms_per_launch\": %.4f, \"Greds_per_s\": %.2f}\n", rep,
                   shape ? "values" : "records", ms / launches, visits * NVAL / (ms / launches * 1e-3) / 1e9);
        }
    }
    CK(cudaFree(a)); CK(cudaFree(dperm));
    return same ? 0 : 2;
}
