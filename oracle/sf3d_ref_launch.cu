// Launcher for the reference's own SF3D texture baker: the CUDA that slangtorch generated from texture_baker.slang
// (ComfyUI-3D-Pack's sf3d/.slangtorch_cache/texture_baker/<hash>/texture_baker_cuda.cu), compiled in place through
// `-I` with nvcc's default flags for sm_90a.  oracle/build_ref.py builds it into
// oracle/_ref/sf3d_texture_baker/libsf3d_texture_baker_ref.so; tests and scripts/bench_uvbake.py call it through ctypes.
//
// Each call builds the TensorViews slangtorch's host wrapper would (byte strides of contiguous tensors, sizes) and
// launches the reference kernel with the caller's block and grid, exactly as `launchRaw(blockSize=, gridSize=)` does.
#include "texture_baker_cuda.cu"

namespace {

TensorView view(const void* data, int ndim, const uint32_t* sizes, uint32_t elem) {
    TensorView t = {};
    t.data = (uint8_t*)data;
    t.dimensionCount = (uint32_t)ndim;
    uint32_t stride = elem;
    for (int d = ndim - 1; d >= 0; d--) {
        t.sizes[d] = sizes[d];
        t.strides[d] = stride;
        stride *= sizes[d];
    }
    return t;
}

}  // namespace

// uv[V,2] fp32, indices[F,3] int32, output[H,W,4] fp32
extern "C" int sf3d_ref_bake_uv(const float* uv, int V, const int32_t* indices, int F, float* output, int H, int W,
                                unsigned bx, unsigned by, unsigned gx, unsigned gy, void* stream) {
    const uint32_t su[2] = {(uint32_t)V, 2u}, si[2] = {(uint32_t)F, 3u}, so[3] = {(uint32_t)H, (uint32_t)W, 4u};
    TensorView a = view(uv, 2, su, 4), b = view(indices, 2, si, 4), c = view(output, 3, so, 4);
    if (gx && gy) __kernel__bake_uv<<<dim3(gx, gy, 1), dim3(bx, by, 1), 0, (cudaStream_t)stream>>>(a, b, c);
    return (int)cudaGetLastError();
}

// attr[V,3] fp32, indices[F,3] int32, rast[H,W,4] fp32, output[H,W,3] fp32
extern "C" int sf3d_ref_interpolate(const float* attr, int V, const int32_t* indices, int F, const float* rast,
                                    float* output, int H, int W, unsigned bx, unsigned by, unsigned gx, unsigned gy,
                                    void* stream) {
    const uint32_t sa[2] = {(uint32_t)V, 3u}, si[2] = {(uint32_t)F, 3u}, sr[3] = {(uint32_t)H, (uint32_t)W, 4u},
                   so[3] = {(uint32_t)H, (uint32_t)W, 3u};
    TensorView a = view(attr, 2, sa, 4), b = view(indices, 2, si, 4), r = view(rast, 3, sr, 4), o = view(output, 3, so, 4);
    if (gx && gy) __kernel__interpolate<<<dim3(gx, gy, 1), dim3(bx, by, 1), 0, (cudaStream_t)stream>>>(a, b, r, o);
    return (int)cudaGetLastError();
}
