#!/bin/bash
# Builds libgs_b200.so in-tree for the H100 (sm_90a; nvcc cross-compiles without a GPU).
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
COMMON="-O3 -std=c++17 -lineinfo -Xcompiler -fPIC $ARCH --expt-relaxed-constexpr ${GS_NVCC_EXTRA}"
rm -rf build && mkdir -p build     # the link takes build/*.o: no object of a renamed or deleted source
pids=()
# preprocess forward: NO FMA contraction (bit-exact integer outputs vs the oracle)
$NVCC $COMMON -fmad=false -c gs_preprocess.cu -o build/gs_preprocess.o & pids+=($!)
$NVCC $COMMON -fmad=false -c dr_raster.cu -o build/dr_raster.o & pids+=($!)
$NVCC $COMMON -fmad=false -c cr_raster.cu -o build/cr_raster.o & pids+=($!)
$NVCC $COMMON -fmad=false -c uv_bake.cu -o build/uv_bake.o & pids+=($!)
$NVCC $COMMON -fmad=false -c pn2_ops.cu -o build/pn2_ops.o & pids+=($!)
# point rasterizer: no FMA contraction (bit-exact projection, pixel centres and distances vs the oracle)
$NVCC $COMMON -fmad=false -c pts_raster.cu -o build/pts_raster.o & pids+=($!)
for f in gs_sort gs_binning gs_composite gs_backward gs_knn gs_train gs_densify gs_loss gs_capi dr_ops ngp_ops ngp_mlp ngp_mcubes ngp_flexicubes ngp_dmc gs_scatter sp_conv gs_attn; do
  $NVCC $COMMON -c $f.cu -o build/$f.o & pids+=($!)
done
for p in "${pids[@]}"; do wait $p; done
$NVCC -shared $ARCH -o ../gs_b200/libgs_b200.so build/*.o -lcudart
echo "built $(realpath ../gs_b200/libgs_b200.so)"
