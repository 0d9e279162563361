#!/bin/bash
# Builds libgs_b200.so in-tree for the H100 (sm_90a; nvcc cross-compiles without a GPU).
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
COMMON="-O3 -std=c++17 -lineinfo -Xcompiler -fPIC $ARCH --expt-relaxed-constexpr ${GS_NVCC_EXTRA}"
mkdir -p build
pids=()
# preprocess forward: NO FMA contraction (bit-exact integer outputs vs the oracle)
$NVCC $COMMON -fmad=false -c gs_preprocess.cu -o build/gs_preprocess.o & pids+=($!)
$NVCC $COMMON -fmad=false -c dr_raster.cu -o build/dr_raster.o & pids+=($!)
$NVCC $COMMON -fmad=false -c cr_raster.cu -o build/cr_raster.o & pids+=($!)
$NVCC $COMMON -fmad=false -c uv_bake.cu -o build/uv_bake.o & pids+=($!)
$NVCC $COMMON -fmad=false -c pn2_ops.cu -o build/pn2_ops.o & pids+=($!)
for f in gs_sort gs_binning gs_composite gs_backward gs_knn gs_train gs_densify gs_loss gs_capi dr_ops dr_capi ngp_ops ngp_mlp ngp_capi ngp_mcubes ngp_flexicubes ngp_dmc gs_scatter sp_conv; do
  $NVCC $COMMON -c $f.cu -o build/$f.o & pids+=($!)
done
# attention (flash_attn drop-in): its own library, linked against libgs_b200.so for the error and launch counters
mkdir -p build/attn
$NVCC $COMMON -c gs_attn.cu -o build/attn/gs_attn.o & pids+=($!)
# point rasterizer (pytorch3d PointsRasterizer / points_projection drop-in): a companion library in the same way;
# no FMA contraction (bit-exact projection, pixel centres and distances vs the oracle)
mkdir -p build/pts
$NVCC $COMMON -fmad=false -c pts_raster.cu -o build/pts/pts_raster.o & pids+=($!)
for p in "${pids[@]}"; do wait $p; done
$NVCC -shared $ARCH -o ../gs_b200/libgs_b200.so build/*.o -lcudart
$NVCC -shared $ARCH -o ../gs_b200/libgs_attn.so build/attn/gs_attn.o -L../gs_b200 -lgs_b200 -lcudart -Xlinker -rpath -Xlinker '$ORIGIN'
$NVCC -shared $ARCH -o ../gs_b200/libgs_pts.so build/pts/pts_raster.o -L../gs_b200 -lgs_b200 -lcudart -Xlinker -rpath -Xlinker '$ORIGIN'
echo "built $(realpath ../gs_b200/libgs_b200.so) $(realpath ../gs_b200/libgs_attn.so) $(realpath ../gs_b200/libgs_pts.so)"
