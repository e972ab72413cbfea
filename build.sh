#!/bin/bash
# Build the in-tree CUDA library for sm_90a (H100) (nvcc cross-compiles without a GPU).
set -e
cd "$(dirname "$0")"
SRC=wespeaker_b200/csrc
OUT=wespeaker_b200/lib
mkdir -p $OUT build
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC --expt-relaxed-constexpr -DWS_BUILD ${EXTRA_NVCC}"
objs=""
pids=""
for f in ws_gemm_tc2 ws_res2_fused ws_conv3x3 ws_cam_dense ws_astp_fused ws_simam ws_dwconv ws_gemm_simt ws_kernels ws_fbank ws_plda ws_conv_host ws_build_ecapa ws_build_2d ws_build_tdnn ws_engine ws_plda_host ws_score ws_diar ws_metrics; do
  if [ ! -f build/$f.o ] || [ $SRC/$f.cu -nt build/$f.o ] || [ $SRC/ws_common.cuh -nt build/$f.o ] || [ $SRC/ws_kernels.cuh -nt build/$f.o ] || [ $SRC/ws_host.h -nt build/$f.o ] || [ $SRC/ws_plan.h -nt build/$f.o ] || [ $SRC/ws_tc_common.cuh -nt build/$f.o ] || [ $SRC/ws_wgmma.cuh -nt build/$f.o ] || [ $SRC/ws_select.cuh -nt build/$f.o ] || [ include/wespeaker_b200.h -nt build/$f.o ]; then
    $NVCC $FLAGS ${PTXAS_V:+-Xptxas -v} -c $SRC/$f.cu -o build/$f.o &
    pids="$pids $!"
  fi
  objs="$objs build/$f.o"
done
for p in $pids; do wait $p; done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o $OUT/libwespeaker_b200.so $objs -lcudart_static -ldl -lrt -lpthread
echo "built $OUT/libwespeaker_b200.so"
