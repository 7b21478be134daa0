#!/bin/bash
# Builds librd_b200.so in-tree for sm_90a (H100; cross-compiles without a GPU).
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -I../../include ${RD_NVCC_EXTRA}"
OBJS=""
for f in rd_gemm rd_kernels rd_obprop_tc rd_tc_gemm rd_tconv rd_obprop_beta rd_attn_small rd_attn_tc rd_head rd_dp rd_influence rd_projection rd_ekfac rd_trak rd_adversarial rd_counterfactual rd_laplace rd_smoothing rd_sensor_attack rd_prefix rd_ood rd_swag rd_active rd_valuation rd_faithfulness rd_model; do
  if [ ! -f $f.o ] || [ $f.cu -nt $f.o ] || [ rd_common.cuh -nt $f.o ] || [ rd_kernels.cuh -nt $f.o ] || \
     [ rd_obprop_tc.cuh -nt $f.o ] || [ rd_tc_common.cuh -nt $f.o ] || [ rd_tc_gemm.cuh -nt $f.o ] || [ rd_wgmma_tf32.cuh -nt $f.o ] || [ rd_influence.cuh -nt $f.o ] || [ rd_dmma.cuh -nt $f.o ] || [ ../../include/raindrop_b200.h -nt $f.o ] || [ build.sh -nt $f.o ]; then
    $NVCC $FLAGS -c $f.cu -o $f.o &
  fi
  OBJS="$OBJS $f.o"
done
wait
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o librd_b200.so $OBJS -lcudart
echo "built $(pwd)/librd_b200.so"
