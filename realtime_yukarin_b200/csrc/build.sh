#!/bin/bash
# Builds libryk.so for sm_90a (H100) in-tree.  Usage: ./build.sh [-j N]
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -Xcompiler -Wno-unused-variable --expt-relaxed-constexpr $RYK_NVCC_EXTRA"
OBJ=${RYK_OBJ_DIR:-_obj}
mkdir -p $OBJ
SRCS="api crepe crepe_tc conv_direct conv_tc s1_fused unet world_analysis world_harvest world_synth features convert denoise echo limiter agc pitch session session_controls session_group session_snapshot reblock snapshot drift"
pids=""
for s in $SRCS; do
  if [ ! -f $OBJ/$s.o ] || [ $s.cu -nt $OBJ/$s.o ] || [ -n "$(find . -maxdepth 1 \( -name '*.h' -o -name '*.cuh' \) -newer $OBJ/$s.o 2>/dev/null)" ] || [ ../../include/ryk.h -nt $OBJ/$s.o ]; then
    $NVCC $FLAGS -c $s.cu -o $OBJ/$s.o &
    pids="$pids $!"
  fi
done
for p in $pids; do wait $p; done
OBJS=""; for s in $SRCS; do OBJS="$OBJS $OBJ/$s.o"; done
$NVCC $ARCH -shared -o ${RYK_LIB_OUT:-libryk.so} $OBJS -L/usr/local/cuda/lib64 -lcufft -Xlinker -rpath -Xlinker /usr/local/cuda/lib64
OUT=${RYK_LIB_OUT:-libryk.so}

echo "built $(pwd)/${RYK_LIB_OUT:-libryk.so}"
