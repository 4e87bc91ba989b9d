#!/bin/bash
# Builds libfidget_cuda.so (sm_90a, H100, only) in-tree and the CPU oracle.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
SRC=fidget_b200/csrc
OUT=${OUT:-fidget_b200/libfidget_cuda.so}
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 \
  -fmad=false -prec-div=true -prec-sqrt=true -ftz=false \
  -Xcompiler -fPIC,-O2,-ffp-contract=off -shared"
if [ "$1" = "-v" ]; then FLAGS="$FLAGS -Xptxas -v"; fi
# EXTRA="-DSOME_SWITCH" OUT=fidget_b200/libfidget_cuda_variant.so ./build.sh builds a variant for FIDGET_B200_LIB
FLAGS="$FLAGS $EXTRA"
# dev_ops.cuh as a string for the tape compiler (compile.cu): NVRTC compiles the same device arithmetic at run time
mkdir -p build
{ echo 'extern const char k_dev_ops_source[] = R"FC_DEV_OPS('; cat $SRC/cuda/dev_ops.cuh; echo ')FC_DEV_OPS";'; } > build/dev_ops_src.cc
$NVCC $FLAGS -o $OUT build/dev_ops_src.cc $SRC/cuda/compile.cu $SRC/cuda/kernels.cu $SRC/cuda/coop.cu $SRC/cuda/bulk.cu $SRC/cuda/tail2d.cu $SRC/cuda/octree.cu $SRC/cuda/effects.cu $SRC/cuda/capi.cu $SRC/cuda/schedule.cu $SRC/cuda/render.cu $SRC/cuda/octree_capi.cu $SRC/cuda/measure.cu $SRC/cuda/volume.cu $SRC/cuda/ray.cu $SRC/cuda/ray_capi.cu $SRC/cuda/mesh.cu $SRC/cuda/contour.cu $SRC/cuda/effects_capi.cu $SRC/cuda/solve.cu $SRC/cuda/solve_capi.cu $SRC/host/tape.cc $SRC/host/host_capi.cc -ldl
make -s -C oracle liboracle.so
# the solver's CPU oracle (oracle/solve.cc) on top of liboracle's point and gradient VM
CXX=$([ -x /usr/bin/g++ ] && echo /usr/bin/g++ || echo g++)
$CXX -std=c++17 -O2 -fPIC -ffp-contract=off -fno-fast-math -Wall -Wno-unused-function -pthread -shared \
  -o oracle/libsolve_oracle.so oracle/solve.cc -Loracle -l:liboracle.so -Wl,-rpath,'$ORIGIN'
echo "built $OUT, oracle/liboracle.so and oracle/libsolve_oracle.so"
