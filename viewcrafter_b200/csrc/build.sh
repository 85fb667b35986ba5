#!/bin/bash
# Build libvc_b200.so in-tree for sm_90a (H100; cross-compiles without a GPU).
set -euo pipefail
cd "$(dirname "$0")"
NVCC=${NVCC:-nvcc}
if ! command -v "$NVCC" >/dev/null 2>&1 && [ -x /usr/local/cuda/bin/nvcc ]; then NVCC=/usr/local/cuda/bin/nvcc; fi
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xcompiler -Wall --expt-relaxed-constexpr ${VC_NVCC_EXTRA:-}"
OUT=${VC_OUT:-../libvc_b200.so}          # VC_OUT / VC_BUILD_DIR / VC_NVCC_EXTRA: side-by-side A/B builds (load with VC_B200_LIB)
BUILD=${VC_BUILD_DIR:-build}
SRCS="host.cu capi.cu gemm_tap.cu attention.cu temporal_attn.cu norm.cu misc.cu peer.cu"
mkdir -p $BUILD
pids=()
for f in $SRCS; do
  $NVCC $FLAGS -c $f -o $BUILD/${f%.cu}.o &
  pids+=($!)
done
for p in "${pids[@]}"; do wait $p; done
$NVCC $ARCH -shared -o $OUT $BUILD/*.o -lcudart
echo "built $(realpath $OUT)"
