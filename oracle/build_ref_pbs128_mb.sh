#!/usr/bin/env bash
# TEST / MEASUREMENT INFRASTRUCTURE -- never on the product path.
#
# Adds the reference's multi-bit 128-bit PBS (src/pbs/programmable_bootstrap_multibit_128.cu, UNMODIFIED, same
# flags as build_ref_cuda.sh) to oracle/_ref/libtfhe_cuda_backend_ref.so, which build_ref_cuda.sh and
# build_ref_pbs128.sh build first.  The translation unit builds on its own and exports the four multi-bit
# `_128` symbols, so tools/bench_squash_multibit.py --lib ref times the reference's
# cuda_multi_bit_programmable_bootstrap_128_async through the same harness, and
# tests/test_noise_squashing_multibit.py checks the two libraries against each other on the same keys.
set -euo pipefail
REF=${REF_ROOT:?set REF_ROOT to a tfhe-rs checkout (build() finds one and sets it)}
CUDA_DIR=$REF/backends/tfhe-cuda-backend/cuda
COMMON=$REF/backends/tfhe-cuda-common/cuda
HERE=$(cd "$(dirname "$0")" && pwd)
OUT=$HERE/_ref
OBJ=$OUT/obj
SO=$OUT/libtfhe_cuda_backend_ref.so
SRC=$CUDA_DIR/src/pbs/programmable_bootstrap_multibit_128.cu
if [ ! -f "$SRC" ]; then
  echo "build_ref_pbs128_mb: $SRC absent -- nothing to build" >&2
  exit 0
fi
[ -f "$SO" ] || { echo "build_ref_pbs128_mb: $SO missing (run build_ref_cuda.sh first)" >&2; exit 1; }
FLAGS=(-gencode arch=compute_90,code=sm_90 -O3 -std=c++17 --no-exceptions
  --expt-relaxed-constexpr -rdc=true --use_fast_math -lineinfo
  -Xcompiler -fPIC -Xcompiler -fopenmp -DCUDA_ARCH=900
  -I"$CUDA_DIR/include" -I"$CUDA_DIR/src" -I"$COMMON/include")
OMB=$OBJ/pbs_programmable_bootstrap_multibit_128.o
if [ ! -f "$OMB" ] || [ "$SRC" -nt "$OMB" ]; then
  nvcc "${FLAGS[@]}" -c "$SRC" -o "$OMB" > "$OMB.log" 2>&1 || { echo "FAILED: $SRC"; tail -30 "$OMB.log"; exit 1; }
fi
# relink when the library lacks the object (an earlier recipe relinked it without) or is older than it
# (grep reads all of nm's output: with -q, nm can die of SIGPIPE and pipefail turns a match into a failure)
if nm -D "$SO" | grep " T cuda_multi_bit_programmable_bootstrap_128_async$" > /dev/null && [ "$SO" -nt "$OMB" ]; then
  echo "up to date: $SO"
  exit 0
fi
nvcc -gencode arch=compute_90,code=sm_90 -shared -Xcompiler -fPIC -Xcompiler -fopenmp \
  "$OBJ"/*.o -o "$SO.tmp" -lcudart -lgomp
mv -f "$SO.tmp" "$SO"
echo "built $SO with the multi-bit 128-bit PBS"
