#!/usr/bin/env bash
# TEST / MEASUREMENT INFRASTRUCTURE -- never on the product path.
#
# Builds the reference's zk-cuda-backend (backends/zk-cuda-backend: BLS12-446
# field arithmetic and Pippenger MSM, UNMODIFIED sources) with plain nvcc for
# sm_90 into oracle/_ref/libzk_cuda_backend_ref.so, with tfhe-cuda-common's
# device.cu and helper_profile.cu (NVTX ranges, compiled out without
# USE_NVTOOLS) that it links against.  Its CMake build is not
# used: it fetches Google Test.  -rdc=true because that build sets separable
# compilation.  The library exports the 25 functions of include/tfhe_b200_zk.h;
# tests/test_zk_msm.py checks parity with it and tools/bench_msm.py --lib ref
# times it.  Objects are rebuilt only when their source is newer.
set -euo pipefail
REF=${REF_ROOT:?set REF_ROOT to a tfhe-rs checkout (build() finds one and sets it)}
ZK=$REF/backends/zk-cuda-backend
COMMON=$REF/backends/tfhe-cuda-common/cuda
HERE=$(cd "$(dirname "$0")" && pwd)
OUT=$HERE/_ref
OBJ=$OUT/obj_zk
SO=$OUT/libzk_cuda_backend_ref.so
if [ ! -d "$ZK/cuda/src" ]; then
  echo "build_ref_zk: $ZK absent -- nothing to build" >&2
  exit 0
fi
mkdir -p "$OBJ"
FLAGS=(-gencode arch=compute_90,code=sm_90 -O3 -std=c++17 --expt-relaxed-constexpr -rdc=true
  -Xcompiler -fPIC -I"$ZK/cuda/include" -I"$ZK/cuda/src" -I"$ZK/src/include" -I"$COMMON/include")
SRCS=("$ZK/cuda/src/primitives/fp.cu" "$ZK/cuda/src/primitives/fp2.cu" "$ZK/cuda/src/primitives/xyzz.cu"
  "$ZK/cuda/src/curve.cu" "$ZK/cuda/src/msm/pippenger/msm_pippenger.cu" "$ZK/cuda/src/msm/msm.cu"
  "$ZK/src/c_wrapper.cu" "$COMMON/src/device.cu" "$COMMON/src/helper_profile.cu")
pids=()
objs=()
for src in "${SRCS[@]}"; do
  o=$OBJ/$(basename "$(dirname "$src")")_$(basename "$src" .cu).o
  objs+=("$o")
  if [ ! -f "$o" ] || [ "$src" -nt "$o" ]; then
    nvcc "${FLAGS[@]}" -c "$src" -o "$o" > "$o.log" 2>&1 &
    pids+=($!)
  fi
done
for p in "${pids[@]}"; do
  wait "$p" || { echo "FAILED: see $OBJ/*.log"; tail -30 "$OBJ"/*.log; exit 1; }
done
newest=$(ls -t "${objs[@]}" | head -1)
if [ -f "$SO" ] && [ "$SO" -nt "$newest" ]; then
  echo "up to date: $SO"
  exit 0
fi
nvcc -gencode arch=compute_90,code=sm_90 -shared -Xcompiler -fPIC "${objs[@]}" -o "$SO.tmp" -lcudart
mv -f "$SO.tmp" "$SO"
echo "built $SO"
