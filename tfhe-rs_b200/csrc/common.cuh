// common.cuh -- error handling and per-device constant tables.
//
// Error behaviour mirrors tfhe-cuda-common/cuda/include/device.h:13-57 of the
// reference: no return codes; a CUDA error or a violated precondition prints
// to stderr and abort()s.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#include "negacyclic_fft.cuh"

#define B200_CHECK(ans)                                                        \
  do {                                                                         \
    cudaError_t code_ = (ans);                                                 \
    if (code_ != cudaSuccess) {                                                \
      std::fprintf(stderr, "Cuda error: %s %s %d\n",                           \
                   cudaGetErrorString(code_), __FILE__, __LINE__);             \
      std::abort();                                                            \
    }                                                                          \
  } while (0)

#define B200_PANIC(format, ...)                                                \
  do {                                                                         \
    std::fprintf(stderr, "%s::%d::%s: panic.\n" format "\n", __FILE__,         \
                 __LINE__, __func__, ##__VA_ARGS__);                           \
    std::abort();                                                              \
  } while (0)

#define B200_PANIC_IF_FALSE(cond, format, ...)                                 \
  do {                                                                         \
    if (!(cond))                                                               \
      B200_PANIC(format "\n\n %s\n", ##__VA_ARGS__, #cond);                    \
  } while (0)

namespace b200 {

constexpr int MAX_GPUS = 16;
constexpr int MAX_LOGM = 13;

// Device-resident, immutable lookup tables, created lazily once per GPU.
struct DeviceTables {
  Fft1024Tables *fft1024 = nullptr;        // pass-2 / pass-3 twiddles
  Fft256Tables *fft256 = nullptr;          // N = 512 register kernel (pbs_n512.cuh)
  Fft4096Tables *fft4096 = nullptr;        // N = 8192 register kernel (pbs_n8192.cuh)
  cplx *gen_tw[MAX_LOGM + 1] = {nullptr};  // generic radix-2 twiddles per logM
  cplx *gen_root[MAX_LOGM + 1] = {nullptr}; // 2N-th roots per logM
  // N = 2048 multi-bit kernels: mono2048[deg][t] = tau^{deg * (1 + 4*bitrev6(t))},
  // deg < 4096, t < 64 (4 MiB, L2 resident).  The 64 lanes of a polynomial
  // group read one contiguous 1 KiB row per rotated GGSW instead of gathering
  // 64 scattered entries of the root table (the gather was ~80 % of the bundle
  // kernel: one L1 line per lane per look-up).
  cplx *mono2048 = nullptr;
};

// returns the tables for `gpu_index`, creating what is missing (thread safe).
// logM == 0: only the N = 2048 register-FFT tables are guaranteed.
const DeviceTables &device_tables(uint32_t gpu_index, uint32_t logM);

void set_device(uint32_t gpu_index);

} // namespace b200
