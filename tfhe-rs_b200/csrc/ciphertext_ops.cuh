// ciphertext_ops.cuh -- the stand-alone integer stages either side of the
// blind rotation, as the reference backend also exports them
// (backends/tfhe-cuda-backend/cuda/include/ciphertext.h:15-32):
//   * sample extraction of an arbitrary coefficient
//     (extract_lwe_sample_from_glwe_ciphertext, tfhe/src/core_crypto/algorithms/
//     glwe_sample_extraction.rs:119-165; reference kernel crypto/ciphertext.cuh:32-54),
//   * the standard modulus switch (fft_impl/common.rs:10-23; torus.cuh:132-138),
//   * the centered-mean modulus switch of one LWE (algorithms/modulus_switch.rs:35-100).
// All exact u64 arithmetic; the PBS kernels fuse the same helpers.
#pragma once
#include "pbs_n2048_phases.cuh"

#include <cuda_runtime.h>

namespace b200 {

// one CTA per extracted LWE (the reference's indexing contract:
// GLWE = id / num_lwes_to_extract_per_glwe, nth = nth_array[id] % stored)
__global__ void __launch_bounds__(256)
glwe_sample_extract_kernel(uint64_t *__restrict__ lwe_out,
                           const uint64_t *__restrict__ glwe_in,
                           const uint32_t *__restrict__ nth_array,
                           uint32_t per_glwe, uint32_t stored_per_glwe,
                           uint32_t k, uint32_t N) {
  const uint32_t id = blockIdx.x;
  const uint64_t *glwe = glwe_in + (uint64_t)(id / per_glwe) * (k + 1) * N;
  uint64_t *out = lwe_out + (uint64_t)id * ((uint64_t)k * N + 1);
  const uint32_t nth = nth_array[id] % stored_per_glwe;
  sample_extract_lwe(out, glwe, N, k, N, nth, threadIdx.x, blockDim.x, SameWord());
}

__global__ void __launch_bounds__(256)
modulus_switch_kernel(uint64_t *__restrict__ out, const uint64_t *__restrict__ in,
                      uint32_t size, uint32_t log_modulus) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < size)
    out[i] = modulus_switch_full(in[i], log_modulus);
}

// one CTA, one LWE: mask plain switch, body switched after the centered-mean
// correction (block-wide reduction of the two error sums)
__global__ void __launch_bounds__(256)
centered_modulus_switch_kernel(uint64_t *__restrict__ out,
                               const uint64_t *__restrict__ in, uint32_t n,
                               uint32_t log_modulus) {
  __shared__ unsigned long long red_half[8];
  __shared__ long long red_dbl[8];
  CenteredMsSums sums;
  for (uint32_t i = threadIdx.x; i < n; i += 256) {
    const uint64_t a = in[i];
    out[i] = modulus_switch_full(a, log_modulus);
    sums.add(a, log_modulus);
  }
  centered_ms_publish_warp(sums, red_half, red_dbl);
  __syncthreads();
  if (threadIdx.x == 0)
    out[n] = modulus_switch_full(centered_ms_body(in[n], red_half, red_dbl, 8, log_modulus),
                                 log_modulus);
}

} // namespace b200
