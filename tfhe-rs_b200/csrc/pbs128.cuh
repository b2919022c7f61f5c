// pbs128.cuh -- the classic 128-bit PBS (noise squashing): u64 LWE in, u128
// accumulator, double-double Fourier key, u128 LWE out.
//
// Schedule: one CTA per LWE (a persistent grid strides over the samples).  At
// the squash shape (k = 2, N = 2048, l = 3) the accumulator is 96 KiB, one
// double-double spectrum 32 KiB and the k + 1 output spectra 96 KiB; the nine
// digit spectra of a step (288 KiB) cannot all be resident.  So a step streams
// its digit polynomials one at a time through ONE spectrum buffer in shared
// memory -- decompose, forward transform, MAC into the output spectra -- and
// the accumulator and the output spectra live in a per-CTA slice of a global
// workspace (L2 resident: one slice per SM).  The inverse transform of each
// output polynomial reuses the shared buffer and is rounded straight into the
// accumulator.  Every (N <= 4096, k, l) runs this one code path; a (k+1)-CTA
// cluster exchanging digit spectra through distributed shared memory would
// tie the grid shape to k and still need the accumulator outside the SM at
// N = 4096.
//
// Reference: backends/tfhe-cuda-backend/cuda/src/pbs/
// programmable_bootstrap_classic_128.cuh (same modulus switch, centered
// correction, rotation, decomposition and sample extraction).
#pragma once
#include "pbs128_phases.cuh"

#include <cuda_runtime.h>

namespace b200 {

constexpr uint32_t PBS128_THREADS = 512;

// dynamic shared memory: one spectrum (M ddc) + the switched mask (n + 1 u32)
static inline size_t pbs128_smem_bytes(uint32_t n, uint32_t N) {
  return (size_t)(N / 2) * sizeof(ddc) + ((size_t)n + 1) * 4;
}
// global workspace slice of one CTA: accumulator + output spectra
static inline size_t pbs128_ws_bytes(uint32_t k, uint32_t N) {
  const size_t b = (size_t)(k + 1) * N * sizeof(u128) +
                   (size_t)(k + 1) * (N / 2) * sizeof(ddc);
  return (b + 255) / 256 * 256;
}

template <uint32_t LOGM>
__global__ void __launch_bounds__(PBS128_THREADS, 1)
pbs128_kernel(u128 *__restrict__ lwe_out, const u128 *__restrict__ lut,
              const uint64_t *__restrict__ lwe_in, const ddc *__restrict__ bsk,
              const ddc *__restrict__ tw, uint32_t n, uint32_t k,
              uint32_t base_log, uint32_t l, uint32_t num_samples,
              int centered_ms, unsigned char *__restrict__ ws,
              size_t ws_stride) {
  constexpr uint32_t M = 1u << LOGM, N = 2 * M, NT = PBS128_THREADS;
  extern __shared__ __align__(16) unsigned char p128_smem[];
  ddc *buf = reinterpret_cast<ddc *>(p128_smem);
  uint32_t *a_hat = reinterpret_cast<uint32_t *>(buf + M);
  __shared__ unsigned long long red_half[NT / 32];
  __shared__ long long red_dbl[NT / 32];
  __shared__ uint32_t b_hat_s;

  u128 *acc = reinterpret_cast<u128 *>(ws + (size_t)blockIdx.x * ws_stride);
  ddc *out = reinterpret_cast<ddc *>(acc + (size_t)(k + 1) * N);
  const uint32_t tid = threadIdx.x;
  const uint32_t log_mod = LOGM + 2; // log2(2N)
  const size_t ggsw_len = (size_t)l * (k + 1) * (k + 1) * M;

  for (uint32_t s = blockIdx.x; s < num_samples; s += gridDim.x) {
    const uint64_t *ct = lwe_in + (uint64_t)s * (n + 1);
    // ---- modulus switch (same as the 64-bit PBS) ---------------------------
    CenteredMsSums sums;
    for (uint32_t i = tid; i < n; i += NT) {
      const uint64_t a = ct[i];
      a_hat[i] = modulus_switch_u64(a, log_mod);
      if (centered_ms)
        sums.add(a, log_mod);
    }
    if (centered_ms)
      centered_ms_publish_warp(sums, red_half, red_dbl);
    __syncthreads();
    if (tid == 0)
      b_hat_s = ms_b_hat(ct[n], centered_ms, red_half, red_dbl, NT / 32, log_mod);
    __syncthreads();
    // ---- acc = LUT * X^{-b_hat} ------------------------------------------------
    rotate_lut(acc, N, lut, k + 1, N, b_hat_s, tid, NT, SameWord());
    __syncthreads();

    // ---- blind rotation ----------------------------------------------------------
    for (uint32_t i = 0; i < n; i++) {
      const uint32_t a = a_hat[i];
      if (a == 0)
        continue;
      const ddc *ggsw = bsk + (size_t)i * ggsw_len;
      for (uint32_t t = 0; t < l; t++)
        for (uint32_t r = 0; r <= k; r++) {
          p128_decompose(acc + (size_t)r * N, buf, N, a, base_log, l, t, tid,
                         NT);
          __syncthreads();
#pragma unroll 1
          for (uint32_t L = 1; L <= LOGM; L++) {
            p128_fwd_level(buf, LOGM, L, tw, tid, NT);
            __syncthreads();
          }
          p128_mac(buf, out, ggsw + ((size_t)t * (k + 1) + r) * (k + 1) * M, M,
                   k, t == 0 && r == 0, tid, NT);
          __syncthreads();
        }
      for (uint32_t c = 0; c <= k; c++) {
        for (uint32_t j = tid; j < M; j += NT)
          buf[j] = out[(size_t)c * M + j];
        __syncthreads();
#pragma unroll 1
        for (uint32_t L = LOGM; L >= 1; L--) {
          p128_inv_level(buf, LOGM, L, tw, tid, NT);
          __syncthreads();
        }
        p128_acc_add(acc + (size_t)c * N, buf, M, tid, NT);
        __syncthreads();
      }
    }

    // ---- sample extraction of coefficient 0 --------------------------------------
    sample_extract_lwe(lwe_out + (uint64_t)s * ((uint64_t)k * N + 1), acc, N, k, N, 0,
                       tid, NT, SameWord());
    __syncthreads(); // the workspace is reused by the next sample of this CTA
  }
}

// standard-domain u128 key polynomial -> double-double spectrum / M, same
// [n][l][k+1][k+1] nesting as the source.  grid = #polynomials.
template <uint32_t LOGM>
__global__ void __launch_bounds__(256)
bsk_convert_128_kernel(ddc *__restrict__ dst, const u128 *__restrict__ src,
                       const ddc *__restrict__ tw) {
  constexpr uint32_t M = 1u << LOGM;
  extern __shared__ __align__(16) unsigned char p128_smem[];
  ddc *buf = reinterpret_cast<ddc *>(p128_smem);
  const uint32_t tid = threadIdx.x;
  p128_load_key_poly(src + (size_t)blockIdx.x * 2 * M, buf, M, tid, 256);
  __syncthreads();
  for (uint32_t L = 1; L <= LOGM; L++) {
    p128_fwd_level(buf, LOGM, L, tw, tid, 256);
    __syncthreads();
  }
  ddc *o = dst + (size_t)blockIdx.x * M;
  for (uint32_t j = tid; j < M; j += 256)
    o[j] = buf[j];
}

// noise squashing, step 1: pack pairs of blocks, in[2i] + mod * in[2i + 1]
// (an odd last block alone).  One thread per output word.
__global__ void __launch_bounds__(256)
squash_pack_pairs_kernel(uint64_t *__restrict__ out,
                         const uint64_t *__restrict__ in, uint32_t lwe_len,
                         uint32_t num_blocks, uint64_t message_modulus) {
  const uint64_t w = (uint64_t)blockIdx.x * 256 + threadIdx.x;
  const uint32_t packed = (num_blocks + 1) / 2;
  if (w >= (uint64_t)packed * lwe_len)
    return;
  const uint64_t p = w / lwe_len, c = w % lwe_len;
  const uint64_t lo = in[(2 * p) * lwe_len + c];
  out[w] = 2 * p + 1 < num_blocks
               ? lo + message_modulus * in[(2 * p + 1) * lwe_len + c]
               : lo;
}

} // namespace b200
