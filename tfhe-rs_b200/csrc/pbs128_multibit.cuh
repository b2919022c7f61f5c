// pbs128_multibit.cuh -- the multi-bit 128-bit PBS (noise squashing with the
// GPU parameters' grouped squashing keys): u64 LWE in, u128 accumulator,
// double-double Fourier key of 2^g GGSWs per group of g mask words, u128 LWE
// out.
//
// Schedule: pbs128_kernel's (pbs128.cuh).  One 512-thread CTA per LWE on a
// persistent grid of at most one CTA per SM; each step streams its digit
// polynomials one at a time through ONE double-double spectrum buffer in
// shared memory, and the accumulator and the k + 1 output spectra live in a
// per-CTA slice of a global workspace reused by the CTA's next sample.
//
// Step (tfhe-rs' multi-bit blind rotation, one per group, n / g steps): the
// degrees of the group are modulus_switch(sum of the selected u64 mask
// words); the digits of the accumulator ITSELF are transformed and multiplied
// by sum_b X^{deg_b} GGSW_b, which is folded slot by slot into the MAC
// (p128_mb_mac: slot pos of X^d is a 2N-th root of unity, read from a
// double-double table); the inverse transforms are ASSIGNED to the
// accumulator.  Exactly one GGSW of a group encrypts 1, so a step multiplies
// the accumulator by X^{deg(s)}.  The alternative -- building each step's
// bundle exactly on the torus and transforming it (the reference) -- costs
// 36 forward transforms per step instead of the fold's 553 k complex FMAs at
// the squash shape, a bundle buffer per LWE and a second kernel; DESIGN.md
// section 8f (multi-bit squashing keys) gives the counts.
//
// Reference semantics: core_crypto/algorithms/
// lwe_multi_bit_programmable_bootstrapping.rs:30-65 (degrees, selection bit),
// backends/tfhe-cuda-backend/cuda/src/pbs/programmable_bootstrap_multibit_128.cuh
// (plain modulus switch of the body, one LUT for every sample, indexes).
#pragma once
#include "pbs128.cuh"

namespace b200 {

constexpr uint32_t PBS128_MB_MAX_GGSW = 16; // 2^g, g <= 4

// dynamic shared memory: one spectrum (M ddc)
static inline size_t pbs128_mb_smem_bytes(uint32_t N) {
  return (size_t)(N / 2) * sizeof(ddc);
}

// out_idx / in_idx: the LWE rows of sample s, or s itself when null
template <uint32_t LOGM>
__global__ void __launch_bounds__(PBS128_THREADS, 1)
pbs128_mb_kernel(u128 *__restrict__ lwe_out,
                 const uint64_t *__restrict__ out_idx,
                 const u128 *__restrict__ lut,
                 const uint64_t *__restrict__ lwe_in,
                 const uint64_t *__restrict__ in_idx,
                 const ddc *__restrict__ bsk, const ddc *__restrict__ tw,
                 const ddc *__restrict__ root, uint32_t n, uint32_t k,
                 uint32_t grouping, uint32_t base_log, uint32_t l,
                 uint32_t num_samples, unsigned char *__restrict__ ws,
                 size_t ws_stride) {
  constexpr uint32_t M = 1u << LOGM, N = 2 * M, NT = PBS128_THREADS;
  extern __shared__ __align__(16) unsigned char p128_smem[];
  ddc *buf = reinterpret_cast<ddc *>(p128_smem);
  __shared__ uint32_t degs[PBS128_MB_MAX_GGSW];
  __shared__ uint32_t b_hat_s;

  u128 *acc = reinterpret_cast<u128 *>(ws + (size_t)blockIdx.x * ws_stride);
  ddc *out = reinterpret_cast<ddc *>(acc + (size_t)(k + 1) * N);
  const uint32_t tid = threadIdx.x;
  const uint32_t log_mod = LOGM + 2; // log2(2N)
  const uint32_t nggsw = 1u << grouping;
  const size_t ggsw_len = (size_t)l * (k + 1) * (k + 1) * M;

  for (uint32_t s = blockIdx.x; s < num_samples; s += gridDim.x) {
    const uint64_t *ct = lwe_in + (in_idx ? in_idx[s] : s) * (uint64_t)(n + 1);
    if (tid == 0)
      b_hat_s = modulus_switch_u64(ct[n], log_mod);
    __syncthreads();
    // ---- acc = LUT * X^{-b_hat} ------------------------------------------------
    rotate_lut(acc, N, lut, k + 1, N, b_hat_s, tid, NT, SameWord());

    // ---- blind rotation, one step per group ------------------------------------
    for (uint32_t i = 0; i < n / grouping; i++) {
      if (tid < nggsw)
        degs[tid] = p128_mb_degree(ct + (size_t)i * grouping, grouping, tid,
                                   log_mod);
      __syncthreads(); // degs, and the accumulator of the previous step
      const ddc *group = bsk + (size_t)i * nggsw * ggsw_len;
      for (uint32_t t = 0; t < l; t++)
        for (uint32_t r = 0; r <= k; r++) {
          p128_decompose_acc(acc + (size_t)r * N, buf, N, base_log, l, t, tid,
                             NT);
          __syncthreads();
#pragma unroll 1
          for (uint32_t L = 1; L <= LOGM; L++) {
            p128_fwd_level(buf, LOGM, L, tw, tid, NT);
            __syncthreads();
          }
          p128_mb_mac(buf, out,
                      group + ((size_t)t * (k + 1) + r) * (k + 1) * M,
                      ggsw_len, nggsw, degs, root, LOGM, k, t == 0 && r == 0,
                      tid, NT);
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
        p128_acc_assign(acc + (size_t)c * N, buf, M, tid, NT);
        __syncthreads();
      }
    }

    // ---- sample extraction of coefficient 0 --------------------------------------
    sample_extract_lwe(lwe_out + (out_idx ? out_idx[s] : s) * ((uint64_t)k * N + 1),
                       acc, N, k, N, 0, tid, NT, SameWord());
    __syncthreads(); // the workspace is reused by the next sample of this CTA
  }
}

// one instance per polynomial size, [log2(N) - 8], with the name
// b200_last_pbs_kernel reports; the key conversion is the classic one
// (bsk_convert_128_kernel) over 2^g / g times as many polynomials
static const struct Pbs128MbInstance {
  decltype(&pbs128_mb_kernel<10>) kernel;
  const char *name;
} PBS128_MB_INSTANCES[] = {
    {pbs128_mb_kernel<7>, "pbs128_mb<256>"},
    {pbs128_mb_kernel<8>, "pbs128_mb<512>"},
    {pbs128_mb_kernel<9>, "pbs128_mb<1024>"},
    {pbs128_mb_kernel<10>, "pbs128_mb<2048>"},
    {pbs128_mb_kernel<11>, "pbs128_mb<4096>"},
};

} // namespace b200
