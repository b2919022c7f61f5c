// pbs_generic.cuh -- any-(N, k, l) PBS kernels, classic and multi-bit.
//
// Covers every parameter set the register-FFT kernel (pbs_n2048.cuh) does not:
// other polynomial sizes (boolean N = 512 / 1024, shortint 1_1 ... 3_3),
// k > 1, l > 1, and the multi-bit PBS.  One CTA per LWE; accumulator, digit
// spectra and output spectra stay in shared memory for the whole rotation.
// The multi-bit key bundle is never materialised (the reference writes it to
// HBM, cuda/src/pbs/programmable_bootstrap_multibit.cuh:739-758): it is folded
// into the Fourier MAC, sum_s B_s(pos) * rho_pos^{deg_s}, straight from L2.
//
// Replaces device_programmable_bootstrap_step_one/_two, _cg, _tbc and the
// device_multi_bit_programmable_bootstrap_* family of the reference.
#pragma once
#include "pbs_generic_phases.cuh"

#include <cuda_runtime.h>

namespace b200 {

struct GenLoader {
  __device__ __forceinline__ cplx operator()(const cplx *p) const {
    const double2 v = __ldcg(reinterpret_cast<const double2 *>(p));
    return cmake(v.x, v.y);
  }
};

// dynamic shared memory layout (bytes):
//   acc   (k+1)*N u64
//   F     l*(k+1)*M cplx
//   out   (k+1)*M cplx
//   a_hat (n+1) u32 (classic)  |  degs 16 u32 (multi-bit)
static inline size_t generic_smem_bytes(uint32_t n, uint32_t k, uint32_t N,
                                        uint32_t l) {
  const size_t M = N / 2;
  return (size_t)(k + 1) * N * 8 + (size_t)l * (k + 1) * M * 16 +
         (size_t)(k + 1) * M * 16 + ((size_t)n + 1 + 16) * 4 + 64;
}

// GLOBAL_WS = false: the working set of one LWE lives in dynamic shared memory,
// grid = num_samples.  GLOBAL_WS = true: parameter sets whose working set does
// not fit one SM's shared memory (N >= 8192, e.g. PARAM_MESSAGE_3_CARRY_3 with
// N = 8192, l = 2: 640 KiB) keep it in a per-CTA slice of a global workspace
// (L2 resident: a few hundred CTAs x < 1 MiB) and a persistent grid strides
// over the samples -- the role of the reference's "no shared memory" variants
// (programmable_bootstrap_classic.cuh: get_buffer_size_full_sm_.. / partial_sm).
//
template <int NTHREADS, bool GLOBAL_WS = false, typename Torus = uint64_t>
__global__ void __launch_bounds__(NTHREADS)
pbs_generic_kernel(Torus *__restrict__ lwe_out,
                   const Torus *__restrict__ out_idx,
                   const Torus *__restrict__ luts,
                   const Torus *__restrict__ lut_idx,
                   const Torus *__restrict__ lwe_in,
                   const Torus *__restrict__ in_idx,
                   const cplx *__restrict__ bsk, const cplx *__restrict__ tw,
                   const cplx *__restrict__ root, uint32_t n, uint32_t k,
                   uint32_t N, uint32_t logM, uint32_t base_log, uint32_t l,
                   uint32_t grouping, uint32_t num_many_lut,
                   uint32_t lut_stride, int centered_ms,
                   int ties_even = 1, uint32_t num_samples = 0,
                   unsigned char *ws = nullptr, size_t ws_stride = 0) {
  extern __shared__ __align__(16) unsigned char smem_dyn[];
  unsigned char *smem_raw =
      GLOBAL_WS ? ws + (size_t)blockIdx.x * ws_stride : smem_dyn;
  if (!GLOBAL_WS)
    num_samples = gridDim.x;
  const uint32_t M = N >> 1;
  uint64_t *acc = reinterpret_cast<uint64_t *>(smem_raw);
  cplx *F = reinterpret_cast<cplx *>(acc + (size_t)(k + 1) * N);
  cplx *out = F + (size_t)l * (k + 1) * M;
  uint32_t *a_hat = reinterpret_cast<uint32_t *>(out + (size_t)(k + 1) * M);
  __shared__ unsigned long long red_half[NTHREADS / 32];
  __shared__ long long red_dbl[NTHREADS / 32];
  __shared__ uint32_t b_hat_s;

  const uint32_t tid = threadIdx.x;
  const uint32_t log_mod = logM + 2; // log2(2N)
  const bool multibit = grouping > 1;
  for (uint32_t s = blockIdx.x; s < num_samples; s += gridDim.x) {
  using Io = TorusIo<Torus>;
  const Torus *ct = lwe_in + (uint64_t)in_idx[s] * (uint64_t)(n + 1);

  // ---- modulus switch --------------------------------------------------
  if (!multibit) {
    CenteredMsSums sums;
    for (uint32_t i = tid; i < n; i += NTHREADS) {
      const uint64_t a = Io::widen(ct[i]);
      a_hat[i] = modulus_switch_u64(a, log_mod);
      if (centered_ms)
        sums.add(a, log_mod);
    }
    if (centered_ms)
      centered_ms_publish_warp(sums, red_half, red_dbl);
  }
  __syncthreads();
  if (tid == 0)
    b_hat_s = ms_b_hat(Io::widen(ct[n]), !multibit && centered_ms, red_half, red_dbl,
                       NTHREADS / 32, log_mod);
  __syncthreads();
  rotate_lut(acc, N, luts + (uint64_t)lut_idx[s] * (uint64_t)((k + 1) * N), k + 1, N,
             b_hat_s, tid, NTHREADS, [](Torus x) { return Io::widen(x); });
  __syncthreads();

  const uint32_t nggsw = multibit ? (1u << grouping) : 1u;
  const uint32_t steps = multibit ? n / grouping : n;
  const size_t ggsw_len = (size_t)l * (k + 1) * (k + 1) * M;
  uint32_t *degs = a_hat; // multi-bit reuses the area (16 entries)

  for (uint32_t i = 0; i < steps; i++) {
    uint32_t a = 0;
    if (multibit) {
      // degrees of the 2^g - 1 rotated GGSWs of this group
      if (tid < nggsw) {
        uint64_t sum = 0;
        for (uint32_t u = 0; u < grouping; u++)
          if ((tid >> (grouping - 1 - u)) & 1u)
            sum += Io::widen(ct[i * grouping + u]);
        degs[tid] = modulus_switch_u64(sum, log_mod);
      }
    } else {
      a = a_hat[i];
      if (a == 0)
        continue;
    }
    gen_decompose(acc, F, N, k, base_log, l, a, multibit, tid, NTHREADS,
                  ties_even != 0);
    __syncthreads();
    for (uint32_t L = 1; L <= logM; L++) {
      gen_fwd_level(F, logM, L, tw, l * (k + 1), tid, NTHREADS);
      __syncthreads();
    }
    gen_mac(F, out, bsk + (size_t)i * nggsw * ggsw_len, N, k, l, nggsw, degs,
            root, tid, NTHREADS, GenLoader());
    __syncthreads();
    for (uint32_t L = logM; L >= 1; L--) {
      gen_inv_level(out, logM, L, tw, k + 1, tid, NTHREADS);
      __syncthreads();
    }
    gen_acc_update(acc, out, N, k, multibit, tid, NTHREADS);
    __syncthreads();
  }

  sample_extract_many_lut(lwe_out, (uint64_t)out_idx[s], num_samples, num_many_lut,
                          lut_stride, acc, N, k, N, tid, NTHREADS,
                          [](uint64_t x) { return Io::narrow(x); });
  __syncthreads(); // the working set is reused by the next sample of this CTA
  } // sample loop
}

// standard-domain polynomial -> spectrum (scaled by 2^-64 / M), natural slot
// order, same [..][t][r][c] nesting as the source.  grid = #polynomials.
template <typename Torus = uint64_t>
__global__ void __launch_bounds__(256)
bsk_convert_generic_kernel(cplx *__restrict__ dst,
                           const Torus *__restrict__ src,
                           const cplx *__restrict__ tw, uint32_t N,
                           uint32_t logM) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  cplx *buf = reinterpret_cast<cplx *>(smem_raw);
  const uint32_t M = N >> 1, tid = threadIdx.x;
  const Torus *p = src + (size_t)blockIdx.x * N;
  const double scale = ldexp(1.0, -64 - (int)logM);
  for (uint32_t j = tid; j < M; j += 256)
    buf[j] = cmake(
        ll_to_double((int64_t)TorusIo<Torus>::widen(p[j])) * scale,
        ll_to_double((int64_t)TorusIo<Torus>::widen(p[j + M])) * scale);
  __syncthreads();
  for (uint32_t L = 1; L <= logM; L++) {
    gen_fwd_level(buf, logM, L, tw, 1, tid, 256);
    __syncthreads();
  }
  cplx *o = dst + (size_t)blockIdx.x * M;
  for (uint32_t j = tid; j < M; j += 256)
    o[j] = buf[j];
}

} // namespace b200
