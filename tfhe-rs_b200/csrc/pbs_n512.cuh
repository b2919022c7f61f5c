// pbs_n512.cuh -- sm_90a register-FFT classic PBS for (N = 512, l = 1,
// k <= 4): PARAM_MESSAGE_1_CARRY_1_KS_PBS (n = 879, k = 4, log B = 23;
// tfhe/src/shortint/parameters/v1_0/classic/tuniform/p_fail_2_minus_128/
// ks_pbs.rs:11-21) and its relatives.  Round 1 and the reference's CUDA backend
// both run this set on generic shared-memory FFT kernels; this is the (2048, 1, 1) design re-cut for a
// transform of 256 complex points.
//
// Replaces host_programmable_bootstrap / device_programmable_bootstrap_*
// (backends/tfhe-cuda-backend/cuda/src/pbs/programmable_bootstrap_classic.cuh)
// for these shapes; restates FourierLweBootstrapKeyView::bootstrap
// (fft64/crypto/bootstrap.rs:294-380,480-520).
//
//   * M = 256 = 16 x 16: 16 threads per polynomial, 16 complex values per thread
//     in registers, ONE exchange per transform -- a 16 x 16 transpose inside a
//     half-warp, ordered by __syncwarp (negacyclic_fft.cuh, xq_*);
//   * one LWE = (k+1) polynomials = 16 (k+1) threads; G LWEs share a CTA and run
//     in lock step, so the Fourier key block of a step (n.b. 100 KiB for k = 4)
//     is requested by G thread groups at once and the second request hits L1;
//   * the accumulator polynomial p is only ever touched by its own 16 threads
//     (rotation stays inside a polynomial): u32 words in shared memory, the
//     thread's own 32 words handed over in registers (p22v4 scheme), warp-level
//     synchronisation; two CTA barriers per step, around the Fourier MAC;
//   * Fourier key layout: [i][column c][row r][b < 16][q < 16] complex128,
//     value at slot pos = 16 q + b, pre-scaled by 2^-64 / 256 * 2^32; thread
//     (c, q) reads 16 contiguous bytes per (r, b), a half-warp 256 contiguous.
#pragma once
#include "pbs_n2048.cuh" // ldcg_cplx, phases
#include "pbs_n512_phases.cuh"

#include <cuda_runtime.h>

namespace b200 {

__constant__ cplx c_fft256_pass1[15];

// read-only, L1-cacheable (small tables shared by every thread group)
__device__ __forceinline__ cplx ldnc_cplx(const cplx *p) {
  const double2 v = __ldg(reinterpret_cast<const double2 *>(p));
  return cmake(v.x, v.y);
}

// key loader of the ring mode's MAC: the shared ring
struct SmemLoader {
  __device__ __forceinline__ cplx operator()(const cplx *p) const { return *p; }
};

// RING: the Fourier key block of a step ((k+1)^2 x 4 KiB, contiguous in the
// layout below) is brought into shared memory by the TMA unit a whole step ahead
// (one slot, cp.async.bulk + mbarrier, as in pbs_n2048_k1_l1_v6_kernel) and is
// shared by the G LWEs of the CTA; one CTA per SM.  !RING: every thread streams
// its key values from L2 through a 3-chunk register ring; two CTAs per SM.
template <int K, int G, bool RING = false>
struct N512Smem {
  static constexpr int P = K + 1;
  cplx xs[G][P][P512_M];       // exchange buffer, then shared spectrum  4 KiB each
  cplx ring[RING ? P * P : 1][RING ? P512_M : 1];
  // rows padded by 16 words: the two polynomials of a warp then sit 16 banks
  // apart and their 32-bit rotated reads / updates do not collide
  uint32_t acc[G][P][P512_N + 16];
  uint16_t a_hat[G][1024 + 8];
  uint32_t b_hat[G];
  unsigned long long red_half[G][4];
  long long red_dbl[G][4];
  unsigned long long bar;
};

// persistent grid (see below), block = 16 (K+1) G
template <int K, int G, bool RING = false>
__global__ void __launch_bounds__(16 * (K + 1) * G, RING ? 1 : 2)
pbs_n512_kernel(uint64_t *__restrict__ lwe_out,
                const uint64_t *__restrict__ out_idx,
                const uint64_t *__restrict__ luts,
                const uint64_t *__restrict__ lut_idx,
                const uint64_t *__restrict__ lwe_in,
                const uint64_t *__restrict__ in_idx,
                const cplx *__restrict__ bsk,
                const Fft256Tables *__restrict__ tables, uint32_t n,
                uint32_t base_log, uint32_t num_samples, uint32_t num_many_lut,
                uint32_t lut_stride, int centered_ms) {
  constexpr int P = K + 1;
  constexpr int TPL = 16 * P; // threads per LWE
  constexpr int NT = TPL * G;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using Smem = N512Smem<K, G, RING>;
  Smem &sm = *reinterpret_cast<Smem *>(smem_raw);
  const int tid = threadIdx.x;
  [[maybe_unused]] auto tma_issue = [&](uint32_t i) {
    if constexpr (RING) {
      constexpr uint32_t bytes = (uint32_t)(P * P * P512_M * sizeof(cplx));
      constexpr uint32_t piece = (uint32_t)(P * P512_M * sizeof(cplx)); // one column
      mbar_arrive_expect_tx(&sm.bar, bytes);
#pragma unroll
      for (int c = 0; c < P; c++)
        tma_bulk_g2s(&sm.ring[c * P][0],
                     bsk + (size_t)i * (P * P * P512_M) + (size_t)c * (P * P512_M),
                     piece, &sm.bar);
    }
  };
  if constexpr (RING) {
    if (tid == 0) {
      mbar_init(&sm.bar, 1);
      mbar_fence_init();
    }
    __syncthreads();
  }
  [[maybe_unused]] uint32_t ring_phase = 0; // completed copies so far (parity of the wait)
  const int lw = tid / TPL;          // LWE of this CTA
  const int tl = tid - lw * TPL;     // thread inside the LWE
  const int p = tl >> 4;             // polynomial (= output column in the MAC)
  const int u = tl & 15;             // thread inside the polynomial
  const uint32_t log_mod = 10;       // log2(2N)
  // PERSISTENT grid: at most two CTAs per SM are launched and every CTA walks the
  // sample list with the grid as stride.  All resident CTAs then sit at (nearly)
  // the same CMUX step at any time, so the slice of the Fourier key in use -- a
  // few steps x 100 KiB for k = 4 -- stays in L2.  The whole key of this set
  // (90 MB) does not fit one L2 partition: with one CTA per sample pair and
  // waves starting at different times the kernel streamed it from HBM again
  // for every wave.
  for (uint32_t grp = blockIdx.x; grp * G < num_samples; grp += gridDim.x) {
  // the last group may hold fewer than G samples: the spare thread groups replay
  // the last sample (all barriers are CTA wide) and do not write
  const uint32_t s_raw = grp * G + lw;
  const bool live = s_raw < num_samples;
  const uint32_t s = live ? s_raw : num_samples - 1;

  // ---- prologue: modulus switch (standard or centered mean) ---------------
  const uint64_t *ct = lwe_in + in_idx[s] * (uint64_t)(n + 1);
  if (tl == 0) {
    sm.red_half[lw][0] = 0;
    sm.red_dbl[lw][0] = 0;
  }
  __syncthreads();
  {
    CenteredMsSums sums;
    for (uint32_t i = tl; i < n; i += TPL) {
      const uint64_t a = ct[i];
      sm.a_hat[lw][i] = (uint16_t)modulus_switch_u64(a, log_mod);
      if (centered_ms)
        sums.add(a, log_mod);
    }
    // per-LWE reduction through shared memory (TPL is not a warp multiple)
    if (centered_ms)
      centered_ms_publish_atomic(sums, &sm.red_half[lw][0], &sm.red_dbl[lw][0]);
  }
  __syncthreads();
  if (tl == 0)
    sm.b_hat[lw] = ms_b_hat(ct[n], centered_ms, &sm.red_half[lw][0],
                            &sm.red_dbl[lw][0], 1, log_mod);
  __syncthreads();
  // ---- prologue: acc = LUT * X^{-b_hat} ------------------------------------
  {
    const uint64_t *lut = luts + lut_idx[s] * (uint64_t)(P * P512_N);
    const uint32_t b_hat = sm.b_hat[lw];
    for (uint32_t j = tl; j < (uint32_t)(P * P512_N); j += TPL) {
      const uint32_t r = j >> 9, jj = j & (P512_N - 1);
      sm.acc[lw][r][jj] =
          torus64_to_32(rot_div_coeff(lut + r * P512_N, P512_N, jj, b_hat));
    }
  }
  __syncthreads();

  uint32_t *acc_p = sm.acc[lw][p];
  cplx *xs_p = sm.xs[lw][p];
  const cplx *xs_l = &sm.xs[lw][0][0];
  const cplx *tw2_src = &tables->pass2[u][0];
  uint32_t own[32];
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    own[j1] = acc_p[16 * j1 + u];
    own[16 + j1] = acc_p[16 * j1 + u + P512_M];
  }
  // (GGSW i, column p) block = [row r][b][q]; this thread reads element q = u
  const cplx *key_col = bsk + (size_t)p * (P * P512_M) + u;
  const size_t key_step = (size_t)P * P * P512_M;

  if constexpr (RING) {
    if (tid == 0 && n > 0)
      tma_issue(0); // the slot is free: every reader of the previous group passed a barrier
  }
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t a = sm.a_hat[lw][i];
    cplx v[16];
    n512_load_digits(acc_p, u, a, base_log, own, v);
    radix16_fwd(v, c_fft256_pass1);
    xq_store_p1(xs_p, u, v);
    __syncwarp();
    xq_load_p2(xs_p, u, v);
    {
      cplx tw2[15];
#pragma unroll
      for (int e = 0; e < 15; e++)
        tw2[e] = ldnc_cplx(tw2_src + e);
      radix16_fwd(v, tw2);
    }
    __syncwarp(); // every lane has read its exchange values
    spec256_store(xs_p, u, v);
    if constexpr (RING) {
      __syncthreads();
      mbar_wait_parity(&sm.bar, ring_phase & 1u);
      ring_phase++;
      // ---- Fourier MAC from shared memory ------------------------------------
      // the thread's own spectrum is still in registers: start with row r = p,
      // then walk the other rows cyclically (16 fewer 128-bit loads per thread)
      n512_mac_ring<P>(v, xs_l, &sm.ring[p * P][0], p, u, SmemLoader());
    } else {
    // the Fourier key of the step streams through a ring of three 8-value chunks
    // (two chunks = 16 x 128-bit loads in flight per thread); the first two are
    // requested before the share barrier
    const cplx *krow = key_col + (size_t)i * key_step;
    cplx kbuf[3][8];
    auto key_chunk = [&](int ch, cplx (&dst)[8]) {
      const int r = ch >> 1, hb = (ch & 1) * 8;
#pragma unroll
      for (int b = 0; b < 8; b++)
        dst[b] = ldcg_cplx(krow + (size_t)r * P512_M + (hb + b) * 16);
    };
    key_chunk(0, kbuf[0]);
    key_chunk(1, kbuf[1]);
    __syncthreads();
    // ---- Fourier MAC: out[b] = sum_r spec_r[b][q] * key[i][p][r][b][q] -------
    // (restated by the CPU replay, tests/emu/emu_p22.cpp n512_mac_regs: moved
    // into a shared function, this loop changes the instances' register
    // allocation)
#pragma unroll
    for (int ch = 0; ch < 2 * P; ch++) {
      const int r = ch >> 1, hb = (ch & 1) * 8;
      if (ch + 2 < 2 * P)
        key_chunk(ch + 2, kbuf[(ch + 2) % 3]);
#pragma unroll
      for (int b = 0; b < 8; b++) {
        const cplx f = xs_l[(size_t)r * P512_M + (hb + b) * 16 + u];
        v[hb + b] = r == 0 ? cmul(f, kbuf[ch % 3][b]) : cfma(f, kbuf[ch % 3][b], v[hb + b]);
      }
    }
    }
    __syncthreads(); // every read of the shared spectra (and of the ring) done
    if constexpr (RING) {
      if (tid == 0 && i + 1 < n)
        tma_issue(i + 1);
    }
    {
      cplx tw2[15];
#pragma unroll
      for (int e = 0; e < 15; e++)
        tw2[e] = ldnc_cplx(tw2_src + e);
      radix16_inv(v, tw2);
    }
    xq_store_p2(xs_p, u, v);
    __syncwarp();
    xq_load_p1(xs_p, u, v);
    radix16_inv(v, c_fft256_pass1);
    n512_acc_update(acc_p, u, v, own);
    __syncwarp(); // the polynomial's 16 threads are its only readers
  }
  __syncthreads();

  // ---- epilogue: sample extract (a16), optional many-LUT --------------------
  if (live) {
    const uint64_t out_len = (uint64_t)K * P512_N + 1;
    for (uint32_t m = 0; m < num_many_lut; m++) {
      const uint32_t nth = m * lut_stride;
      uint64_t *out =
          lwe_out + ((uint64_t)m * num_samples + out_idx[s]) * out_len;
      for (uint32_t w = tl; w < (uint32_t)(K * P512_N); w += TPL) {
        const uint32_t r = w >> 9, tt = w & (P512_N - 1);
        const uint32_t x = tt <= nth ? sm.acc[lw][r][nth - tt]
                                     : 0u - sm.acc[lw][r][P512_N + nth - tt];
        out[w] = (uint64_t)x << 32;
      }
      if (tl == 0)
        out[(size_t)K * P512_N] = (uint64_t)sm.acc[lw][K][nth] << 32;
    }
  }
  __syncthreads(); // the working set is reused by the next sample group
  } // persistent loop
  (void)NT;
}

// ---------------------------------------------------------------------------
// BSK conversion for this kernel: standard-domain u64 polynomial, source order
// [i][row r][column c][N] (level count 1) -> spectrum scaled by 2^-64 / 256 *
// 2^32, stored at [i][c][r][b][q].  grid = n (k+1)^2 / 2 (two polynomials per
// warp), block = 32.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(32)
bsk_convert_n512_kernel(cplx *__restrict__ dst, const uint64_t *__restrict__ src,
                        const Fft256Tables *__restrict__ tables, uint32_t P,
                        uint32_t total_polys) {
  __shared__ cplx xb[2][P512_M];
  const int hw = threadIdx.x >> 4, u = threadIdx.x & 15;
  uint32_t poly = blockIdx.x * 2 + hw;
  const bool live = poly < total_polys;
  if (!live)
    poly = total_polys - 1;
  const uint32_t c = poly % P, r = (poly / P) % P, i = poly / (P * P);
  const uint64_t *src_p = src + (size_t)poly * P512_N;
  cplx v[16];
  n512_key_load(src_p, u, v);
  radix16_fwd(v, c_fft256_pass1);
  xq_store_p1(xb[hw], u, v);
  __syncwarp();
  xq_load_p2(xb[hw], u, v);
  radix16_fwd(v, tables->pass2[u]);
  if (live) {
    cplx *out = dst + (((size_t)i * P + c) * P + r) * P512_M;
    spec256_store(out, u, v);
  }
}

} // namespace b200
