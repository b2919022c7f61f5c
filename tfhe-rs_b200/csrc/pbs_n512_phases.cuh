// pbs_n512_phases.cuh -- arithmetic of the N = 512, l = 1, k <= 4 register
// PBS kernel (pbs_n512.cuh): rotate + decompose, the Fourier MAC of the key
// ring mode, the accumulator update and the key conversion's load.  Shared by the
// CUDA kernels and the CPU replay (tests/emu/emu_p22.cpp).
#pragma once
#include "negacyclic_fft.cuh"
#include "pbs_n2048_phases.cuh"

#define P512_N 512
#define P512_M 256

// rotate + decompose for N = 512 (p22v4_load_digits with stride 16): thread u
// holds complex coefficients j = 16*j1 + u (re <- coefficient j, im <- j + 256)
B200_HD void n512_load_digits(const uint32_t *acc_p, int u,
                                                 uint32_t a, uint32_t base_log,
                                                 const uint32_t own[32],
                                                 cplx v[16]) {
  const uint32_t d = a & (P512_N - 1);
  const bool neg0 = (a >> 9) != 0u; // a >= N
  const uint32_t half = 1u << (31 - base_log);
  const uint32_t sh = 32 - base_log;
  const int32_t tie_below = (int32_t)(0x80000000u + half);
  const int32_t plus_half_base = (int32_t)(1u << (base_log - 1));
  const uint32_t base4 = ((uint32_t)u - d) * 4u; // 4 * (j - d) for j1 = 0
  const unsigned char *accb = reinterpret_cast<const unsigned char *>(acc_p);
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    const uint32_t ub0 = base4 + 64u * j1;       // 4 * (j - d)
    const uint32_t ub1 = ub0 + 4u * P512_M;      // 4 * (j + M - d)
    const uint32_t ib0 = ub0 & (4u * P512_N - 4u);
    const uint32_t r0 = *reinterpret_cast<const uint32_t *>(accb + ib0);
    const uint32_t r1 =
        *reinterpret_cast<const uint32_t *>(accb + (ib0 ^ (4u * P512_M)));
    const bool n0 = ((int32_t)ub0 < 0) != neg0;
    const bool n1 = ((int32_t)ub1 < 0) != neg0;
    const uint32_t x0 = n0 ? (0u - r0) - own[j1] : r0 - own[j1];
    const uint32_t x1 = n1 ? (0u - r1) - own[16 + j1] : r1 - own[16 + j1];
    int32_t d0 = (int32_t)(x0 + half) >> sh;
    int32_t d1 = (int32_t)(x1 + half) >> sh;
    // balanced tie (decomposer.rs:163-188): x in [2^31, 2^31 + half) -> +B/2
    if ((int32_t)x0 < tie_below)
      d0 = plus_half_base;
    if ((int32_t)x1 < tie_below)
      d1 = plus_half_base;
    v[j1] = cmake(int_to_double(d0), int_to_double(d1));
  }
}

B200_HD void n512_acc_update(uint32_t *acc_p, int u,
                                                const cplx v[16],
                                                uint32_t own[32]) {
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    const uint32_t j = 16u * j1 + (uint32_t)u;
    // own[] is the current accumulator word: no read of shared memory
    own[j1] += scaled_double_to_torus32(v[j1].re);
    own[16 + j1] += scaled_double_to_torus32(v[j1].im);
    acc_p[j] = own[j1];
    acc_p[j + P512_M] = own[16 + j1];
  }
}

// Fourier MAC of the ring mode for thread (column p, element u): out[b] =
// sum_r spec_r[b][u] * key[p][r][b][u] from the step's key block `kcol` (the
// P rows of column p).  The thread's own spectrum (row p) is still in v, so the
// sum starts at row r = p and walks the other rows cyclically; xs_l holds the
// P spectra of the LWE.
template <int P, typename Load>
B200_HD void n512_mac_ring(cplx v[16], const cplx *xs_l, const cplx *kcol, int p,
                           int u, Load load) {
  {
    const cplx *kp = kcol + (size_t)p * P512_M + u;
#pragma unroll
    for (int b = 0; b < 16; b++)
      v[b] = cmul(v[b], load(kp + b * 16));
  }
#pragma unroll
  for (int rr = 1; rr < P; rr++) {
    int r = p + rr;
    if (r >= P)
      r -= P;
    const cplx *fr = xs_l + (size_t)r * P512_M + u;
    const cplx *kr = kcol + (size_t)r * P512_M + u;
#pragma unroll
    for (int b = 0; b < 16; b++)
      v[b] = cfma(fr[b * 16], load(kr + b * 16), v[b]);
  }
}

// key conversion: thread u's 16 complex values of the standard-domain
// polynomial src_p, scaled by 2^-64 / 256 * 2^32 = 2^-40
B200_HD void n512_key_load(const uint64_t *src_p, int u, cplx v[16]) {
  const double scale = 9.094947017729282379150390625e-13;
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    const uint32_t j = 16u * j1 + u;
    v[j1] = cmake(ll_to_double((int64_t)src_p[j]) * scale,
                  ll_to_double((int64_t)src_p[j + P512_M]) * scale);
  }
}
