// pbs_generic_phases.cuh -- phases of the any-(N, k, l) PBS kernel (classic
// and multi-bit).  Same transform as negacyclic_fft.cuh (twist-free,
// slot `pos` = value at t^(1 + 4*bitrev(pos))) but done with plain radix-2
// levels on shared memory so that it works for every power-of-two N.  Shared
// by the CUDA kernels (pbs_generic.cuh) and the CPU CTA emulator (tests/emu).
//
// Reference semantics: see pbs_n2048_phases.cuh; multi-bit additionally
//   algorithms/lwe_multi_bit_programmable_bootstrapping.rs:30-65 (degrees),
//   :116-156 (bundle = sum_s GGSW_s * X^deg_s), :806-845 (acc <- bundle (x) acc)
#pragma once
#include "pbs_n2048_phases.cuh"

// twiddle table for size M = 2^logM: entry (2^(L-1) - 1 + u) = tw(L, u),
// L = 1..logM, u < 2^(L-1)  -> M - 1 entries.  root table: 4M entries,
// root[e] = exp(i pi e / (2M)) (the 2N-th roots, for multi-bit monomials).
// host-side table generation
static inline void b200_fill_generic_tables(uint32_t logM, cplx *tw,
                                            cplx *root) {
  for (uint32_t L = 1; L <= logM; L++)
    for (uint32_t u = 0; u < (1u << (L - 1)); u++)
      tw[(1u << (L - 1)) - 1 + u] = b200_tw(logM, L, u);
  if (root) {
    const long double pi = 3.14159265358979323846264338327950288L;
    const uint32_t cnt = 4u << logM;
    for (uint32_t e = 0; e < cnt; e++) {
      const long double a = pi * (long double)e / (long double)(2u << logM);
      root[e].re = (double)cosl(a);
      root[e].im = (double)sinl(a);
    }
  }
}

// Torus = uint64_t: the 64-bit ABI.  Torus = uint32_t: the u32 torus of
// cuda_programmable_bootstrap_lwe_ciphertext_vector_32_async (ciphertexts,
// accumulators AND index vectors are u32, programmable_bootstrap.h:72-79): words
// are widened to the top half of a u64 on the way in and rounded back to 32
// bits on the way out; the blind rotation itself is the same 64-bit path.
template <typename Torus> struct TorusIo {
  static constexpr uint32_t SHIFT = 64 - 8 * sizeof(Torus);
  B200_HD static uint64_t widen(Torus x) {
    return (uint64_t)x << SHIFT;
  }
  B200_HD static Torus narrow(uint64_t x) {
    if constexpr (SHIFT == 0)
      return (Torus)x;
    else
      return (Torus)((x + ((uint64_t)1 << (SHIFT - 1))) >> SHIFT);
  }
};

// one forward level L over `npolys` consecutive polynomials of M complex
B200_HD void gen_fwd_level(cplx *buf, uint32_t logM, uint32_t L,
                           const cplx *tw, uint32_t npolys, uint32_t tid,
                           uint32_t nthreads) {
  const uint32_t M = 1u << logM, h = M >> L; // pair distance
  const uint32_t total = npolys * (M >> 1);
  for (uint32_t w = tid; w < total; w += nthreads) {
    const uint32_t poly = w >> (logM - 1), bf = w & ((M >> 1) - 1);
    const uint32_t u = bf / h, off = bf % h;
    cplx *p = buf + (size_t)poly * M + u * 2 * h + off;
    const cplx s = tw[(1u << (L - 1)) - 1 + u];
    const cplx a = p[0], t = cmul(s, p[h]);
    p[0] = cadd(a, t);
    p[h] = csub(a, t);
  }
}
// inverse of the same level, up to a factor 2
B200_HD void gen_inv_level(cplx *buf, uint32_t logM, uint32_t L,
                           const cplx *tw, uint32_t npolys, uint32_t tid,
                           uint32_t nthreads) {
  const uint32_t M = 1u << logM, h = M >> L;
  const uint32_t total = npolys * (M >> 1);
  for (uint32_t w = tid; w < total; w += nthreads) {
    const uint32_t poly = w >> (logM - 1), bf = w & ((M >> 1) - 1);
    const uint32_t u = bf / h, off = bf % h;
    cplx *p = buf + (size_t)poly * M + u * 2 * h + off;
    const cplx s = tw[(1u << (L - 1)) - 1 + u];
    const cplx A = p[0], B = p[h];
    p[0] = cadd(A, B);
    p[h] = cmulc(csub(A, B), s);
  }
}

// generic signed decomposition state (decomposer.rs:163-188, iter.rs:131-151)
B200_HD uint64_t decomp_init_state(uint64_t x, uint32_t base_log,
                                   uint32_t level_count) {
  const uint32_t R = base_log * level_count;
  uint64_t r = x >> (64 - R - 1);
  const uint64_t rb = r & 1u;
  r = (r + 1) >> 1;
  r &= (R == 64) ? ~(uint64_t)0 : (((uint64_t)1 << R) - 1);
  const uint64_t bal = (((r - 1) | (rb << (R - 1))) & r) >> (R - 1);
  return r - (bal << R);
}
// same, with an exact tie of the dropped bits rounded to EVEN instead of up.
// Used by the multi-bit PBS paths only: their accumulator is re-assigned from
// f64 every step and is therefore a multiple of a large power of two (the f64
// ulp of the pre-wrap sum), so exact ties are common -- 1 in 8 for g = 4 -- and
// always-up biases every coefficient the same way (see digits_u32 in
// pbs_multibit_n2048_phases.cuh for the measured effect).  The keyswitch and
// the classic PBS keep the reference rule above.
B200_HD uint64_t decomp_init_state_even(uint64_t x, uint32_t base_log,
                                        uint32_t level_count) {
  const uint32_t R = base_log * level_count;
  const uint32_t drop = 64 - R; // >= 1
  const uint64_t low = x & (((uint64_t)1 << drop) - 1);
  const uint64_t half = (uint64_t)1 << (drop - 1);
  const uint64_t q = x >> drop;
  const uint64_t rb = (uint64_t)((low > half) | ((low == half) & (q & 1u)));
  uint64_t r = (q + rb) & ((((uint64_t)1 << R) - 1));
  const uint64_t bal = (((r - 1) | (rb << (R - 1))) & r) >> (R - 1);
  return r - (bal << R);
}
B200_HD int64_t decomp_next_digit(uint64_t *state, uint32_t base_log) {
  const uint64_t mask = ((uint64_t)1 << base_log) - 1;
  const uint64_t res = *state & mask;
  uint64_t st = (uint64_t)((int64_t)*state >> base_log);
  const uint64_t carry = (((res - 1) | st) & res) >> (base_log - 1);
  st += carry;
  *state = st;
  return (int64_t)(res - (carry << base_log));
}

// (p * X^a)[j] - p[j] for general N (a in [1, 2N)), or p[j] itself if a == 0
B200_HD uint64_t gen_rot_sub_coeff(const uint64_t *p, uint32_t N, uint32_t j,
                                   uint32_t a) {
  const uint32_t d = a & (N - 1);
  const bool neg0 = a >= N;
  const bool wrap = j < d;
  const uint32_t jj = wrap ? j + N - d : j - d;
  const uint64_t x = p[jj];
  return ((neg0 != wrap) ? (uint64_t)0 - x : x) - p[j];
}

// phase: decompose the (k+1) polynomials of ct1 (= acc*X^a - acc, or acc when
// `multibit`) into F[t][r][j] = (digit_t(j), digit_t(j+M))
B200_HD void gen_decompose(const uint64_t *acc, cplx *F, uint32_t N,
                           uint32_t k, uint32_t base_log, uint32_t l,
                           uint32_t a, bool multibit, uint32_t tid,
                           uint32_t nthreads, bool ties_even = true) {
  const uint32_t M = N >> 1;
  const uint32_t total = (k + 1) * M;
  const bool even = multibit && ties_even;
  for (uint32_t w = tid; w < total; w += nthreads) {
    const uint32_t r = w / M, j = w % M;
    const uint64_t *p = acc + (size_t)r * N;
    const uint64_t x0 = multibit ? p[j] : gen_rot_sub_coeff(p, N, j, a);
    const uint64_t x1 = multibit ? p[j + M] : gen_rot_sub_coeff(p, N, j + M, a);
    uint64_t s0 = even ? decomp_init_state_even(x0, base_log, l)
                       : decomp_init_state(x0, base_log, l);
    uint64_t s1 = even ? decomp_init_state_even(x1, base_log, l)
                       : decomp_init_state(x1, base_log, l);
    for (uint32_t t = 0; t < l; t++) {
      const int64_t d0 = decomp_next_digit(&s0, base_log);
      const int64_t d1 = decomp_next_digit(&s1, base_log);
      F[((size_t)t * (k + 1) + r) * M + j] =
          cmake(ll_to_double(d0), ll_to_double(d1));
    }
  }
}

// bit reversal of the low `bits` bits
B200_HD uint32_t gen_bitrev(uint32_t x, uint32_t bits) {
#if defined(__CUDA_ARCH__)
  return __brev(x) >> (32 - bits);
#else
  uint32_t r = 0;
  for (uint32_t i = 0; i < bits; i++)
    if (x & (1u << i))
      r |= 1u << (bits - 1 - i);
  return r;
#endif
}

// phase: out[c][pos] = sum_{t,r} F[t][r][pos] * G[t][r][c][pos] where, for
// multi-bit, G = sum_s B_s * X^{deg_s} evaluated at slot pos.  `ggsw` points
// at the first GGSW of the step ([s][t][r][c][M] for multi-bit).
template <typename LoadBsk>
B200_HD void gen_mac(const cplx *F, cplx *out, const cplx *ggsw, uint32_t N,
                     uint32_t k, uint32_t l, uint32_t nggsw,
                     const uint32_t *degs, const cplx *root, uint32_t tid,
                     uint32_t nthreads, LoadBsk load_bsk) {
  const uint32_t M = N >> 1;
  uint32_t logM = 0;
  while ((1u << logM) < M)
    logM++;
  const size_t ggsw_len = (size_t)l * (k + 1) * (k + 1) * M;
  for (uint32_t pos = tid; pos < M; pos += nthreads) {
    cplx mono[15]; // nggsw - 1 <= 15 (grouping factor <= 4)
    if (nggsw > 1) {
      const uint32_t kf = gen_bitrev(pos, logM);
      for (uint32_t s = 1; s < nggsw; s++) {
        const uint32_t e = (degs[s] * (1u + 4u * kf)) & (2 * N - 1);
        mono[s - 1] = root[e];
      }
    }
    for (uint32_t c = 0; c <= k; c++) {
      cplx accu = cmake(0.0, 0.0);
      for (uint32_t t = 0; t < l; t++)
        for (uint32_t r = 0; r <= k; r++) {
          const size_t off =
              (((size_t)t * (k + 1) + r) * (k + 1) + c) * M + pos;
          cplx gval = load_bsk(ggsw + off);
          for (uint32_t s = 1; s < nggsw; s++)
            gval = cfma(load_bsk(ggsw + s * ggsw_len + off), mono[s - 1], gval);
          accu = cfma(F[((size_t)t * (k + 1) + r) * M + pos], gval, accu);
        }
      out[(size_t)c * M + pos] = accu;
    }
  }
}

// phase: acc (+)= torus(out)
B200_HD void gen_acc_update(uint64_t *acc, const cplx *out, uint32_t N,
                            uint32_t k, bool assign, uint32_t tid,
                            uint32_t nthreads) {
  const uint32_t M = N >> 1;
  const uint32_t total = (k + 1) * M;
  for (uint32_t w = tid; w < total; w += nthreads) {
    const uint32_t c = w / M, j = w % M;
    const cplx v = out[w];
    uint64_t *p = acc + (size_t)c * N;
    const uint64_t a0 = double_to_torus64(v.re), a1 = double_to_torus64(v.im);
    if (assign) {
      p[j] = a0;
      p[j + M] = a1;
    } else {
      p[j] += a0;
      p[j + M] += a1;
    }
  }
}
