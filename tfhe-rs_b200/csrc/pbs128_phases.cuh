// pbs128_phases.cuh -- phases of the 128-bit classic PBS (pbs128.cuh): the
// double-double negacyclic transform, the u128 signed decomposition, the
// spectral MAC and the rounding back into the u128 accumulator.  Shared by the
// CUDA kernels and the CPU model (tests/emu/emu_pbs128.cpp).
//
// The transform is the one of pbs_generic_phases.cuh in double-double: a
// polynomial of N coefficients is packed as M = N/2 complex values
// (p[j], p[j + M]), radix-2 levels, slot `pos` = value at t^(1 + 4*bitrev(pos))
// for t a primitive 2N-th root of unity.  It works in the integers' own scale:
// the key spectrum is divided by M at conversion so that the inverse levels
// (each a factor 2) return the exact negacyclic product plus rounding.
//
// Reference semantics (tfhe-rs, u128 torus):
//   commons/math/decomposition/decomposer.rs (SignedDecomposer::
//   init_decomposer_state: rounding of the dropped bits, balanced state),
//   commons/math/decomposition/iter.rs (digits, least significant first, the
//   balanced carry), algorithms/lwe_programmable_bootstrapping (CMUX
//   acc += GGSW (x) (acc * X^a - acc), sample extraction).
#pragma once
#include "dd.cuh"
#include "pbs_generic_phases.cuh"

// twiddle table for M = 2^logM, entry (2^(L-1) - 1 + u) = tw(L, u) of
// b200_tw in double-double: M - 1 entries (host)
static inline void b200_fill_dd_twiddles(uint32_t logM, ddc *tw) {
  for (uint32_t L = 1; L <= logM; L++)
    for (uint32_t u = 0; u < (1u << (L - 1)); u++) {
      const uint64_t e = (uint64_t)(1 + 4 * b200_bitrev(u, L - 1)) << (logM - L);
      tw[(1u << (L - 1)) - 1 + u] = dd_unit_root(e, (uint64_t)4 << logM);
    }
}

// one forward level L of one polynomial of M = 2^logM double-double values
B200_HD void p128_fwd_level(ddc *buf, uint32_t logM, uint32_t L,
                            const ddc *tw, uint32_t tid, uint32_t nthreads) {
  const uint32_t h = (1u << logM) >> L; // pair distance
  for (uint32_t bf = tid; bf < (1u << (logM - 1)); bf += nthreads) {
    const uint32_t u = bf / h, off = bf % h;
    ddc *p = buf + u * 2 * h + off;
    const ddc a = p[0], t = ddc_mul(tw[(1u << (L - 1)) - 1 + u], p[h]);
    p[0] = ddc_add(a, t);
    p[h] = ddc_sub(a, t);
  }
}
// inverse of the same level, up to a factor 2
B200_HD void p128_inv_level(ddc *buf, uint32_t logM, uint32_t L,
                            const ddc *tw, uint32_t tid, uint32_t nthreads) {
  const uint32_t h = (1u << logM) >> L;
  for (uint32_t bf = tid; bf < (1u << (logM - 1)); bf += nthreads) {
    const uint32_t u = bf / h, off = bf % h;
    ddc *p = buf + u * 2 * h + off;
    const ddc A = p[0], B = p[h];
    p[0] = ddc_add(A, B);
    p[h] = ddc_mulc(ddc_sub(A, B), tw[(1u << (L - 1)) - 1 + u]);
  }
}

// SignedDecomposer<u128>::init_decomposer_state (R = base_log * l <= 128)
B200_HD u128 decomp128_init_state(u128 x, uint32_t base_log, uint32_t l) {
  const uint32_t R = base_log * l;
  if (R == 128)
    return x; // every bit is represented: nothing to round
  u128 r = x >> (127 - R);
  const u128 rb = r & 1u;
  r = ((r + 1) >> 1) & ((((u128)1) << R) - 1);
  const u128 bal = (((r - 1) | (rb << (R - 1))) & r) >> (R - 1);
  return r - (bal << R);
}
// next digit, least significant first, with the balanced carry
B200_HD i128 decomp128_next_digit(u128 *state, uint32_t base_log) {
  const u128 mask = base_log >= 128 ? ~(u128)0 : (((u128)1) << base_log) - 1;
  const u128 res = *state & mask;
  u128 st = base_log >= 128 ? (u128)((i128)*state >> 127)
                            : (u128)((i128)*state >> base_log);
  const u128 carry = (((res - 1) | st) & res) >> (base_log - 1);
  st += carry;
  *state = st;
  return base_log >= 128 ? (i128)res : (i128)(res - (carry << base_log));
}

// (p * X^a)[j] - p[j] for a in [1, 2N)
B200_HD u128 p128_rot_sub(const u128 *p, uint32_t N, uint32_t j, uint32_t a) {
  const uint32_t d = a & (N - 1);
  const bool wrap = j < d;
  const u128 x = p[wrap ? j + N - d : j - d];
  return (((a >= N) != wrap) ? (u128)0 - x : x) - p[j];
}

// digit polynomial t (t = 0: least significant) of acc_r * X^a - acc_r into
// buf, as M double-double complex values
B200_HD void p128_decompose(const u128 *acc_r, ddc *buf, uint32_t N,
                            uint32_t a, uint32_t base_log, uint32_t l,
                            uint32_t t, uint32_t tid, uint32_t nthreads) {
  const uint32_t M = N >> 1;
  for (uint32_t j = tid; j < M; j += nthreads) {
    u128 s0 = decomp128_init_state(p128_rot_sub(acc_r, N, j, a), base_log, l);
    u128 s1 = decomp128_init_state(p128_rot_sub(acc_r, N, j + M, a), base_log, l);
    i128 d0 = 0, d1 = 0;
    for (uint32_t u = 0; u <= t; u++) {
      d0 = decomp128_next_digit(&s0, base_log);
      d1 = decomp128_next_digit(&s1, base_log);
    }
    buf[j] = ddc_make(i128_to_dd((u128)d0), i128_to_dd((u128)d1));
  }
}

// out[c][pos] (+)= buf[pos] * G[c][pos], c = 0..k; `g` points at the
// [k+1][M] key spectra of one (level, row) of a GGSW
B200_HD void p128_mac(const ddc *buf, ddc *out, const ddc *g, uint32_t M,
                      uint32_t k, bool first, uint32_t tid,
                      uint32_t nthreads) {
  for (uint32_t pos = tid; pos < M; pos += nthreads) {
    const ddc f = buf[pos];
    for (uint32_t c = 0; c <= k; c++) {
      ddc *o = out + (size_t)c * M + pos;
      const ddc gv = g[(size_t)c * M + pos];
      *o = first ? ddc_mul(f, gv) : ddc_fma(f, gv, *o);
    }
  }
}

// acc_c += round(buf) modulo 2^128 (buf: one inverse-transformed polynomial)
B200_HD void p128_acc_add(u128 *acc_c, const ddc *buf, uint32_t M,
                          uint32_t tid, uint32_t nthreads) {
  for (uint32_t j = tid; j < M; j += nthreads) {
    const ddc v = buf[j];
    acc_c[j] += dd_to_u128(v.re);
    acc_c[j + M] += dd_to_u128(v.im);
  }
}

// standard-domain u128 polynomial -> buf (signed value / M, packed)
B200_HD void p128_load_key_poly(const u128 *p, ddc *buf, uint32_t M,
                                uint32_t tid, uint32_t nthreads) {
  const double inv_m = 1.0 / (double)M; // exact: M is a power of two
  for (uint32_t j = tid; j < M; j += nthreads)
    buf[j] = ddc_make(dd_scale(i128_to_dd(p[j]), inv_m),
                      dd_scale(i128_to_dd(p[j + M]), inv_m));
}

// ---- multi-bit (pbs128_multibit.cuh) ----------------------------------------
// the 2N-th roots of unity in double-double, root[e] = exp(i pi e / N) for
// e < 2N = 4M (host): slot pos of X^d is root[d (1 + 4 bitrev(pos)) mod 2N]
static inline void b200_fill_dd_roots(uint32_t logM, ddc *root) {
  const uint64_t cnt = (uint64_t)4 << logM;
  for (uint64_t e = 0; e < cnt; e++)
    root[e] = dd_unit_root(e, cnt);
}

// monomial degree of GGSW `b` of a group of g mask words
// (modulus_switch_multi_bit): the selected u64 words are summed, then switched
// once; mask word u is selected by bit g - 1 - u of b (selection_bit)
B200_HD uint32_t p128_mb_degree(const uint64_t *mask, uint32_t g, uint32_t b,
                                uint32_t log_mod) {
  uint64_t sum = 0;
  for (uint32_t u = 0; u < g; u++)
    if ((b >> (g - 1 - u)) & 1u)
      sum += mask[u];
  return modulus_switch_u64(sum, log_mod);
}

// digit polynomial t of acc_r itself into buf (the multi-bit step decomposes
// the accumulator, not acc * X^a - acc)
B200_HD void p128_decompose_acc(const u128 *acc_r, ddc *buf, uint32_t N,
                                uint32_t base_log, uint32_t l, uint32_t t,
                                uint32_t tid, uint32_t nthreads) {
  const uint32_t M = N >> 1;
  for (uint32_t j = tid; j < M; j += nthreads) {
    u128 s0 = decomp128_init_state(acc_r[j], base_log, l);
    u128 s1 = decomp128_init_state(acc_r[j + M], base_log, l);
    i128 d0 = 0, d1 = 0;
    for (uint32_t u = 0; u <= t; u++) {
      d0 = decomp128_next_digit(&s0, base_log);
      d1 = decomp128_next_digit(&s1, base_log);
    }
    buf[j] = ddc_make(i128_to_dd((u128)d0), i128_to_dd((u128)d1));
  }
}

// out[c][pos] (+)= buf[pos] * sum_b X^{deg_b} G_b[c][pos], c = 0..k: the
// multi-bit bundle folded into the MAC slot by slot.  `g` points at the
// [k+1][M] key spectra of one (level, row) of GGSW 0 of the group; GGSW b is
// `ggsw_len` ddc further per b.  degs[b] for b = 1..nggsw-1.
B200_HD void p128_mb_mac(const ddc *buf, ddc *out, const ddc *g,
                         size_t ggsw_len, uint32_t nggsw, const uint32_t *degs,
                         const ddc *root, uint32_t logM, uint32_t k,
                         bool first, uint32_t tid, uint32_t nthreads) {
  const uint32_t M = 1u << logM, emask = (4u << logM) - 1;
  for (uint32_t pos = tid; pos < M; pos += nthreads) {
    const ddc f = buf[pos];
    const uint32_t kf = 1u + 4u * gen_bitrev(pos, logM);
    for (uint32_t c = 0; c <= k; c++) {
      const size_t off = (size_t)c * M + pos;
      ddc gv = g[off];
      for (uint32_t b = 1; b < nggsw; b++)
        gv = ddc_fma(g[b * ggsw_len + off], root[(degs[b] * kf) & emask], gv);
      ddc *o = out + off;
      *o = first ? ddc_mul(f, gv) : ddc_fma(f, gv, *o);
    }
  }
}

// acc_c = round(buf) modulo 2^128
B200_HD void p128_acc_assign(u128 *acc_c, const ddc *buf, uint32_t M,
                             uint32_t tid, uint32_t nthreads) {
  for (uint32_t j = tid; j < M; j += nthreads) {
    const ddc v = buf[j];
    acc_c[j] = dd_to_u128(v.re);
    acc_c[j + M] = dd_to_u128(v.im);
  }
}
