// pbs_n2048_phases.cuh -- per-thread phases of the (N=2048, k=1, l=1) blind
// rotation, shared by the sm_90a kernel (pbs_n2048.cuh) and the CPU CTA
// emulator (tests/emu).  One CTA = one LWE; 128 threads = 2 groups of 64;
// group g owns GLWE polynomial g (0 = mask, 1 = body): it decomposes and
// forward-transforms ct1[g], then accumulates output column g.
//
// Reference semantics restated here (tfhe/src/core_crypto/...):
//   fft_impl/fft64/crypto/bootstrap.rs:318-365   blind_rotate_assign loop
//   algorithms/polynomial_algorithms.rs:544-583  X^-b rotation of the LUT
//   algorithms/polynomial_algorithms.rs:662-730  ct1 = ct0*X^a - ct0
//   commons/math/decomposition/decomposer.rs:163-188  closest representable
//   fft_impl/fft64/crypto/ggsw.rs:483-602        external product
//   algorithms/glwe_sample_extraction.rs:119-165 sample extract
#pragma once
#include "negacyclic_fft.cuh"

#include <type_traits>
#include <utility>

#define P22_N 2048
#define P22_M 1024
#define P22_GROUP 64

// Signed level-1 digit of x for a single-level decomposition of base 2^B:
// the closest representable value, balanced on ties (decomposer.rs:163-188
// followed by iter.rs:131-151 with level_count = 1, which returns the state
// itself as a value in [-B/2, B/2]).
B200_HD int32_t digit_l1(uint64_t x, uint32_t base_log) {
  uint32_t r = (uint32_t)(x >> (64 - base_log - 1));
  const uint32_t rb = r & 1u;
  r = (r + 1u) >> 1;
  r &= (1u << base_log) - 1u;
  const uint32_t bal = (((r - 1u) | (rb << (base_log - 1))) & r) >> (base_log - 1);
  return (int32_t)(r - (bal << base_log));
}

// (p * X^a)[j] - p[j] for one polynomial held in shared memory, a in [1, 2N)
B200_HD uint64_t rot_sub_coeff(const uint64_t *p, uint32_t j, uint32_t a) {
  const uint32_t d = a & (P22_N - 1);
  const bool neg0 = a >= P22_N;
  const bool wrap = j < d;
  const uint32_t jj = wrap ? j + P22_N - d : j - d;
  const uint64_t x = p[jj];
  const bool neg = neg0 != wrap;
  return (neg ? (uint64_t)0 - x : x) - p[j];
}

// phase 1: digits of ct1[g] into pass-1 registers (thread t holds complex
// coefficients j = 64*j1 + t, j1 = 0..15: re <- coef j, im <- coef j + 1024)
B200_HD void p22_load_digits(const uint64_t *acc_g, int t, uint32_t a,
                             uint32_t base_log, cplx v[16]) {
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    const uint32_t j = 64u * j1 + (uint32_t)t;
    const int32_t d0 = digit_l1(rot_sub_coeff(acc_g, j, a), base_log);
    const int32_t d1 = digit_l1(rot_sub_coeff(acc_g, j + P22_M, a), base_log);
    v[j1] = cmake(int_to_double(d0), int_to_double(d1));
  }
}

// Fourier-domain MAC for output column g (k = 1, l = 1):
//   out = F[0] * B[0][g] + F[1] * B[1][g]
// `own` = this group's spectrum (registers, pass-3 layout), `other` = the
// other group's spectrum in the shared spectrum layout (b*64 + t).
// bsk_ig points at the 2 x 1024 complex block of (GGSW i, column g):
// [r][b][t].  Result overwrites `own`.
template <typename LoadBsk>
B200_HD void p22_mac(cplx own[16], const cplx *other, const cplx *bsk_ig,
                     int t, int g, LoadBsk load_bsk) {
#pragma unroll
  for (int b = 0; b < 16; b++) {
    const cplx f_other = other[b * 64 + t];
    const cplx f0 = g == 0 ? own[b] : f_other;
    const cplx f1 = g == 0 ? f_other : own[b];
    const cplx b0 = load_bsk(bsk_ig + (0 * 16 + b) * 64 + t);
    const cplx b1 = load_bsk(bsk_ig + (1 * 16 + b) * 64 + t);
    own[b] = cfma(f1, b1, cmul(f0, b0));
  }
}

// final phase: add the inverse transform back on the torus.  The 1/M scale
// of the inverse is folded into the Fourier BSK at conversion time.
B200_HD void p22_acc_update(uint64_t *acc_g, int t, const cplx v[16]) {
  // the register-FFT key layout carries an extra 2^32 (see
  // scaled_double_to_torus32); the 64-bit accumulator path undoes it
  const double unscale = 2.3283064365386963e-10; // 2^-32
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    const uint32_t j = 64u * j1 + (uint32_t)t;
    acc_g[j] += double_to_torus64(v[j1].re * unscale);
    acc_g[j + P22_M] += double_to_torus64(v[j1].im * unscale);
  }
}

// ===========================================================================
// The integer stages either side of every blind rotation, shared by all PBS
// kernels and their CPU replays: the modulus switch of the input LWE (standard
// or centered mean), acc = LUT * X^{-b_hat}, and the many-LUT sample extract.
// ===========================================================================

// LUT * X^{-b_hat} coefficient j (polynomial_wrapping_monic_monomial_div)
template <typename Word>
B200_HD Word rot_div_coeff(const Word *lut, uint32_t N, uint32_t j,
                           uint32_t b_hat) {
  const uint32_t d = b_hat & (N - 1);
  const bool neg0 = b_hat >= N;
  const uint32_t s = j + d;
  const bool wrap = s >= N;
  const Word x = lut[wrap ? s - N : s];
  return (neg0 != wrap) ? (Word)0 - x : x;
}

// modulus switch to 2^log_modulus, rounded (fft_impl/common.rs:10-23)
B200_HD uint64_t modulus_switch_full(uint64_t x, uint32_t log_modulus) {
  return (x + ((uint64_t)1 << (63 - log_modulus))) >> (64 - log_modulus);
}

// the same, to 2N <= 2^32
B200_HD uint32_t modulus_switch_u64(uint64_t x, uint32_t log_modulus) {
  return (uint32_t)modulus_switch_full(x, log_modulus);
}

// per-element terms of the centered-mean body correction
// (algorithms/modulus_switch.rs:55-100): returns half error, accumulates the
// doubled halving error.
B200_HD int64_t centered_ms_half_error(uint64_t a, uint32_t log_modulus,
                                       int64_t *halving_error_doubled) {
  const uint64_t rounded = (uint64_t)modulus_switch_u64(a, log_modulus)
                           << (64 - log_modulus);
  const int64_t err = (int64_t)(rounded - a);
  const int64_t half = err / 2;
  *halving_error_doubled = 2 * half - err;
  return half;
}

// sample-extract of coefficient nth: mask word t of polynomial A
// Poly: anything indexable by coefficient (a pointer, or the bit-packed reader
// of the decompression, compression.cuh); the word type is the one it reads
// (u64, or u128 for the squashed-noise unpacking, keyswitch128.cuh)
template <typename Poly, typename Word = std::decay_t<decltype(std::declval<const Poly &>()[0])>>
B200_HD Word sample_extract_mask_coeff(const Poly &A, uint32_t N, uint32_t nth,
                                       uint32_t t) {
  return t <= nth ? A[nth - t] : (Word)0 - A[N + nth - t];
}

// A thread's share of the two sums of the centered-mean correction, over the
// mask words it switches.  Integer sums: every grouping gives the same words.
struct CenteredMsSums {
  unsigned long long half = 0;
  long long dbl = 0;
  B200_HD void add(uint64_t a, uint32_t log_modulus) {
    int64_t d;
    half += (unsigned long long)centered_ms_half_error(a, log_modulus, &d);
    dbl += d;
  }
};

// The body plus the centered-mean correction.  The sums of the whole mask
// arrive as `nslots` partial sums (one per warp, or a single shared total):
// ds / 2 truncates toward zero, so it is taken once, on the total.
B200_HD uint64_t centered_ms_body(uint64_t body, const unsigned long long *half,
                                  const long long *dbl, int nslots,
                                  uint32_t log_modulus) {
  uint64_t hs = 0;
  int64_t ds = 0;
  for (int w = 0; w < nslots; w++) {
    hs += half[w];
    ds += dbl[w];
  }
  return body + (hs - (uint64_t)(ds / 2)) - ((uint64_t)1 << (63 - log_modulus));
}

// b_hat: the body switched to 2N, with or without the centered correction
B200_HD uint32_t ms_b_hat(uint64_t body, bool centered,
                          const unsigned long long *half, const long long *dbl,
                          int nslots, uint32_t log_modulus) {
  if (centered)
    body = centered_ms_body(body, half, dbl, nslots, log_modulus);
  return modulus_switch_u64(body, log_modulus);
}

#if defined(__CUDACC__)
// Publish step of the warp form of the sum reduction (thread counts that are
// multiples of 32): each warp's total goes to slot threadIdx.x / 32.  After
// the caller's barrier one thread reads the slots (nslots = warps).
__device__ __forceinline__ void centered_ms_publish_warp(CenteredMsSums s,
                                                         unsigned long long *half,
                                                         long long *dbl) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    s.half += __shfl_xor_sync(0xffffffffu, s.half, off);
    s.dbl += __shfl_xor_sync(0xffffffffu, s.dbl, off);
  }
  if ((threadIdx.x & 31) == 0) {
    half[threadIdx.x >> 5] = s.half;
    dbl[threadIdx.x >> 5] = s.dbl;
  }
}

// Publish step of the shared-memory form (groups that are not warp multiples,
// or several LWEs per CTA): atomic adds into one slot, zeroed before an
// earlier barrier.  After the caller's barrier nslots = 1.
__device__ __forceinline__ void centered_ms_publish_atomic(const CenteredMsSums &s,
                                                           unsigned long long *half,
                                                           long long *dbl) {
  atomicAdd(half, s.half);
  atomicAdd(reinterpret_cast<unsigned long long *>(dbl), (unsigned long long)s.dbl);
}
#endif

// acc = LUT * X^{-b_hat} for `rows` polynomials of N coefficients: flat
// coefficient j = r N + c for j = first, first + step, ...; acc rows are
// acc_stride words apart; cvt maps the LUT word to the accumulator word.
template <typename Acc, typename Word, typename Cvt>
B200_HD void rotate_lut(Acc *acc, uint32_t acc_stride, const Word *lut,
                        uint32_t rows, uint32_t N, uint32_t b_hat,
                        uint32_t first, uint32_t step, Cvt cvt) {
  for (uint32_t j = first; j < rows * N; j += step) {
    const uint32_t r = j / N, c = j % N;
    (acc + (size_t)r * acc_stride)[c] = cvt(rot_div_coeff(lut + (size_t)r * N, N, c, b_hat));
  }
}

// The LWE extracted at coefficient nth of the GLWE in acc (k mask rows, then
// the body row, acc_stride words apart): mask word w = r N + t for
// w = first, first + step, ..., and the body, word k N, by the thread with
// first = 0; cvt maps the accumulator word to the output word.
template <typename Out, typename Acc, typename Cvt>
B200_HD void sample_extract_lwe(Out *out, const Acc *acc, uint32_t acc_stride,
                                uint32_t k, uint32_t N, uint32_t nth,
                                uint32_t first, uint32_t step, Cvt cvt) {
  for (uint32_t w = first; w < k * N; w += step) {
    // r = 0 spelled out for k = 1: the compiler does not derive it from
    // w < N, and the row split changed the register allocation of the
    // multi-bit N = 2048 kernels
    const uint32_t r = k > 1 ? w / N : 0, t = w - r * N;
    out[w] = cvt(sample_extract_mask_coeff(acc + (size_t)r * acc_stride, N, nth, t));
  }
  if (first == 0)
    out[(size_t)k * N] = cvt(acc[(size_t)k * acc_stride + nth]);
}

// Many-LUT output layout: LUT m of the sample goes to coefficient
// nth = m * lut_stride and to LWE m * batch + out_idx of lwe_out.
template <typename Out, typename Acc, typename Cvt>
B200_HD void sample_extract_many_lut(Out *lwe_out, uint64_t out_idx, uint64_t batch,
                                     uint32_t num_many_lut, uint32_t lut_stride,
                                     const Acc *acc, uint32_t acc_stride,
                                     uint32_t k, uint32_t N, uint32_t first,
                                     uint32_t step, Cvt cvt) {
  const uint64_t out_len = (uint64_t)k * N + 1;
  for (uint32_t m = 0; m < num_many_lut; m++)
    sample_extract_lwe(lwe_out + ((uint64_t)m * batch + out_idx) * out_len, acc,
                       acc_stride, k, N, m * lut_stride, first, step, cvt);
}

// word conversions of the two helpers above
struct SameWord {
  template <typename T> B200_HD T operator()(T x) const { return x; }
};
// the 32-bit accumulators keep bits 63..32 of the torus word
struct Torus32To64 {
  B200_HD uint64_t operator()(uint32_t x) const { return (uint64_t)x << 32; }
};

// ===========================================================================
// v2 phases: 32-bit running accumulator.
//
// Only the top l*base_log + 1 (= 24) bits of an accumulator word are ever read
// back (by the decomposition), and the f64 transform itself only carries ~32
// meaningful bits per step, so the blind rotation keeps the top 32 bits of
// every coefficient (the reference GPU kernel does the same,
// programmable_bootstrap_classic.cuh:373-378,657-660); the LWE written at the
// end is that word shifted back to bits 63..32.  Halves the accumulator's
// shared-memory footprint and traffic and turns the u64 integer work of the
// rotate/decompose step into u32 work.
// ===========================================================================

// round(xs) mod 2^32 for xs = x * 2^32 (the factor 2^32 is folded into the
// Fourier key at conversion time), in THREE fp64 adds and no conversion:
//   t = xs + 1.5*2^84          rounds xs to a multiple of 2^32 (ulp there)
//   u = (1.5*2^52 + 1.5*2^84) - t = 1.5*2^52 - high(xs)          (exact)
//   y = xs + u = 1.5*2^52 + low(xs), rounded to an integer by the add
// and the low mantissa word of y is the answer (two's complement).
// Valid for |xs| < 2^83; the products of a CMUX stay below 2^68.
B200_HD uint32_t scaled_double_to_torus32(double xs) {
  const double m52 = 6755399441055744.0;              // 1.5 * 2^52
  const double m84 = 29014219670751100192948224.0;    // 1.5 * 2^84
  const double t = xs + m84;
  const double u = (m52 + m84) - t;
  const double y = xs + u;
#if defined(__CUDA_ARCH__)
  return (uint32_t)__double2loint(y);
#else
  uint64_t bits;
  __builtin_memcpy(&bits, &y, 8);
  return (uint32_t)bits;
#endif
}

B200_HD void p22v2_acc_update(uint32_t *acc_g, int t, const cplx v[16]) {
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    const uint32_t j = 64u * j1 + (uint32_t)t;
    acc_g[j] += scaled_double_to_torus32(v[j1].re);
    acc_g[j + P22_M] += scaled_double_to_torus32(v[j1].im);
  }
}

// top 32 bits of a 64-bit torus word, rounded to nearest
B200_HD uint32_t torus64_to_32(uint64_t x) {
  return (uint32_t)((x + 0x80000000ull) >> 32);
}
struct Torus64To32 {
  B200_HD uint32_t operator()(uint64_t x) const { return torus64_to_32(x); }
};

// MAC with explicit software prefetch: the 16 "own-row" key values are loaded
// by the caller before the last forward pass (their L2 latency hides behind the
// pass and the share barrier); the 16 "other-row" values are requested in one
// batch as soon as the own-row products have freed their registers.
// `bsk_oth` points at row (1 - g) of the (GGSW i, column g) block.  The group
// is a run-time value on purpose: one copy of the loop body for both groups
// (two template instances doubled the I-cache footprint: 24 % no_instruction
// stalls in the first v3 capture).
template <typename LoadBsk>
B200_HD void p22v3_mac(cplx own[16], const cplx b_own[16], const cplx *other,
                       const cplx *bsk_oth, int t, LoadBsk load_bsk) {
  cplx b_oth[16];
#pragma unroll
  for (int b = 0; b < 16; b++)
    own[b] = cmul(own[b], b_own[b]);
#pragma unroll
  for (int b = 0; b < 16; b++)
    b_oth[b] = load_bsk(bsk_oth + b * 64 + t);
#pragma unroll
  for (int b = 0; b < 16; b++)
    own[b] = cfma(other[b * 64 + t], b_oth[b], own[b]);
}

// Lean rotate + decompose for the 32-bit accumulator (v3).
//  * (acc * X^a)[j] = s * acc[(j - a) mod 2N]: the index is one add + one mask
//    on a per-thread base, the sign a 3-input XOR of two masks;
//  * the single-level signed digit is an arithmetic shift of the rounded word,
//    ((int32)(x + half)) >> (32 - B) in [-B/2, B/2), plus the reference's
//    balanced tie rule (decomposer.rs:61-68,163-188): the field value B/2 stays
//    +B/2 when the rounding bit is 0, i.e. when x is in [2^31, 2^31 + half).
B200_HD void p22v3_load_digits(const uint32_t *acc_g, int t, uint32_t a,
                               uint32_t base_log, cplx v[16]) {
  const uint32_t d = a & (P22_N - 1);
  const uint32_t neg0 = 0u - (a >> 11);            // all ones if a >= N
  const uint32_t half = 1u << (31 - base_log);
  const uint32_t sh = 32 - base_log;
  const uint32_t base = (uint32_t)t - d;           // (j - d) before masking
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    const uint32_t j = 64u * j1 + (uint32_t)t;
    const uint32_t u0 = base + 64u * j1;           // j - d      (mod 2^32)
    const uint32_t u1 = u0 + P22_M;                // j + M - d
    // j < d  <=>  (j - d) negative as 32-bit (|j - d| < 2^31)
    const uint32_t m0 = (uint32_t)((int32_t)u0 >> 31) ^ neg0;
    const uint32_t m1 = (uint32_t)((int32_t)u1 >> 31) ^ neg0;
    const uint32_t x0 = (acc_g[u0 & (P22_N - 1)] ^ m0) - m0 - acc_g[j];
    const uint32_t x1 = (acc_g[u1 & (P22_N - 1)] ^ m1) - m1 - acc_g[j + P22_M];
    int32_t d0 = (int32_t)(x0 + half) >> sh;
    int32_t d1 = (int32_t)(x1 + half) >> sh;
    if ((x0 ^ 0x80000000u) < half)
      d0 = (int32_t)(1u << (base_log - 1));
    if ((x1 ^ 0x80000000u) < half)
      d1 = (int32_t)(1u << (base_log - 1));
    v[j1] = cmake(int_to_double(d0), int_to_double(d1));
  }
}

// ===========================================================================
// v4 phases (round 2): same results as p22v3_load_digits / p22v2_acc_update,
// fewer integer instructions and 32 fewer shared-memory loads per thread and
// step.  A per-phase clock profile of the round-1 kernel put rotate + decompose at 10-16 % of a
// CMUX step for ~450 integer instructions and 64 LDS per thread.
//  * the thread's OWN 32 accumulator words are handed over in registers from
//    the accumulator update of the previous step (`own`: live only across the
//    barrier between two steps, while the 64 transform registers are dead);
//  * rotated source index in BYTE units: one add + one mask for coefficient j,
//    one XOR for coefficient j + N/2;
//  * tie rule as one signed compare against a uniform constant.
// ===========================================================================
template <int CVT = 0>
B200_HD void p22v4_load_digits(const uint32_t *acc_g, int t, uint32_t a,
                               uint32_t base_log, const uint32_t own[32],
                               cplx v[16]) {
  const uint32_t d = a & (P22_N - 1);
  const uint32_t neg0 = 0u - (a >> 11);            // all ones if a >= N
  const uint32_t half = 1u << (31 - base_log);
  const uint32_t sh = 32 - base_log;
  const int32_t tie_below = (int32_t)(0x80000000u + half);
  const int32_t plus_half_base = (int32_t)(1u << (base_log - 1));
  const uint32_t base4 = ((uint32_t)t - d) * 4u;   // 4 * (j - d) for j1 = 0
  const unsigned char *accb = reinterpret_cast<const unsigned char *>(acc_g);
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    const uint32_t ub0 = base4 + 256u * j1;        // 4 * (j - d)
    const uint32_t ub1 = ub0 + 4u * P22_M;         // 4 * (j + M - d)
    const uint32_t ib0 = ub0 & (4u * P22_N - 4u);  // byte offset of (j - d) mod N
    const uint32_t r0 = *reinterpret_cast<const uint32_t *>(accb + ib0);
    const uint32_t r1 =
        *reinterpret_cast<const uint32_t *>(accb + (ib0 ^ (4u * P22_M)));
    uint32_t x0, x1;
    if ((CVT & 2) == 0) {
      const uint32_t m0 = (uint32_t)((int32_t)ub0 >> 31) ^ neg0;
      const uint32_t m1 = (uint32_t)((int32_t)ub1 >> 31) ^ neg0;
      x0 = (r0 ^ m0) - m0 - own[j1];
      x1 = (r1 ^ m1) - m1 - own[16 + j1];
    } else {
      // sign as a predicate: one compare + one predicated negate-and-subtract
      const bool n0 = ((int32_t)ub0 < 0) != (neg0 != 0u);
      const bool n1 = ((int32_t)ub1 < 0) != (neg0 != 0u);
      x0 = n0 ? (0u - r0) - own[j1] : r0 - own[j1];
      x1 = n1 ? (0u - r1) - own[16 + j1] : r1 - own[16 + j1];
    }
    int32_t d0 = (int32_t)(x0 + half) >> sh;
    int32_t d1 = (int32_t)(x1 + half) >> sh;
    // balanced tie (decomposer.rs:163-188): x in [2^31, 2^31 + half) -> +B/2
    if ((int32_t)x0 < tie_below)
      d0 = plus_half_base;
    if ((int32_t)x1 < tie_below)
      d1 = plus_half_base;
    if ((CVT & 1) == 0)
      v[j1] = cmake(int_to_double(d0), int_to_double(d1));
    else
      v[j1] = cmake(int_to_double_splice(d0), int_to_double_splice(d1));
  }
}

B200_HD void p22v4_acc_update(uint32_t *acc_g, int t, const cplx v[16],
                              uint32_t own[32]) {
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    const uint32_t j = 64u * j1 + (uint32_t)t;
    // The accumulator word is READ BACK from shared memory although own[] holds
    // it: that ends own[]'s live range at the rotate + decompose phase and gives
    // the transforms and the MAC 32 more registers.  `own[j1] += ...` (no read)
    // was 5 % slower on the 253-register N = 2048 kernel where it was first tuned
    // (it is what the N = 512 kernel does, where the registers are there).
    own[j1] = acc_g[j] + scaled_double_to_torus32(v[j1].re);
    own[16 + j1] = acc_g[j + P22_M] + scaled_double_to_torus32(v[j1].im);
    acc_g[j] = own[j1];
    acc_g[j + P22_M] = own[16 + j1];
  }
}

B200_HD void p22v4_own_init(const uint32_t *acc_g, int t, uint32_t own[32]) {
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    own[j1] = acc_g[64 * j1 + t];
    own[16 + j1] = acc_g[64 * j1 + t + P22_M];
  }
}
