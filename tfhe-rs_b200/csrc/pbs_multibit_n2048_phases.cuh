// pbs_multibit_n2048_phases.cuh -- per-thread phases of the multi-bit blind
// rotation for (N = 2048, k = 1, l <= 2, grouping factor <= 4), built from the
// same register transform as the classic kernel.  Shared by the CUDA kernel
// (pbs_multibit_n2048.cuh) and the CPU CTA emulator.
//
// Reference semantics (tfhe/src/core_crypto/algorithms/
// lwe_multi_bit_programmable_bootstrapping.rs): per group of g mask elements,
//   bundle = GGSW_0 + sum_{s>=1} GGSW_s * X^{deg_s}            (:116-156)
//   acc   <- bundle (x) acc   (external product into a zeroed buffer, :806-845)
// with deg_s = mod_switch(sum of the mask elements selected by s) (:30-65).
// The bundle is never materialised here: at spectrum slot `pos` (root
// rho = tau^(1 + 4*bitrev10(pos))) it is sum_s B_s(pos) * rho^{deg_s}, folded
// into the Fourier MAC.  For the slots pos = 16*t + b of one thread,
//   rho^{deg} = tau^{deg*(1 + 4*bitrev6(t))} * zeta^{(deg * bitrev4(b)) mod 16},
//   zeta = exp(i*pi/8),
// i.e. one table look-up per (thread, s) and a 16-entry constant table.
#pragma once
#include "pbs_n2048_phases.cuh"

// signed digits of a 32-bit torus word for level_count = l (l * B <= 30),
// digit[0] = level l (least significant), as decomposer.rs:163-188 +
// iter.rs:131-151 on the word's top bits -- with ONE deliberate difference in
// the closest-representable rounding: an exact tie of the dropped bits rounds
// to EVEN instead of up.  The reference rounds half up on a 64-bit word whose
// low bits are essentially never an exact tie; here the word is the 32-bit
// ROUNDED accumulator, the tie is hit by 2^-(32-R) of all values (25 % for
// R = 30) and always-up would add a +2^-33 bias to every coefficient -- a
// DC-like error that the binary key (mean 1/2) amplifies by N/2 in the phase:
// measured 7.6x the reference's noise formula on PARAM_MULTI_BIT_GROUP_3
// (l = 2, B = 2^15), 0.21x with the even tie (tests/noise_check.py).
// `ties_even` = false restores the reference's round-half-up bit for bit
// (b200_set_multibit_tie_rule / B200_MULTIBIT_TIES=reference).
template <int MAXL>
B200_HD void digits_u32(uint32_t x, uint32_t base_log, uint32_t l,
                        int32_t d[MAXL], bool ties_even = true) {
  if (l == 1) {
    // single level: the digit is the closest representable itself, i.e. the
    // top base_log bits of the rounded word read as a signed field; 7 integer
    // instructions instead of ~25 (the rotate-free multi-bit step is otherwise
    // dominated by this).  rounding increment: half (reference, ties up) or
    // half - 1 + lsb(q) (ties to even); the balanced rule keeps +B/2 when the
    // field is exactly B/2 and the rounding did not increment it.
    const uint32_t drop1 = 32 - base_log, half1 = 1u << (drop1 - 1);
    const uint32_t add =
        ties_even ? half1 - 1u + ((x >> drop1) & 1u) : half1;
    int32_t dg = (int32_t)(x + add) >> drop1;
    const int32_t lim = (int32_t)(0x80000000u + half1 + (ties_even ? 1u : 0u));
    if ((int32_t)x < lim)
      dg = (int32_t)(1u << (base_log - 1));
    d[0] = dg;
    return;
  }
  const uint32_t R = base_log * l;
  const uint32_t drop = 32 - R; // >= 2
  const uint32_t low = x & ((1u << drop) - 1u), half = 1u << (drop - 1);
  const uint32_t q = x >> drop;
  // rounding decision `rb`: up above the half, to even on the half
  const uint32_t rb =
      (low > half) | ((low == half) & ((q & 1u) | (ties_even ? 0u : 1u)));
  uint32_t r = (q + rb) & ((1u << R) - 1u);
  const uint32_t bal = (((r - 1u) | (rb << (R - 1))) & r) >> (R - 1);
  uint32_t st = r - (bal << R);
  const uint32_t mask = (1u << base_log) - 1u;
#pragma unroll
  for (int t = 0; t < MAXL; t++) {
    if ((uint32_t)t < l) {
      const uint32_t res = st & mask;
      st = (uint32_t)((int32_t)st >> base_log);
      const uint32_t carry = (((res - 1u) | st) & res) >> (base_log - 1);
      st += carry;
      d[t] = (int32_t)(res - (carry << base_log));
    }
  }
}

// digits_u32 specialised for l = 2: the same digits word for word (checked on
// 2^27 words against digits_u32<2> by tests/test_emulator.py), about 20 integer
// instructions instead of 32.  The rounded word is kept SIGNED (arithmetic
// shift of x + increment), which is the balanced representative except for
// the value +2^(R-1) reached without a rounding increment, restored by hand.
B200_HD void digits2_u32(uint32_t x, uint32_t base_log, int32_t d[2],
                         bool ties_even = true) {
  const uint32_t drop = 32 - 2 * base_log; // >= 2
  const uint32_t half = 1u << (drop - 1);
  const uint32_t add = ties_even ? half - 1u + ((x >> drop) & 1u) : half;
  int32_t st = (int32_t)(x + add) >> drop;
  const int32_t m = (int32_t)x >> drop; // not incremented
  const int32_t lim = (int32_t)0x80000000 >> drop;
  if ((st > m ? st : m) == lim) // st == m == -2^(R-1)
    st = -lim;
  const uint32_t mask = (1u << base_log) - 1u;
  const uint32_t res0 = (uint32_t)st & mask;
  int32_t st1 = st >> base_log;
  const uint32_t c0 = (((res0 - 1u) | (uint32_t)st1) & res0) >> (base_log - 1);
  st1 += (int32_t)c0;
  d[0] = (int32_t)(res0 - (c0 << base_log));
  const uint32_t res1 = (uint32_t)st1 & mask;
  const uint32_t st2 = (uint32_t)(st1 >> base_log);
  const uint32_t c1 = (((res1 - 1u) | st2) & res1) >> (base_log - 1);
  d[1] = (int32_t)(res1 - (c1 << base_log));
}

// digits of level index `lvl` of the thread's 32 accumulator words
// (acc_lo[j1] = coefficient 64*j1 + t, acc_hi[j1] = coefficient + 1024)
B200_HD void mb_load_digits(const uint32_t acc_lo[16], const uint32_t acc_hi[16],
                            uint32_t base_log, uint32_t l, uint32_t lvl,
                            cplx v[16], bool ties_even = true) {
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    int32_t d0[2], d1[2];
    digits_u32<2>(acc_lo[j1], base_log, l, d0, ties_even);
    digits_u32<2>(acc_hi[j1], base_log, l, d1, ties_even);
    v[j1] = cmake(int_to_double(lvl ? d0[1] : d0[0]),
                  int_to_double(lvl ? d1[1] : d1[0]));
  }
}

// monomial base of GGSW s at this thread: tau^{deg * (1 + 4*bitrev6(t))}
B200_HD uint32_t mb_base_exponent(uint32_t deg, int t) {
  uint32_t r6 = 0;
#pragma unroll
  for (int i = 0; i < 6; i++)
    r6 |= (((uint32_t)t >> i) & 1u) << (5 - i);
  return (deg * (1u + 4u * r6)) & (2 * P22_N - 1);
}
B200_HD uint32_t mb_bitrev4(uint32_t b) {
  return ((b & 1u) << 3) | ((b & 2u) << 1) | ((b & 4u) >> 1) | ((b & 8u) >> 3);
}

// The whole Fourier MAC of one step for one output column (16 spectrum slots of
// this thread), software pipelined: the 2^g * l * 2 key rows of a slot are
// walked in chunks of <= 16 rows (GGSW-major), and the loads of the next chunk
// -- across slot boundaries too -- are issued before the current chunk is
// consumed, so every thread keeps 16 independent 128-bit key loads in flight.
// slot_rows(b) returns the key rows of slot b as a pointer to [lvl][r][s][64];
// out_slot(b, v) receives the result of slot b.
template <int NGGSW, int L, typename LoadBsk, typename SlotRows,
          typename OutSlot>
B200_HD void mb_mac_step(const cplx *sp, const cplx *mono_base, const cplx *zeta,
                         const uint32_t *degs, int t, LoadBsk load_bsk,
                         SlotRows slot_rows, OutSlot out_slot) {
  constexpr int ITEMS = NGGSW * L * 2; // key rows per slot
  constexpr int CH = ITEMS < 16 ? ITEMS : 16;
  constexpr int NCH = ITEMS / CH;
  constexpr int SLOTS_PER_ITER = (NCH & 1) ? 2 : 1; // keeps buffer parity static
  cplx buf[2][CH];
  // item i of a slot: s = i / (2L), lvl = (i / 2) % L, r = i % 2
  auto issue = [&](int b, int ch, cplx *dst) {
    const cplx *rows = slot_rows(b);
#pragma unroll
    for (int i = 0; i < CH; i++) {
      const int item = ch * CH + i;
      const int s = item / (2 * L), lvl = (item / 2) % L, r = item % 2;
      dst[i] = load_bsk(rows + ((size_t)(lvl * 2 + r) * NGGSW + s) * 64 + t);
    }
  };
  issue(0, 0, buf[0]);
#pragma unroll 1
  for (int b0 = 0; b0 < 16; b0 += SLOTS_PER_ITER) {
#pragma unroll
    for (int bb = 0; bb < SLOTS_PER_ITER; bb++) {
      const int b = b0 + bb;
      const uint32_t rb = mb_bitrev4((uint32_t)b);
      cplx gval[L][2];
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) {
        const int cur = (bb * NCH + ch) & 1;
        if (ch + 1 < NCH)
          issue(b, ch + 1, buf[cur ^ 1]);
        else if (b + 1 < 16)
          issue(b + 1, 0, buf[cur ^ 1]);
#pragma unroll
        for (int i = 0; i < CH; i += 2 * L) {
          const int s = (ch * CH + i) / (2 * L);
          if (s == 0) {
#pragma unroll
            for (int lvl = 0; lvl < L; lvl++)
#pragma unroll
              for (int r = 0; r < 2; r++)
                gval[lvl][r] = buf[cur][i + lvl * 2 + r];
          } else {
            const cplx mono =
                cmul(mono_base[s - 1], zeta[(degs[s] * rb) & 15u]);
#pragma unroll
            for (int lvl = 0; lvl < L; lvl++)
#pragma unroll
              for (int r = 0; r < 2; r++)
                gval[lvl][r] =
                    cfma(buf[cur][i + lvl * 2 + r], mono, gval[lvl][r]);
          }
        }
      }
      cplx out = cmake(0.0, 0.0);
#pragma unroll
      for (int lvl = 0; lvl < L; lvl++)
#pragma unroll
        for (int r = 0; r < 2; r++)
          // spectra parked as SP[lvl][r][b*64 + t]
          out = cfma(sp[((size_t)(lvl * 2 + r) * 16 + b) * 64 + t],
                     gval[lvl][r], out);
      out_slot(b, out);
    }
  }
}

// One entry of the low-latency mode's bundle (mb_bundle_kernel): at spectrum
// slot (b, t) of one (group, column), for every level and row,
//   bundle = B_0 + sum_{s >= 1} B_s * rho^{deg_s}
// summed GGSW by GGSW from s = 1, the monomial as in mb_mac_step.  key(s, lvl,
// r) gives the key value, mono_row(deg) = tau^{deg * (1 + 4*bitrev6(t))}, rb =
// bitrev4(b).
template <int NGGSW, int L, typename Key, typename MonoRow>
B200_HD void mb_bundle_entry(Key key, MonoRow mono_row, const cplx *zeta,
                             const uint32_t *degs, uint32_t rb,
                             cplx acc[L][2]) {
#pragma unroll
  for (int lvl = 0; lvl < L; lvl++)
#pragma unroll
    for (int r = 0; r < 2; r++)
      acc[lvl][r] = key(0u, lvl, r);
#pragma unroll
  for (uint32_t sigma = 1; sigma < (uint32_t)NGGSW; sigma++) {
    const uint32_t deg = degs[sigma];
    const cplx mono = cmul(mono_row(deg), zeta[(deg * rb) & 15u]);
#pragma unroll
    for (int lvl = 0; lvl < L; lvl++)
#pragma unroll
      for (int r = 0; r < 2; r++)
        acc[lvl][r] = cfma(key(sigma, lvl, r), mono, acc[lvl][r]);
  }
}

B200_HD void mb_acc_assign(uint32_t acc_lo[16], uint32_t acc_hi[16],
                           const cplx v[16]) {
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    acc_lo[j1] = scaled_double_to_torus32(v[j1].re);
    acc_hi[j1] = scaled_double_to_torus32(v[j1].im);
  }
}
