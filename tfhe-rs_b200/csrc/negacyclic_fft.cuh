// negacyclic_fft.cuh -- twist-free negacyclic transform used by every kernel.
//
// What it computes (same map as tfhe-rs `FftView::forward_as_integer` /
// `add_backward_in_place_as_torus`, tfhe/src/core_crypto/fft_impl/fft64/math/
// fft/mod.rs:380-496, up to the private ordering of the spectrum):
//   a real polynomial p of size N is folded to M = N/2 complex coefficients
//   z_j = p_j + i p_{j+M}; the transform evaluates Z(x) = sum_j z_j x^j at the
//   M roots of x^M = i, i.e. at x = t^(4k+1), t = exp(i pi / N).  Pointwise
//   products of such spectra are negacyclic products mod X^N + 1.
//
// How (not the reference's twist + cyclic FFT): the roots of
// x^n = e^{i phi} split into those of x^{n/2} = +-e^{i phi/2}, so
//   Z mod (x^n - c)  ->  (Z_lo + s Z_hi, Z_lo - s Z_hi),  s = sqrt(c),
// recursively.  There is no separate twist pass and no untwist: the first
// four levels use twiddles that are the same for every thread (compile-time
// constants in the constant bank), the remaining ones are loop-invariant per
// thread and live in registers for the whole blind rotation.
//
// Level L (1-based) splits sub-block u (L-1 path bits, first split = MSB) with
//   tw(L,u) = t^{(1 + 4*bitrev_{L-1}(u)) * 2^(logM - L)},   t = exp(i pi/(2M)).
// Output slot `pos` (in-place order) holds the value at x = t^(1+4*bitrev(pos)).
// Two levels are fused into one radix-4 step (24 operations per 4 points
// forward, 28 inverse -- 26.5 inside a radix-16 pass, see radix16_inv).
#pragma once
#include "hd.cuh"

// ---------------------------------------------------------------------------
// radix-4 steps.  Elements (a,b,c,d) sit at x, x+h, x+2h, x+3h; level L pairs
// distance 2h with s1 = tw(L,u); level L+1 pairs distance h with
// s2 = tw(L+1, 2u) on the "+" half and i*s2 on the "-" half; s3 = s1*s2.
// ---------------------------------------------------------------------------
B200_HD void radix4_fwd(cplx &a, cplx &b, cplx &c, cplx &d, const cplx s1,
                        const cplx s2, const cplx s3) {
  const cplx t0 = cfma(s1, c, a);                 // a + s1 c
  const cplx t1 = cmake(two_a_minus(a.re, t0.re), two_a_minus(a.im, t0.im)); // a - s1 c
  const cplx bb = cmul(s2, b);
  const cplx t2 = cfma(s3, d, bb);                // s2 b + s3 d
  const cplx t3 = cmake(two_a_minus(bb.re, t2.re), two_a_minus(bb.im, t2.im)); // s2 b - s3 d
  a = cadd(t0, t2);
  b = csub(t0, t2);
  c = cmake(t1.re - t3.im, t1.im + t3.re);        // t1 + i t3
  d = cmake(t1.re + t3.im, t1.im - t3.re);        // t1 - i t3
}

// exact inverse of radix4_fwd up to a factor 4
B200_HD void radix4_inv(cplx &a, cplx &b, cplx &c, cplx &d, const cplx s1,
                        const cplx s2, const cplx s3) {
  const cplx t0 = cadd(a, b);
  const cplx t2 = csub(a, b);
  const cplx t1 = cadd(c, d);
  const cplx e = csub(c, d);
  const cplx t3 = cmake(e.im, -e.re);             // -i (c - d)
  a = cadd(t0, t1);
  c = cmulc(csub(t0, t1), s1);
  b = cmulc(cadd(t2, t3), s2);
  d = cmulc(csub(t2, t3), s3);
}

// ---------------------------------------------------------------------------
// Twiddle bookkeeping for M = 1024 (N = 2048) split as 16 x 4 x 16.
// ---------------------------------------------------------------------------
// pass 1 (levels 1-4): 15 constants, identical for all threads:
//   [0..2]   layer A: s1=tw(1,0) s2=tw(2,0) s3
//   [3+3u..] layer B, u=0..3: s1=tw(3,u) s2=tw(4,2u) s3
// pass 2 (levels 5-6): per q = 0..15: s1=tw(5,q) s2=tw(6,2q) s3      -> [16][3]
// pass 3 (levels 7-10): per u6 = 0..63:
//   [0..2]   layer A: s1=tw(7,u6) s2=tw(8,2u6) s3
//   [3+3u..] layer B, u=0..3: s1=tw(9,4u6+u) s2=tw(10,2(4u6+u)) s3  -> [64][15]
struct Fft1024Tables {
  cplx pass1[15];
  cplx pass2[16][3];
  cplx pass3[64][15];
};

// host-side table generation (extended precision)
#include <cmath>
static inline uint32_t b200_bitrev(uint32_t x, uint32_t bits) {
  uint32_t r = 0;
  for (uint32_t i = 0; i < bits; i++)
    if (x & (1u << i))
      r |= 1u << (bits - 1 - i);
  return r;
}
// tw(L,u) for transform size M = 2^logM
static inline cplx b200_tw(uint32_t logM, uint32_t L, uint32_t u) {
  const long double pi = 3.14159265358979323846264338327950288L;
  const uint64_t e =
      (uint64_t)(1 + 4 * b200_bitrev(u, L - 1)) << (logM - L); // units pi/(2M)
  const uint64_t period = (uint64_t)4 << logM;                 // 4M = 2N
  const long double ang =
      pi * (long double)(e % period) / (long double)((uint64_t)2 << logM);
  cplx r;
  r.re = (double)cosl(ang);
  r.im = (double)sinl(ang);
  return r;
}
static inline cplx b200_cmul_ld(cplx a, cplx b) {
  // s3 = s1*s2 evaluated in extended precision then rounded once
  const long double re =
      (long double)a.re * b.re - (long double)a.im * b.im;
  const long double im =
      (long double)a.re * b.im + (long double)a.im * b.re;
  cplx r;
  r.re = (double)re;
  r.im = (double)im;
  return r;
}
static inline void b200_triple(cplx *dst, uint32_t logM, uint32_t L,
                               uint32_t u) {
  // exact angles: s3 = tw(L,u)*tw(L+1,2u) computed from the summed exponent
  const long double pi = 3.14159265358979323846264338327950288L;
  dst[0] = b200_tw(logM, L, u);
  dst[1] = b200_tw(logM, L + 1, 2 * u);
  const uint64_t e1 = (uint64_t)(1 + 4 * b200_bitrev(u, L - 1)) << (logM - L);
  const uint64_t e2 = (uint64_t)(1 + 4 * b200_bitrev(2 * u, L))
                      << (logM - L - 1);
  const uint64_t period = (uint64_t)4 << logM;
  const long double ang = pi * (long double)((e1 + e2) % period) /
                          (long double)((uint64_t)2 << logM);
  dst[2].re = (double)cosl(ang);
  dst[2].im = (double)sinl(ang);
}
static inline void b200_fill_fft1024_tables(Fft1024Tables *t) {
  const uint32_t lm = 10;
  b200_triple(&t->pass1[0], lm, 1, 0);
  for (uint32_t u = 0; u < 4; u++)
    b200_triple(&t->pass1[3 + 3 * u], lm, 3, u);
  for (uint32_t q = 0; q < 16; q++)
    b200_triple(&t->pass2[q][0], lm, 5, q);
  for (uint32_t u6 = 0; u6 < 64; u6++) {
    b200_triple(&t->pass3[u6][0], lm, 7, u6);
    for (uint32_t u = 0; u < 4; u++)
      b200_triple(&t->pass3[u6][3 + 3 * u], lm, 9, 4 * u6 + u);
  }
}

// ---------------------------------------------------------------------------
// In-register radix-16 passes on v[16].  `tw` points at 15 twiddles laid out
// as documented above (layer A triple, then four layer-B triples).
// ---------------------------------------------------------------------------
B200_HD void radix16_fwd(cplx v[16], const cplx *tw) {
#pragma unroll
  for (int m = 0; m < 4; m++)
    radix4_fwd(v[m], v[m + 4], v[m + 8], v[m + 12], tw[0], tw[1], tw[2]);
#pragma unroll
  for (int u = 0; u < 4; u++)
    radix4_fwd(v[4 * u], v[4 * u + 1], v[4 * u + 2], v[4 * u + 3],
               tw[3 + 3 * u], tw[4 + 3 * u], tw[5 + 3 * u]);
}

// radix4_inv without its three output multiplications: b, c, d are left to be
// multiplied by conj(s2), conj(s1), conj(s3) by whoever consumes them
B200_HD void radix4_inv_pending(cplx &a, cplx &b, cplx &c, cplx &d) {
  const cplx t0 = cadd(a, b);
  const cplx t2 = csub(a, b);
  const cplx t1 = cadd(c, d);
  const cplx e = csub(c, d);
  const cplx t3 = cmake(e.im, -e.re);
  a = cadd(t0, t1);
  c = csub(t0, t1);
  b = cadd(t2, t3);
  d = csub(t2, t3);
}
// radix4_inv on inputs that still carry pending factors conj(p0..p3): the
// products fuse with the first additions (x0 p0* + x1 p1* is a multiply and a
// fused multiply-add, the difference one more FMA: 10 operations per pair
// instead of 8 for the two products + 4 for sum and difference)
B200_HD void radix4_inv_fused(cplx &a, cplx &b, cplx &c, cplx &d, const cplx p0,
                              const cplx p1, const cplx p2, const cplx p3,
                              const cplx s1, const cplx s2, const cplx s3) {
  const cplx A = cmulc(a, p0);
  const cplx t0 = cfmac(b, p1, A);
  const cplx t2 = cmake(two_a_minus(A.re, t0.re), two_a_minus(A.im, t0.im));
  const cplx C = cmulc(c, p2);
  const cplx t1 = cfmac(d, p3, C);
  const cplx e = cmake(two_a_minus(C.re, t1.re), two_a_minus(C.im, t1.im));
  const cplx t3 = cmake(e.im, -e.re);
  a = cadd(t0, t1);
  c = cmulc(csub(t0, t1), s1);
  b = cmulc(cadd(t2, t3), s2);
  d = cmulc(csub(t2, t3), s3);
}

// Layer B (four radix-4 steps with their own twiddle triples) leaves its output
// multiplications pending; layer A's steps 1..3 take element m of every layer-B
// step, i.e. four values with pending conj(s2) / conj(s1) / conj(s3) of the four
// triples, and fuse them into their first additions: 212 operations instead of
// 224 (the forward pass needs 192).
B200_HD void radix16_inv(cplx v[16], const cplx *tw) {
#pragma unroll
  for (int u = 0; u < 4; u++)
    radix4_inv_pending(v[4 * u], v[4 * u + 1], v[4 * u + 2], v[4 * u + 3]);
  radix4_inv(v[0], v[4], v[8], v[12], tw[0], tw[1], tw[2]);
  // element 1 = "b" (pending conj s2 = tw[4 + 3u]), 2 = "c" (s1 = tw[3 + 3u]),
  // 3 = "d" (s3 = tw[5 + 3u])
  radix4_inv_fused(v[1], v[5], v[9], v[13], tw[4], tw[7], tw[10], tw[13], tw[0],
                   tw[1], tw[2]);
  radix4_inv_fused(v[2], v[6], v[10], v[14], tw[3], tw[6], tw[9], tw[12], tw[0],
                   tw[1], tw[2]);
  radix4_inv_fused(v[3], v[7], v[11], v[15], tw[5], tw[8], tw[11], tw[14], tw[0],
                   tw[1], tw[2]);
}

// pass 2: registers r = 4*bl + a, all four radix-4 steps of a thread belong to
// the same sub-problem q = t >> 2 and share one twiddle triple tw2[0..2]
B200_HD void pass2_fwd(cplx v[16], const cplx *tw2) {
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
    radix4_fwd(v[4 * bl], v[4 * bl + 1], v[4 * bl + 2], v[4 * bl + 3], tw2[0],
               tw2[1], tw2[2]);
}
B200_HD void pass2_inv(cplx v[16], const cplx *tw2) {
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
    radix4_inv(v[4 * bl], v[4 * bl + 1], v[4 * bl + 2], v[4 * bl + 3], tw2[0],
               tw2[1], tw2[2]);
}

// ---------------------------------------------------------------------------
// Shared-memory exchanges between the passes (one 1024-complex buffer per
// polynomial, 64 threads per polynomial; `t` is the thread index inside that
// 64-thread group).
//
// pass-1 layout: thread t = j0 holds v[q], q = j1 path position (0..15)
// pass-2 layout: thread t = 4*q + bh holds v[4*bl + a], j0 = 16*a + 4*bh + bl
//                (one q per thread -> a single twiddle triple per thread)
// pass-3 layout: thread t = u6 = 4*q + a' holds v[b], slot pos = 16*t + b
//
// X1 slot of element (q, j0):  q*64 + (j0 ^ (((j0 >> 3) & 1) << 1) ^ (q & 1))
// X2 slot of element (row = 4q + a', b):
//     row*16 + (b ^ ((b >> 3) << 1) ^ (((row & 3) << 1) | ((row >> 2) & 1)))
// Both XOR swizzles make every quarter-warp of every 128-bit access (stores
// and loads, forward and inverse direction) hit 8 distinct 16-byte bank
// groups, i.e. all four exchange patterns are bank-conflict free.
// ---------------------------------------------------------------------------
B200_HD int x1_slot(int q, int j0) {
  return q * 64 + (j0 ^ (((j0 >> 3) & 1) << 1) ^ (q & 1));
}
B200_HD int x2_slot(int row, int b) {
  return row * 16 + (b ^ ((b >> 3) << 1) ^ (((row & 3) << 1) | ((row >> 2) & 1)));
}

B200_HD void x1_store_p1(cplx *buf, int t, const cplx v[16]) {
#pragma unroll
  for (int q = 0; q < 16; q++)
    buf[x1_slot(q, t)] = v[q];
}
B200_HD void x1_load_p1(const cplx *buf, int t, cplx v[16]) {
#pragma unroll
  for (int q = 0; q < 16; q++)
    v[q] = buf[x1_slot(q, t)];
}
B200_HD void x1_load_p2(const cplx *buf, int t, cplx v[16]) {
  const int q = t >> 2, bh = t & 3;
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
#pragma unroll
    for (int a = 0; a < 4; a++)
      v[4 * bl + a] = buf[x1_slot(q, 16 * a + 4 * bh + bl)];
}
B200_HD void x1_store_p2(cplx *buf, int t, const cplx v[16]) {
  const int q = t >> 2, bh = t & 3;
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
#pragma unroll
    for (int a = 0; a < 4; a++)
      buf[x1_slot(q, 16 * a + 4 * bh + bl)] = v[4 * bl + a];
}
B200_HD void x2_store_p2(cplx *buf, int t, const cplx v[16]) {
  const int q = t >> 2, bh = t & 3;
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
#pragma unroll
    for (int a = 0; a < 4; a++)
      buf[x2_slot(4 * q + a, 4 * bh + bl)] = v[4 * bl + a];
}
B200_HD void x2_load_p2(const cplx *buf, int t, cplx v[16]) {
  const int q = t >> 2, bh = t & 3;
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
#pragma unroll
    for (int a = 0; a < 4; a++)
      v[4 * bl + a] = buf[x2_slot(4 * q + a, 4 * bh + bl)];
}
B200_HD void x2_load_p3(const cplx *buf, int t, cplx v[16]) {
#pragma unroll
  for (int b = 0; b < 16; b++)
    v[b] = buf[x2_slot(t, b)];
}
B200_HD void x2_store_p3(cplx *buf, int t, const cplx v[16]) {
#pragma unroll
  for (int b = 0; b < 16; b++)
    buf[x2_slot(t, b)] = v[b];
}
// ---------------------------------------------------------------------------
// Exchange 1 for the shuffle variant of exchange 2 (x2_shfl.cuh): the
// pass-2 work is assigned as  lane p + 8 m of warp w  <->  (sub-problem
// q = 8 w + p, quarter bh = m), so that the four threads of a sub-problem sit
// on lanes p, p + 8, p + 16, p + 24 and exchange 2 is a 4 x 4 block transpose
// between those lanes and lanes 4 p .. 4 p + 3 of the same warp.  A quarter-warp now holds 8 different q and one j0, hence
// the swizzle by q & 7:  X1T slot of element (q, j0) = q*64 + (j0 ^ (q & 7)).
// Conflict-free for all four access patterns (emu_exchange_conflict_audit).
// ---------------------------------------------------------------------------
B200_HD int x1t_slot(int q, int j0) { return q * 64 + (j0 ^ (q & 7)); }
B200_HD int x1t_q(int t) { return ((t >> 5) << 3) | (t & 7); }
B200_HD int x1t_bh(int t) { return (t >> 3) & 3; }
B200_HD void x1t_store_p1(cplx *buf, int t, const cplx v[16]) {
#pragma unroll
  for (int q = 0; q < 16; q++)
    buf[x1t_slot(q, t)] = v[q];
}
B200_HD void x1t_load_p1(const cplx *buf, int t, cplx v[16]) {
#pragma unroll
  for (int q = 0; q < 16; q++)
    v[q] = buf[x1t_slot(q, t)];
}
B200_HD void x1t_load_p2(const cplx *buf, int t, cplx v[16]) {
  const int q = x1t_q(t), bh = x1t_bh(t);
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
#pragma unroll
    for (int a = 0; a < 4; a++)
      v[4 * bl + a] = buf[x1t_slot(q, 16 * a + 4 * bh + bl)];
}
B200_HD void x1t_store_p2(cplx *buf, int t, const cplx v[16]) {
  const int q = x1t_q(t), bh = x1t_bh(t);
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
#pragma unroll
    for (int a = 0; a < 4; a++)
      buf[x1t_slot(q, 16 * a + 4 * bh + bl)] = v[4 * bl + a];
}
// ---------------------------------------------------------------------------
// Exchange 1 for the lane-pair layout (half-warp exchange 2, x2h_* in
// x2_shfl.cuh): warp w holds t = 16 w + i (i = lane & 15) of BOTH polynomials,
// polynomial 0 on lanes 0-15 and polynomial 1 on lanes 16-31, each in its own
// buffer.  Pass-2 work: half-lane p + 4 m <-> (sub-problem q = 4 w + p,
// quarter bh = m).  A pass-2 quarter-warp holds 4 q (p = 0..3) and 2 quarters,
// so the j0 it reads differ in bit 2 (bh) and in bits 0-1 only through the
// swizzle by q & 3:  X1H slot of element (q, j0) = q*64 + (j0 ^ (q & 3)).  A
// pass-1 quarter-warp holds 8 aligned consecutive j0 and one q.  Both sides hit
// 8 distinct 16-byte bank groups (emu_lanepair_conflict_audit).
// Warp w's pass-2 accesses stay in rows 4 w .. 4 w + 3 of each buffer.
// ---------------------------------------------------------------------------
B200_HD int x1h_slot(int q, int j0) { return q * 64 + (j0 ^ (q & 3)); }
B200_HD int x1h_q(int t) { return ((t >> 4) << 2) | (t & 3); }
B200_HD int x1h_bh(int t) { return (t >> 2) & 3; }
B200_HD void x1h_store_p1(cplx *buf, int t, const cplx v[16]) {
#pragma unroll
  for (int q = 0; q < 16; q++)
    buf[x1h_slot(q, t)] = v[q];
}
B200_HD void x1h_load_p1(const cplx *buf, int t, cplx v[16]) {
#pragma unroll
  for (int q = 0; q < 16; q++)
    v[q] = buf[x1h_slot(q, t)];
}
B200_HD void x1h_load_p2(const cplx *buf, int t, cplx v[16]) {
  const int q = x1h_q(t), bh = x1h_bh(t);
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
#pragma unroll
    for (int a = 0; a < 4; a++)
      v[4 * bl + a] = buf[x1h_slot(q, 16 * a + 4 * bh + bl)];
}
B200_HD void x1h_store_p2(cplx *buf, int t, const cplx v[16]) {
  const int q = x1h_q(t), bh = x1h_bh(t);
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
#pragma unroll
    for (int a = 0; a < 4; a++)
      buf[x1h_slot(q, 16 * a + 4 * bh + bl)] = v[4 * bl + a];
}
// spectrum layout used for sharing and for the Fourier BSK: index b*64 + t
B200_HD void spec_store(cplx *buf, int t, const cplx v[16]) {
#pragma unroll
  for (int b = 0; b < 16; b++)
    buf[b * 64 + t] = v[b];
}

// frequency slot of (thread t, register b) in pass-3 layout: pos = 16 t + b,
// value = Z(t^(1 + 4*bitrev10(pos))).
B200_HD int fft1024_pos(int t, int b) { return 16 * t + b; }

// ===========================================================================
// M = 256 (N = 512) split as 16 x 16: 16 threads per polynomial, 16 complex
// values per thread, ONE exchange per transform (a 16 x 16 transpose inside a
// half-warp: warp-level synchronisation only).
//   pass 1 (levels 1-4): thread u holds coefficients j = 16*j1 + u in v[j1];
//           twiddles identical for all threads (15 constants)
//   pass 2 (levels 5-8): thread q holds sub-problem q, v[b]; per q:
//           [0..2] layer A: s1=tw(5,q) s2=tw(6,2q) s3; [3+3u..] layer B, u<4:
//           s1=tw(7,4q+u) s2=tw(8,2(4q+u)) s3                      -> [16][15]
// Output slot pos = 16*q + b holds Z(t^(1 + 4*bitrev8(pos))), t = exp(i pi/512).
// Exchange slot of element (q, u): q*16 + (u ^ (q & 7)) -- both the pass-1
// side (8 consecutive u, one q) and the pass-2 side (8 consecutive q, one u)
// of a quarter-warp hit 8 distinct 16-byte bank groups.
// ===========================================================================
struct Fft256Tables {
  cplx pass1[15];
  cplx pass2[16][15];
};
static inline void b200_fill_fft256_tables(Fft256Tables *t) {
  const uint32_t lm = 8;
  b200_triple(&t->pass1[0], lm, 1, 0);
  for (uint32_t u = 0; u < 4; u++)
    b200_triple(&t->pass1[3 + 3 * u], lm, 3, u);
  for (uint32_t q = 0; q < 16; q++) {
    b200_triple(&t->pass2[q][0], lm, 5, q);
    for (uint32_t u = 0; u < 4; u++)
      b200_triple(&t->pass2[q][3 + 3 * u], lm, 7, 4 * q + u);
  }
}
B200_HD int xq_slot(int q, int u) { return q * 16 + (u ^ (q & 7)); }
// pass-1 side: thread u <-> element (q = register, u)
B200_HD void xq_store_p1(cplx *buf, int u, const cplx v[16]) {
#pragma unroll
  for (int q = 0; q < 16; q++)
    buf[xq_slot(q, u)] = v[q];
}
B200_HD void xq_load_p1(const cplx *buf, int u, cplx v[16]) {
#pragma unroll
  for (int q = 0; q < 16; q++)
    v[q] = buf[xq_slot(q, u)];
}
// pass-2 side: thread q <-> element (q, u = register)
B200_HD void xq_load_p2(const cplx *buf, int q, cplx v[16]) {
#pragma unroll
  for (int u = 0; u < 16; u++)
    v[u] = buf[xq_slot(q, u)];
}
B200_HD void xq_store_p2(cplx *buf, int q, const cplx v[16]) {
#pragma unroll
  for (int u = 0; u < 16; u++)
    buf[xq_slot(q, u)] = v[u];
}
// spectrum layout for sharing and for the Fourier key: index b*16 + q
B200_HD void spec256_store(cplx *buf, int q, const cplx v[16]) {
#pragma unroll
  for (int b = 0; b < 16; b++)
    buf[b * 16 + q] = v[b];
}

// ===========================================================================
// M = 4096 (N = 8192) split as 16 x 16 x 16: 256 threads per polynomial, 16
// complex values per thread, three radix-16 passes, two exchanges.
//   pass 1 (levels 1-4):  thread t holds coefficients j = 256*j1 + t in v[j1];
//           15 constants (same for all threads)
//   exchange 1 (across the 256 threads, shared memory + CTA barrier): element
//           (q1, m, b), t = 16 m + b, moves from (thread (m,b), register q1) to
//           (thread 16 q1 + b, register m); buffer slot q1*256 + 16 m + b -- the
//           region [256 q1, 256 q1 + 256) is read only by half-warp q1
//   pass 2 (levels 5-8):  per q1: s1=tw(5,q1) s2=tw(6,2q1) s3, then for u<4
//           s1=tw(7,4q1+u) s2=tw(8,2(4q1+u)) s3                       -> [16][15]
//   exchange 2 (inside the half-warp q1, in its own region of the buffer,
//           __syncwarp): the 16 x 16 transpose of the N = 512 kernel (xq_*)
//   pass 3 (levels 9-12): per u8 = 16 q1 + q2: tw(9,u8), tw(10,2u8), s3, then
//           for u<4 tw(11,4u8+u), tw(12,2(4u8+u)), s3                  -> [256][15]
// Output: thread t3 = 16 q1 + q2 holds v[b]; slot pos = 16 t3 + b holds
// Z(t^(1 + 4*bitrev12(pos))), t = exp(i pi / 8192).
// ===========================================================================
struct Fft4096Tables {
  cplx pass1[15];
  cplx pass2[16][15];
  cplx pass3[256][15];
};
static inline void b200_fill_fft4096_tables(Fft4096Tables *t) {
  const uint32_t lm = 12;
  b200_triple(&t->pass1[0], lm, 1, 0);
  for (uint32_t u = 0; u < 4; u++)
    b200_triple(&t->pass1[3 + 3 * u], lm, 3, u);
  for (uint32_t q = 0; q < 16; q++) {
    b200_triple(&t->pass2[q][0], lm, 5, q);
    for (uint32_t u = 0; u < 4; u++)
      b200_triple(&t->pass2[q][3 + 3 * u], lm, 7, 4 * q + u);
  }
  for (uint32_t u8 = 0; u8 < 256; u8++) {
    b200_triple(&t->pass3[u8][0], lm, 9, u8);
    for (uint32_t u = 0; u < 4; u++)
      b200_triple(&t->pass3[u8][3 + 3 * u], lm, 11, 4 * u8 + u);
  }
}
// exchange 1 of the 4096-point transform (no swizzle needed: every 128-bit
// access of a quarter-warp covers 8 consecutive slots)
B200_HD void xg_store_p1(cplx *buf, int t, const cplx v[16]) {
#pragma unroll
  for (int q1 = 0; q1 < 16; q1++)
    buf[q1 * 256 + t] = v[q1];
}
B200_HD void xg_load_p1(const cplx *buf, int t, cplx v[16]) {
#pragma unroll
  for (int q1 = 0; q1 < 16; q1++)
    v[q1] = buf[q1 * 256 + t];
}
B200_HD void xg_load_p2(const cplx *buf, int t2, cplx v[16]) {
  const int q1 = t2 >> 4, b = t2 & 15;
#pragma unroll
  for (int m = 0; m < 16; m++)
    v[m] = buf[q1 * 256 + 16 * m + b];
}
B200_HD void xg_store_p2(cplx *buf, int t2, const cplx v[16]) {
  const int q1 = t2 >> 4, b = t2 & 15;
#pragma unroll
  for (int m = 0; m < 16; m++)
    buf[q1 * 256 + 16 * m + b] = v[m];
}
