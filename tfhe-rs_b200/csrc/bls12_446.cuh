// bls12_446.cuh -- BLS12-446 field and curve arithmetic (tfhe-zk-pok's PKE v2
// curve), __host__ __device__ so the CPU tests compile the same code with g++.
//
// Fp: the 446-bit prime p = (x - 1)^2 r / 3 + x, r = x^4 - x^2 + 1, of the
// seed x = -0x600_8204000000020001, in Montgomery form with R = 2^448.  In
// memory an element is 7 x u64 little-endian limbs (the C ABI's Fp).  Device
// code multiplies on 14 x u32 limbs with PTX carry chains (CIOS: each of the
// 14 rows is a mad.lo chain and a mad.hi chain for a * b_i, then the same for
// m * p); host code on 7 x u64 limbs with unsigned __int128.  p < R / 4, so a
// CIOS row never overflows 15 words; every value a function returns is fully
// reduced (< p), so results compare word for word.
// Fp2 = Fp[u] / (u^2 + 1) (p = 3 mod 4), Karatsuba multiplication.
// G1: y^2 = x^3 + 1 over Fp; G2: the M-type twist y^2 = x^3 + (1 + u).
// Buckets are XYZZ points (x = X / ZZ, y = Y / ZZZ, ZZ^3 = ZZZ^2; the identity
// has ZZ = 0), updated by the a = 0 formulas of the EFD (madd-2008-s,
// add-2008-s, dbl-2008-s-1, mdbl-2008-s-1), with P + P sent to doubling and
// P + (-P) to the identity.
#pragma once
#include <cstdint>

#include "../../include/tfhe_b200_zk.h"

#ifdef __CUDACC__
#define ZK_HD __host__ __device__ __forceinline__
#else
#define ZK_HD inline
#endif

namespace zk {

constexpr int NL = 7;                       // u64 limbs
constexpr int SCALAR_BITS = 320;            // the ABI's Scalar width
constexpr uint64_t PINV = 0xcd63fd900035fffdULL;  // -p^-1 mod 2^64

ZK_HD uint64_t p_limb(int i) {
  constexpr uint64_t v[NL] = {0x311c0026aab0aaabULL, 0x56ee4528c573b5ccULL, 0x824e6dc3e23acdeeULL,
                              0x0f75a64bbac71602ULL, 0x0095a4b78a02fe32ULL, 0x200fc34965aad640ULL,
                              0x3cdee0fb28c5e535ULL};
  return v[i];
}
// R^2 mod p (to Montgomery form)
ZK_HD uint64_t r2_limb(int i) {
  constexpr uint64_t v[NL] = {0x2aff01dddc752b45ULL, 0x92c772a7421ccf5bULL, 0x140eef29c347dad6ULL,
                              0xf5a1400c22ea595eULL, 0x99d91c9fec145218ULL, 0x3bb6537f90143d4bULL,
                              0x3627854c9be7974fULL};
  return v[i];
}
// R mod p (1 in Montgomery form)
ZK_HD uint64_t one_limb(int i) {
  constexpr uint64_t v[NL] = {0x3b8fff65553d5554ULL, 0xa446eb5cea3128cfULL, 0xf6c648f07714c846ULL,
                              0xc22966d114e3a7f5ULL, 0xfda96d21d7f40737ULL, 0x7fc0f2da6954a6ffULL,
                              0x0c847c135ce86b2bULL};
  return v[i];
}
// the group order r (299 bits)
ZK_HD uint64_t r_limb(int i) {
  constexpr uint64_t v[5] = {0x0428001400040001ULL, 0x7bb9b0e8d8ca3461ULL, 0xd04c98ccc4c050bcULL,
                             0x7995b34995830fa4ULL, 0x00000511b70539f2ULL};
  return v[i];
}

// ---------------------------------------------------------------- Fp ------

ZK_HD void fp_zero(Fp &a) {
#pragma unroll
  for (int i = 0; i < NL; i++) a.limb[i] = 0;
}
ZK_HD void fp_one(Fp &a) {  // Montgomery form
#pragma unroll
  for (int i = 0; i < NL; i++) a.limb[i] = one_limb(i);
}
ZK_HD bool fp_is_zero(const Fp &a) {
  uint64_t t = 0;
#pragma unroll
  for (int i = 0; i < NL; i++) t |= a.limb[i];
  return t == 0;
}
ZK_HD bool fp_eq(const Fp &a, const Fp &b) {
  uint64_t t = 0;
#pragma unroll
  for (int i = 0; i < NL; i++) t |= a.limb[i] ^ b.limb[i];
  return t == 0;
}

#ifdef __CUDA_ARCH__
// ---- device: 14 x u32 limbs, PTX carry chains ----
__device__ __forceinline__ uint32_t p32(int j) { return (uint32_t)(p_limb(j >> 1) >> (32 * (j & 1))); }

__device__ __forceinline__ void split(uint32_t r[14], const Fp &a) {
#pragma unroll
  for (int i = 0; i < NL; i++) {
    r[2 * i] = (uint32_t)a.limb[i];
    r[2 * i + 1] = (uint32_t)(a.limb[i] >> 32);
  }
}
__device__ __forceinline__ void join(Fp &a, const uint32_t r[14]) {
#pragma unroll
  for (int i = 0; i < NL; i++) a.limb[i] = ((uint64_t)r[2 * i + 1] << 32) | r[2 * i];
}

// r = t - p if t >= p else t (t < 2p)
__device__ __forceinline__ void reduce_once(uint32_t t[14]) {
  uint32_t d[14], borrow;
  asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(d[0]) : "r"(t[0]), "r"(p32(0)));
#pragma unroll
  for (int j = 1; j < 14; j++)
    asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(d[j]) : "r"(t[j]), "r"(p32(j)));
  asm volatile("subc.u32 %0, 0, 0;" : "=r"(borrow));
#pragma unroll
  for (int j = 0; j < 14; j++) t[j] = borrow ? t[j] : d[j];
}

// t[0..14] += a[0..13] * b  (t < 2^479 before and after)
__device__ __forceinline__ void mac_row(uint32_t t[15], const uint32_t a[14], uint32_t b) {
  asm volatile("mad.lo.cc.u32 %0, %1, %2, %0;" : "+r"(t[0]) : "r"(a[0]), "r"(b));
#pragma unroll
  for (int j = 1; j < 14; j++)
    asm volatile("madc.lo.cc.u32 %0, %1, %2, %0;" : "+r"(t[j]) : "r"(a[j]), "r"(b));
  asm volatile("addc.u32 %0, %0, 0;" : "+r"(t[14]));
  asm volatile("mad.hi.cc.u32 %0, %1, %2, %0;" : "+r"(t[1]) : "r"(a[0]), "r"(b));
#pragma unroll
  for (int j = 1; j < 13; j++)
    asm volatile("madc.hi.cc.u32 %0, %1, %2, %0;" : "+r"(t[j + 1]) : "r"(a[j]), "r"(b));
  asm volatile("madc.hi.u32 %0, %1, %2, %0;" : "+r"(t[14]) : "r"(a[13]), "r"(b));
}
// t[0..14] += m * p
__device__ __forceinline__ void mac_row_p(uint32_t t[15], uint32_t m) {
  asm volatile("mad.lo.cc.u32 %0, %1, %2, %0;" : "+r"(t[0]) : "r"(m), "r"(p32(0)));
#pragma unroll
  for (int j = 1; j < 14; j++)
    asm volatile("madc.lo.cc.u32 %0, %1, %2, %0;" : "+r"(t[j]) : "r"(m), "r"(p32(j)));
  asm volatile("addc.u32 %0, %0, 0;" : "+r"(t[14]));
  asm volatile("mad.hi.cc.u32 %0, %1, %2, %0;" : "+r"(t[1]) : "r"(m), "r"(p32(0)));
#pragma unroll
  for (int j = 1; j < 13; j++)
    asm volatile("madc.hi.cc.u32 %0, %1, %2, %0;" : "+r"(t[j + 1]) : "r"(m), "r"(p32(j)));
  asm volatile("madc.hi.u32 %0, %1, %2, %0;" : "+r"(t[14]) : "r"(m), "r"(p32(13)));
}

// one out-of-line copy (about 800 instructions): a point formula calls it a
// dozen times, and inlining each would overflow the instruction cache
__device__ __noinline__ Fp fp_mul_call(const Fp a, const Fp b) {
  uint32_t x[14], y[14], t[15];
  Fp c;
  split(x, a);
  split(y, b);
#pragma unroll
  for (int j = 0; j < 15; j++) t[j] = 0;
#pragma unroll
  for (int i = 0; i < 14; i++) {
    mac_row(t, x, y[i]);
    mac_row_p(t, t[0] * (uint32_t)PINV);
#pragma unroll
    for (int j = 0; j < 14; j++) t[j] = t[j + 1];  // t[0] is 0
    t[14] = 0;
  }
  reduce_once(t);
  join(c, t);
  return c;
}
__device__ __forceinline__ void fp_mul(Fp &c, const Fp &a, const Fp &b) { c = fp_mul_call(a, b); }

__device__ __forceinline__ void fp_add(Fp &c, const Fp &a, const Fp &b) {
  uint32_t x[14], y[14];
  split(x, a);
  split(y, b);
  asm volatile("add.cc.u32 %0, %0, %1;" : "+r"(x[0]) : "r"(y[0]));
#pragma unroll
  for (int j = 1; j < 14; j++) asm volatile("addc.cc.u32 %0, %0, %1;" : "+r"(x[j]) : "r"(y[j]));
  reduce_once(x);  // a + b < 2p < 2^448: no carry out
  join(c, x);
}

__device__ __forceinline__ void fp_sub(Fp &c, const Fp &a, const Fp &b) {
  uint32_t x[14], y[14], borrow, s[14];
  split(x, a);
  split(y, b);
  asm volatile("sub.cc.u32 %0, %0, %1;" : "+r"(x[0]) : "r"(y[0]));
#pragma unroll
  for (int j = 1; j < 14; j++) asm volatile("subc.cc.u32 %0, %0, %1;" : "+r"(x[j]) : "r"(y[j]));
  asm volatile("subc.u32 %0, 0, 0;" : "=r"(borrow));
  // add p back where a < b
  asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(s[0]) : "r"(x[0]), "r"(p32(0) & borrow));
#pragma unroll
  for (int j = 1; j < 14; j++)
    asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(s[j]) : "r"(x[j]), "r"(p32(j) & borrow));
  join(c, s);
}

#else
// ---- host: 7 x u64 limbs, unsigned __int128 ----
typedef unsigned __int128 u128;

inline void reduce_once64(uint64_t t[NL]) {
  uint64_t d[NL], borrow = 0;
  for (int j = 0; j < NL; j++) {
    u128 s = (u128)t[j] - p_limb(j) - borrow;
    d[j] = (uint64_t)s;
    borrow = (uint64_t)(s >> 64) & 1;
  }
  if (!borrow)
    for (int j = 0; j < NL; j++) t[j] = d[j];
}

inline void fp_mul(Fp &c, const Fp &a, const Fp &b) {
  uint64_t t[NL + 1] = {0};
  for (int i = 0; i < NL; i++) {
    uint64_t carry = 0;
    for (int j = 0; j < NL; j++) {
      u128 s = (u128)a.limb[j] * b.limb[i] + t[j] + carry;
      t[j] = (uint64_t)s;
      carry = (uint64_t)(s >> 64);
    }
    t[NL] += carry;
    uint64_t m = t[0] * PINV;
    u128 s = (u128)m * p_limb(0) + t[0];
    carry = (uint64_t)(s >> 64);
    for (int j = 1; j < NL; j++) {
      s = (u128)m * p_limb(j) + t[j] + carry;
      t[j - 1] = (uint64_t)s;
      carry = (uint64_t)(s >> 64);
    }
    s = (u128)t[NL] + carry;
    t[NL - 1] = (uint64_t)s;
    t[NL] = (uint64_t)(s >> 64);
  }
  reduce_once64(t);
  for (int j = 0; j < NL; j++) c.limb[j] = t[j];
}

inline void fp_add(Fp &c, const Fp &a, const Fp &b) {
  uint64_t t[NL], carry = 0;
  for (int j = 0; j < NL; j++) {
    u128 s = (u128)a.limb[j] + b.limb[j] + carry;
    t[j] = (uint64_t)s;
    carry = (uint64_t)(s >> 64);
  }
  reduce_once64(t);
  for (int j = 0; j < NL; j++) c.limb[j] = t[j];
}

inline void fp_sub(Fp &c, const Fp &a, const Fp &b) {
  uint64_t t[NL], borrow = 0;
  for (int j = 0; j < NL; j++) {
    u128 s = (u128)a.limb[j] - b.limb[j] - borrow;
    t[j] = (uint64_t)s;
    borrow = (uint64_t)(s >> 64) & 1;
  }
  uint64_t mask = 0 - borrow, carry = 0;
  for (int j = 0; j < NL; j++) {
    u128 s = (u128)t[j] + (p_limb(j) & mask) + carry;
    c.limb[j] = (uint64_t)s;
    carry = (uint64_t)(s >> 64);
  }
}
#endif

ZK_HD void fp_sqr(Fp &c, const Fp &a) { fp_mul(c, a, a); }
ZK_HD void fp_neg(Fp &c, const Fp &a) {
  Fp z;
  fp_zero(z);
  fp_sub(c, z, a);
}
ZK_HD void fp_to_montgomery(Fp &c, const Fp &a) {
  Fp r2;
#pragma unroll
  for (int i = 0; i < NL; i++) r2.limb[i] = r2_limb(i);
  fp_mul(c, a, r2);
}
ZK_HD void fp_from_montgomery(Fp &c, const Fp &a) {
  Fp one;
  fp_zero(one);
  one.limb[0] = 1;
  fp_mul(c, a, one);
}
ZK_HD void fp_to_montgomery(Fp2 &c, const Fp2 &a) {
  fp_to_montgomery(c.c0, a.c0), fp_to_montgomery(c.c1, a.c1);
}
ZK_HD void fp_from_montgomery(Fp2 &c, const Fp2 &a) {
  fp_from_montgomery(c.c0, a.c0), fp_from_montgomery(c.c1, a.c1);
}
// a^(p - 2) (Fermat); 0 maps to 0
inline void fp_inv(Fp &c, const Fp &a) {
  Fp acc, base = a;
  fp_one(acc);
  for (int i = 0; i < NL; i++) {
    uint64_t e = p_limb(i) - (i == 0 ? 2 : 0);  // p is odd and > 2: no borrow
    for (int b = 0; b < 64; b++) {
      if ((e >> b) & 1) fp_mul(acc, acc, base);
      fp_sqr(base, base);
    }
  }
  c = acc;
}

// ---------------------------------------------------------------- Fp2 -----

ZK_HD void fp_zero(Fp2 &a) { fp_zero(a.c0), fp_zero(a.c1); }
ZK_HD void fp_one(Fp2 &a) { fp_one(a.c0), fp_zero(a.c1); }
ZK_HD bool fp_is_zero(const Fp2 &a) { return fp_is_zero(a.c0) && fp_is_zero(a.c1); }
ZK_HD bool fp_eq(const Fp2 &a, const Fp2 &b) { return fp_eq(a.c0, b.c0) && fp_eq(a.c1, b.c1); }
ZK_HD void fp_add(Fp2 &c, const Fp2 &a, const Fp2 &b) { fp_add(c.c0, a.c0, b.c0), fp_add(c.c1, a.c1, b.c1); }
ZK_HD void fp_sub(Fp2 &c, const Fp2 &a, const Fp2 &b) { fp_sub(c.c0, a.c0, b.c0), fp_sub(c.c1, a.c1, b.c1); }
ZK_HD void fp_neg(Fp2 &c, const Fp2 &a) { fp_neg(c.c0, a.c0), fp_neg(c.c1, a.c1); }
// (a0 + a1 u)(b0 + b1 u) = a0 b0 - a1 b1 + ((a0 + a1)(b0 + b1) - a0 b0 - a1 b1) u
ZK_HD void fp_mul(Fp2 &c, const Fp2 &a, const Fp2 &b) {
  Fp v0, v1, s, t;
  fp_mul(v0, a.c0, b.c0);
  fp_mul(v1, a.c1, b.c1);
  fp_add(s, a.c0, a.c1);
  fp_add(t, b.c0, b.c1);
  fp_mul(s, s, t);
  fp_sub(s, s, v0);
  fp_sub(c.c1, s, v1);
  fp_sub(c.c0, v0, v1);
}
// (a0 + a1 u)^2 = (a0 + a1)(a0 - a1) + 2 a0 a1 u
ZK_HD void fp_sqr(Fp2 &c, const Fp2 &a) {
  Fp s, d, m;
  fp_add(s, a.c0, a.c1);
  fp_sub(d, a.c0, a.c1);
  fp_mul(m, a.c0, a.c1);
  fp_mul(c.c0, s, d);
  fp_add(c.c1, m, m);
}
inline void fp_inv(Fp2 &c, const Fp2 &a) {
  Fp n, t;
  fp_sqr(n, a.c0);
  fp_sqr(t, a.c1);
  fp_add(n, n, t);
  fp_inv(n, n);
  fp_mul(c.c0, a.c0, n);
  fp_mul(t, a.c1, n);
  fp_neg(c.c1, t);
}

// ---------------------------------------------------------------- curves --

// curve coefficient b in Montgomery form: 1 for G1, 1 + u for G2
ZK_HD void curve_b(Fp &b) { fp_one(b); }
ZK_HD void curve_b(Fp2 &b) { fp_one(b.c0), fp_one(b.c1); }

template <class F> struct Xyzz {
  F X, Y, ZZ, ZZZ;
};

template <class F> ZK_HD void xyzz_set_identity(Xyzz<F> &p) {
  fp_zero(p.X), fp_zero(p.Y), fp_zero(p.ZZ), fp_zero(p.ZZZ);
}
template <class F> ZK_HD bool xyzz_is_identity(const Xyzz<F> &p) { return fp_is_zero(p.ZZ); }

// r = 2 p (dbl-2008-s-1, a = 0); a point with Y = 0 doubles to the identity
template <class F> ZK_HD void xyzz_dbl(Xyzz<F> &r, const Xyzz<F> &p) {
  F U, V, W, S, M, t;
  fp_add(U, p.Y, p.Y);
  fp_sqr(V, U);
  fp_mul(W, U, V);
  fp_mul(S, p.X, V);
  fp_sqr(M, p.X);
  fp_add(t, M, M);
  fp_add(M, t, M);
  fp_mul(r.ZZ, V, p.ZZ);
  fp_mul(r.ZZZ, W, p.ZZZ);
  fp_mul(W, W, p.Y);
  fp_sqr(t, M);
  fp_sub(t, t, S);
  fp_sub(r.X, t, S);
  fp_sub(S, S, r.X);
  fp_mul(S, M, S);
  fp_sub(r.Y, S, W);
}

// r = 2 (x, y) for an affine point (mdbl-2008-s-1)
template <class F> ZK_HD void xyzz_dbl_affine(Xyzz<F> &r, const F &x, const F &y) {
  F U, V, W, S, M, t;
  fp_add(U, y, y);
  fp_sqr(V, U);
  fp_mul(W, U, V);
  fp_mul(S, x, V);
  fp_sqr(M, x);
  fp_add(t, M, M);
  fp_add(M, t, M);
  r.ZZ = V;
  r.ZZZ = W;
  fp_mul(W, W, y);
  fp_sqr(t, M);
  fp_sub(t, t, S);
  fp_sub(r.X, t, S);
  fp_sub(S, S, r.X);
  fp_mul(S, M, S);
  fp_sub(r.Y, S, W);
}

// acc += (x, y), an affine point that is not the identity (madd-2008-s)
template <class F> ZK_HD void xyzz_add_affine(Xyzz<F> &acc, const F &x, const F &y) {
  if (xyzz_is_identity(acc)) {
    acc.X = x, acc.Y = y;
    fp_one(acc.ZZ), fp_one(acc.ZZZ);
    return;
  }
  F P, R, PP, PPP, Q, t;
  fp_mul(P, x, acc.ZZ);
  fp_sub(P, P, acc.X);
  fp_mul(R, y, acc.ZZZ);
  fp_sub(R, R, acc.Y);
  if (fp_is_zero(P)) {
    if (fp_is_zero(R))
      xyzz_dbl_affine(acc, x, y);
    else
      xyzz_set_identity(acc);
    return;
  }
  fp_sqr(PP, P);
  fp_mul(PPP, P, PP);
  fp_mul(Q, acc.X, PP);
  fp_mul(acc.ZZ, acc.ZZ, PP);
  fp_mul(acc.ZZZ, acc.ZZZ, PPP);
  fp_sqr(t, R);
  fp_sub(t, t, PPP);
  fp_sub(t, t, Q);
  fp_sub(acc.X, t, Q);
  fp_sub(Q, Q, acc.X);
  fp_mul(Q, R, Q);
  fp_mul(t, acc.Y, PPP);
  fp_sub(acc.Y, Q, t);
}

// acc += q (add-2008-s)
template <class F> ZK_HD void xyzz_add(Xyzz<F> &acc, const Xyzz<F> &q) {
  if (xyzz_is_identity(q))
    return;
  if (xyzz_is_identity(acc)) {
    acc = q;
    return;
  }
  F U1, S1, P, R, PP, PPP, Q, t;
  fp_mul(U1, acc.X, q.ZZ);
  fp_mul(P, q.X, acc.ZZ);
  fp_sub(P, P, U1);
  fp_mul(S1, acc.Y, q.ZZZ);
  fp_mul(R, q.Y, acc.ZZZ);
  fp_sub(R, R, S1);
  if (fp_is_zero(P)) {
    if (fp_is_zero(R))
      xyzz_dbl(acc, acc);
    else
      xyzz_set_identity(acc);
    return;
  }
  fp_sqr(PP, P);
  fp_mul(PPP, P, PP);
  fp_mul(Q, U1, PP);
  fp_mul(acc.ZZ, acc.ZZ, q.ZZ);
  fp_mul(acc.ZZ, acc.ZZ, PP);
  fp_mul(acc.ZZZ, acc.ZZZ, q.ZZZ);
  fp_mul(acc.ZZZ, acc.ZZZ, PPP);
  fp_sqr(t, R);
  fp_sub(t, t, PPP);
  fp_sub(t, t, Q);
  fp_sub(acc.X, t, Q);
  fp_sub(Q, Q, acc.X);
  fp_mul(Q, R, Q);
  fp_mul(t, S1, PPP);
  fp_sub(acc.Y, Q, t);
}

// (X, Y, ZZ, ZZZ) -> homogeneous (X ZZZ, Y ZZ, ZZ ZZZ); the identity -> (0, 0, 0)
template <class F, class Proj> ZK_HD void xyzz_to_projective(Proj &r, const Xyzz<F> &p) {
  fp_mul(r.X, p.X, p.ZZZ);
  fp_mul(r.Y, p.Y, p.ZZ);
  fp_mul(r.Z, p.ZZ, p.ZZZ);
}

// y^2 == x^3 + b, coordinates in Montgomery form
template <class F> ZK_HD bool on_curve_mont(const F &x, const F &y) {
  F l, r, b;
  fp_sqr(l, y);
  fp_sqr(r, x);
  fp_mul(r, r, x);
  curve_b(b);
  fp_add(r, r, b);
  return fp_eq(l, r);
}

// ---------------------------------------------------------------- scalars -

// number of signed c-bit windows of a 320-bit scalar: one more than the full
// windows, so the top window absorbs the last carry (it holds 320 mod c < c
// bits plus the carry, at most 2^(c-1): never negative)
ZK_HD int num_windows(int c) { return SCALAR_BITS / c + 1; }

// signed c-bit digits of k (5 x u64): k = sum d_w 2^(c w), d_w in
// (-2^(c-1), 2^(c-1)]; writes num_windows(c) digits
ZK_HD void signed_digits(int32_t *d, const uint64_t k[5], int c) {
  const int W = num_windows(c);
  uint32_t carry = 0;
  for (int w = 0; w < W; w++) {
    const int bit = w * c;
    uint64_t v = 0;
    if (bit < SCALAR_BITS) {
      const int limb = bit >> 6, off = bit & 63;
      v = k[limb] >> off;
      if (off + c > 64 && limb + 1 < 5)
        v |= k[limb + 1] << (64 - off);
      v &= (1ULL << c) - 1;
    }
    int64_t raw = (int64_t)v + carry;
    if (raw > (int64_t)1 << (c - 1)) {
      d[w] = (int32_t)(raw - ((int64_t)1 << c));
      carry = 1;
    } else {
      d[w] = (int32_t)raw;
      carry = 0;
    }
  }
}

}  // namespace zk
