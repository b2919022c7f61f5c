// CPU build of tfhe-rs_b200/csrc/bls12_446.cuh (its unsigned __int128 path):
// the field, XYZZ point and window-digit code that the MSM kernels run,
// exported for tests/test_zk_msm.py.  All elements are in Montgomery form.
#include "../../tfhe-rs_b200/csrc/bls12_446.cuh"

#include <cstddef>
#include <cstring>

using namespace zk;

template <class A> static Xyzz<decltype(A::x)> from_affine(const A &p) {
  Xyzz<decltype(A::x)> r;
  xyzz_set_identity(r);
  if (!p.infinity)
    xyzz_add_affine(r, p.x, p.y);
  return r;
}

template <class A> static void to_affine(A &out, const Xyzz<decltype(A::x)> &p) {
  std::memset(&out, 0, sizeof(out));
  if (xyzz_is_identity(p)) {
    out.infinity = true;
    return;
  }
  decltype(A::x) zz, zzz;
  fp_inv(zz, p.ZZ);
  fp_inv(zzz, p.ZZZ);
  fp_mul(out.x, p.X, zz);
  fp_mul(out.y, p.Y, zzz);
}

// mode 0: p + q by a mixed addition (q affine), 1: by an XYZZ addition,
// 2: 2 p by XYZZ doubling; 3: as 1, and the sum's homogeneous projective
// form (X ZZZ, Y ZZ, ZZ ZZZ) in *proj
template <class A, class Proj> static void point_op(int mode, A *out, Proj *proj, const A *p, const A *q) {
  auto acc = from_affine(*p);
  if (mode == 0 && !q->infinity)
    xyzz_add_affine(acc, q->x, q->y);
  if (mode == 1 || mode == 3)
    xyzz_add(acc, from_affine(*q));
  if (mode == 2)
    xyzz_dbl(acc, acc);
  if (mode == 3)
    xyzz_to_projective(*proj, acc);
  to_affine(*out, acc);
}

extern "C" {

void zk_constants(uint64_t *p, uint64_t *r2, uint64_t *one, uint64_t *pinv, uint64_t *r) {
  for (int i = 0; i < NL; i++) p[i] = p_limb(i), r2[i] = r2_limb(i), one[i] = one_limb(i);
  for (int i = 0; i < 5; i++) r[i] = r_limb(i);
  *pinv = PINV;
}

// op: 0 add, 1 sub, 2 mul, 3 square, 4 negate, 5 invert, 6 to Montgomery, 7 from Montgomery
void zk_fp_op(int op, Fp *c, const Fp *a, const Fp *b) {
  switch (op) {
  case 0: fp_add(*c, *a, *b); break;
  case 1: fp_sub(*c, *a, *b); break;
  case 2: fp_mul(*c, *a, *b); break;
  case 3: fp_sqr(*c, *a); break;
  case 4: fp_neg(*c, *a); break;
  case 5: fp_inv(*c, *a); break;
  case 6: fp_to_montgomery(*c, *a); break;
  case 7: fp_from_montgomery(*c, *a); break;
  }
}

void zk_fp2_op(int op, Fp2 *c, const Fp2 *a, const Fp2 *b) {
  switch (op) {
  case 0: fp_add(*c, *a, *b); break;
  case 1: fp_sub(*c, *a, *b); break;
  case 2: fp_mul(*c, *a, *b); break;
  case 3: fp_sqr(*c, *a); break;
  case 4: fp_neg(*c, *a); break;
  case 5: fp_inv(*c, *a); break;
  }
}

void zk_g1_op(int mode, G1Point *out, G1ProjectivePoint *proj, const G1Point *p, const G1Point *q) {
  point_op(mode, out, proj, p, q);
}

void zk_g2_op(int mode, G2Point *out, G2ProjectivePoint *proj, const G2Point *p, const G2Point *q) {
  point_op(mode, out, proj, p, q);
}

bool zk_g1_on_curve_mont(const G1Point *p) { return on_curve_mont(p->x, p->y); }
bool zk_g2_on_curve_mont(const G2Point *p) { return on_curve_mont(p->x, p->y); }

// sizes and field offsets of the ABI structs as the header lays them out
void zk_struct_layout(uint64_t *out) {
  const uint64_t v[] = {sizeof(Fp), sizeof(Fp2), sizeof(Scalar), sizeof(G1Point), offsetof(G1Point, y),
                        offsetof(G1Point, infinity), sizeof(G2Point), offsetof(G2Point, y),
                        offsetof(G2Point, infinity), sizeof(G1ProjectivePoint), offsetof(G1ProjectivePoint, Z),
                        sizeof(G2ProjectivePoint), offsetof(G2ProjectivePoint, Z), alignof(G1Point)};
  std::memcpy(out, v, sizeof(v));
}

int zk_num_windows(int c) { return num_windows(c); }

void zk_signed_digits(int32_t *d, const uint64_t *k, int c) { signed_digits(d, k, c); }
}
