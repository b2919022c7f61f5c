/* tfhe_b200_zk.h -- the C ABI of zk-cuda-backend (BLS12-446 multi-scalar
 * multiplication for tfhe-zk-pok's PKE v2 proofs), exported by
 * libtfhe_cuda_backend_b200.so.
 *
 * The 25 functions and the struct layouts are those of
 * backends/zk-cuda-backend/src/bindings.rs, so that crate links against this
 * library unchanged.  Field elements are 7 x u64 little-endian limbs; a
 * Scalar is 5 x u64 (any 320-bit value is accepted).  The MSM entry points
 * take affine points in Montgomery form (R = 2^448) and return a homogeneous
 * projective point in Montgomery form, the identity with Z = 0; both return
 * with the result written to host memory.  The b200_ functions at the end
 * are this engine's additions (introspection of the calling thread's last
 * MSM). */
#ifndef TFHE_B200_ZK_H
#define TFHE_B200_ZK_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st *cudaStream_t;

typedef struct Fp {
  uint64_t limb[7];
} Fp;

typedef struct Fp2 {
  Fp c0;
  Fp c1;
} Fp2;

typedef struct BigInt {
  uint64_t limb[5];
} BigInt;
typedef BigInt Scalar;

typedef struct G1Point {
  Fp x;
  Fp y;
  bool infinity;
} G1Point;

typedef struct G2Point {
  Fp2 x;
  Fp2 y;
  bool infinity;
} G2Point;

typedef struct G1ProjectivePoint {
  Fp X;
  Fp Y;
  Fp Z;
} G1ProjectivePoint;

typedef struct G2ProjectivePoint {
  Fp2 X;
  Fp2 Y;
  Fp2 Z;
} G2ProjectivePoint;

/* host helpers: coordinates in Montgomery form unless stated */
void affine_to_projective_g1_wrapper(G1ProjectivePoint *proj, const G1Point *affine);
void affine_to_projective_g2_wrapper(G2ProjectivePoint *proj, const G2Point *affine);
void projective_to_affine_g1_wrapper(G1Point *affine, const G1ProjectivePoint *proj);
void projective_to_affine_g2_wrapper(G2Point *affine, const G2ProjectivePoint *proj);
void g1_point_at_infinity_wrapper(G1Point *point);
void g2_point_at_infinity_wrapper(G2Point *point);
void g1_projective_point_at_infinity_wrapper(G1ProjectivePoint *point);
void g2_projective_point_at_infinity_wrapper(G2ProjectivePoint *point);
bool g1_is_infinity_wrapper(const G1Point *point);
bool g2_is_infinity_wrapper(const G2Point *point);

/* device arrays, caller scratch of pippenger_scratch_size_g{1,2}_wrapper(n)
 * bytes, points in Montgomery form; returns after *h_result is written */
void g1_msm_unmanaged_wrapper_async(cudaStream_t stream, uint32_t gpu_index, G1ProjectivePoint *h_result,
                                    const G1Point *d_points, const Scalar *d_scalars, uint32_t n,
                                    G1ProjectivePoint *d_scratch);
void g2_msm_unmanaged_wrapper_async(cudaStream_t stream, uint32_t gpu_index, G2ProjectivePoint *h_result,
                                    const G2Point *d_points, const Scalar *d_scalars, uint32_t n,
                                    G2ProjectivePoint *d_scratch);
size_t pippenger_scratch_size_g1_wrapper(uint32_t n, uint32_t gpu_index);
size_t pippenger_scratch_size_g2_wrapper(uint32_t n, uint32_t gpu_index);

/* host arrays; device memory from the stream-ordered pool, counted in
 * *size_tracker; synchronizes `stream` */
void g1_msm_managed_wrapper(cudaStream_t stream, uint32_t gpu_index, G1ProjectivePoint *result,
                            const G1Point *points, const Scalar *scalars, uint32_t n, bool points_in_montgomery,
                            uint64_t *size_tracker);
void g2_msm_managed_wrapper(cudaStream_t stream, uint32_t gpu_index, G2ProjectivePoint *result,
                            const G2Point *points, const Scalar *scalars, uint32_t n, bool points_in_montgomery,
                            uint64_t *size_tracker);

/* Montgomery form -> normal form */
void g1_from_montgomery_wrapper(G1Point *result, const G1Point *point);
void g2_from_montgomery_wrapper(G2Point *result, const G2Point *point);
void fp_to_montgomery_wrapper(Fp *result, const Fp *value);
void fp_from_montgomery_wrapper(Fp *result, const Fp *value);
/* Montgomery projective -> normal-form (X/Z, Y/Z, 1); Z = 0 stays 0 */
void g1_projective_from_montgomery_normalized_wrapper(G1ProjectivePoint *result, const G1ProjectivePoint *point);
void g2_projective_from_montgomery_normalized_wrapper(G2ProjectivePoint *result, const G2ProjectivePoint *point);
/* normal-form coordinates */
bool is_on_curve_g1_wrapper(const G1Point *point);
bool is_on_curve_g2_wrapper(const G2Point *point);
/* the group order r, 5 x u64 */
void scalar_modulus_limbs_wrapper(uint64_t *limbs);

/* additions: the calling thread's last MSM -- its window size, window count,
 * points per accumulation task, segments per window and kernel names
 * ("c=.. windows=.. task=.. segments=.. kernels=a,b,..") and the host time of
 * its window combination in microseconds */
const char *b200_last_msm_config(void);
double b200_last_msm_combine_us(void);

#ifdef __cplusplus
}
#endif

#endif
