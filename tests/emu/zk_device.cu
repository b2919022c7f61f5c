// sm_90a build of tfhe-rs_b200/csrc/bls12_446.cuh's device path (the PTX
// carry chains on 14 x u32 limbs that the MSM kernels inline), exported for
// tests/test_zk_device_arith.py.  Each function runs one batch: it allocates,
// copies in, makes one launch, copies out, frees and returns the first
// cudaError_t.  Field elements are in Montgomery form except the input of
// "to Montgomery" and the output of "from Montgomery".  Points are raw XYZZ
// (X, Y, ZZ, ZZZ), so a test sees ZZ and ZZZ as the device left them.
#include "../../tfhe-rs_b200/csrc/bls12_446.cuh"

#include <cuda_runtime.h>

using namespace zk;

namespace {

constexpr int T = 128;

// op: 0 add, 1 sub, 2 mul, 3 square, 4 negate, 6 to Montgomery, 7 from
// Montgomery (the codes of zk_host.cpp's zk_fp_op; 5, invert, is host-only)
template <class F> __device__ void field_op(int op, F &c, const F &a, const F &b) {
  switch (op) {
  case 0: fp_add(c, a, b); break;
  case 1: fp_sub(c, a, b); break;
  case 2: fp_mul(c, a, b); break;
  case 3: fp_sqr(c, a); break;
  case 4: fp_neg(c, a); break;
  case 6: fp_to_montgomery(c, a); break;
  case 7: fp_from_montgomery(c, a); break;
  }
}

template <class F> __global__ void __launch_bounds__(T) field_kernel(int op, uint32_t n, F *c, const F *a, const F *b) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    field_op(op, c[i], a[i], b[i]);
}

// mode 0: p + (q.X, q.Y) by a mixed addition (q must be affine, ZZ = ZZZ = 1,
// and not the identity), 1: p + q by an XYZZ addition, 2: 2 p by XYZZ
// doubling, 3: p's homogeneous projective form (X ZZZ, Y ZZ, ZZ ZZZ) in
// (X, Y, ZZ), ZZZ zeroed
template <class F> __global__ void __launch_bounds__(T)
    point_kernel(int mode, uint32_t n, Xyzz<F> *out, const Xyzz<F> *p, const Xyzz<F> *q) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  Xyzz<F> acc = p[i];
  if (mode == 0) {
    xyzz_add_affine(acc, q[i].X, q[i].Y);
  } else if (mode == 1) {
    xyzz_add(acc, q[i]);
  } else if (mode == 2) {
    xyzz_dbl(acc, acc);
  } else {
    struct {
      F X, Y, Z;
    } r;
    xyzz_to_projective(r, p[i]);
    acc.X = r.X, acc.Y = r.Y, acc.ZZ = r.Z;
    fp_zero(acc.ZZZ);
  }
  out[i] = acc;
}

__global__ void __launch_bounds__(T) digits_kernel(uint32_t n, int32_t *out, const Scalar *k, int c) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  int32_t d[SCALAR_BITS / 4 + 1];
  uint64_t s[5];
  for (int j = 0; j < 5; j++) s[j] = k[i].limb[j];
  signed_digits(d, s, c);
  const int W = num_windows(c);
  for (int w = 0; w < W; w++) out[(size_t)i * W + w] = d[w];
}

// device copies of `ins`, one launch of `run` on them and an output buffer of
// out_bytes, the output copied back; the first error wins
template <class Run>
cudaError_t batch(void *out, size_t out_bytes, const void *a, size_t a_bytes, const void *b, size_t b_bytes,
                  Run run) {
  void *d_out = nullptr, *d_a = nullptr, *d_b = nullptr;
  cudaError_t e = cudaMalloc(&d_out, out_bytes);
  if (e == cudaSuccess)
    e = cudaMalloc(&d_a, a_bytes);
  if (e == cudaSuccess && b_bytes)
    e = cudaMalloc(&d_b, b_bytes);
  if (e == cudaSuccess)
    e = cudaMemcpy(d_a, a, a_bytes, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && b_bytes)
    e = cudaMemcpy(d_b, b, b_bytes, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    run(d_out, d_a, d_b);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess)
    e = cudaMemcpy(out, d_out, out_bytes, cudaMemcpyDeviceToHost);
  cudaFree(d_out);
  cudaFree(d_a);
  cudaFree(d_b);
  return e;
}

unsigned blocks(uint32_t n) { return (n + T - 1) / T; }

template <class F> cudaError_t field_batch(int op, uint32_t n, F *out, const F *a, const F *b, int max_op) {
  if (op < 0 || op > max_op || op == 5 || n == 0)
    return cudaErrorInvalidValue;
  const size_t bytes = (size_t)n * sizeof(F);
  return batch(out, bytes, a, bytes, b, bytes, [&](void *o, void *x, void *y) {
    field_kernel<F><<<blocks(n), T>>>(op, n, (F *)o, (const F *)x, (const F *)y);
  });
}

template <class F>
cudaError_t point_batch(int mode, uint32_t n, Xyzz<F> *out, const Xyzz<F> *p, const Xyzz<F> *q) {
  if (mode < 0 || mode > 3 || n == 0)
    return cudaErrorInvalidValue;
  const size_t bytes = (size_t)n * sizeof(Xyzz<F>);
  return batch(out, bytes, p, bytes, q, bytes, [&](void *o, void *x, void *y) {
    point_kernel<F><<<blocks(n), T>>>(mode, n, (Xyzz<F> *)o, (const Xyzz<F> *)x, (const Xyzz<F> *)y);
  });
}

}  // namespace

extern "C" {

// n elements of 7 x u64 (Fp) or 2 x 7 x u64 (Fp2) each; b is read for every
// op (pass a copy of a for the unary ones)
int zk_dev_fp_op(int op, uint32_t n, Fp *out, const Fp *a, const Fp *b) { return field_batch(op, n, out, a, b, 7); }
int zk_dev_fp2_op(int op, uint32_t n, Fp2 *out, const Fp2 *a, const Fp2 *b) {
  return field_batch(op, n, out, a, b, 4);
}

// n XYZZ points (4 x Fp, or 4 x Fp2) each; see point_kernel for the modes
int zk_dev_g1_op(int mode, uint32_t n, Xyzz<Fp> *out, const Xyzz<Fp> *p, const Xyzz<Fp> *q) {
  return point_batch(mode, n, out, p, q);
}
int zk_dev_g2_op(int mode, uint32_t n, Xyzz<Fp2> *out, const Xyzz<Fp2> *p, const Xyzz<Fp2> *q) {
  return point_batch(mode, n, out, p, q);
}

// num_windows(c) signed digits of each of n scalars, row by row
int zk_dev_signed_digits(uint32_t n, int32_t *out, const Scalar *scalars, int c) {
  if (c < 4 || c > 16 || n == 0)
    return cudaErrorInvalidValue;
  const int W = num_windows(c);
  return batch(out, (size_t)n * W * sizeof(int32_t), scalars, (size_t)n * sizeof(Scalar), nullptr, 0,
               [&](void *o, void *x, void *) { digits_kernel<<<blocks(n), T>>>(n, (int32_t *)o, (const Scalar *)x, c); });
}
}
