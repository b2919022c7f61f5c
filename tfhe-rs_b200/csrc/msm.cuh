// msm.cuh -- Pippenger multi-scalar multiplication sum k_i P_i over BLS12-446
// G1 and G2 (one template over the affine point type, G1Point or G2Point).
//
// Phases, one kernel each (the host side is b200::msm_run in b200_backend.cu):
//  1. msm_digits_kernel: signed c-bit window digits of every scalar, as
//     (key = window * B + |digit| - 1, value = point index | sign) pairs;
//     a zero digit gets the key nb = W * B, which sorts past every bucket.
//  2. cub::DeviceRadixSort of the pairs by key, so every bucket is one run.
//  3. msm_bucket_bounds_kernel / msm_task_count_kernel / cub scan /
//     msm_accumulate_kernel / msm_bucket_tree_kernel: each bucket's run is
//     cut into tasks of at most `task` points; one thread sums a task with
//     mixed additions, and the tasks of a bucket are then added pairwise in
//     log2(n / task) tree passes.  A bucket holding all n points (every scalar
//     equal) is n / task parallel tasks, not one thread walking n points.
//  4. msm_bucket_reduce_kernel: running sums over segments of L buckets; a
//     segment yields sum_j (j + 1) B_j over its buckets and its plain sum.
//  5. msm_window_sum_kernel: per window, the segment totals plus s L times
//     each segment's plain sum, added in a shared-memory tree.
//     The Horner step over windows (about 320 dependent doublings) runs on
//     the host: see DESIGN section 8k.
#pragma once
#include <cstdint>

#include "bls12_446.cuh"

namespace b200 {

constexpr uint32_t MSM_NEG = 0x80000000u;  // value bit: the digit is negative

template <class A> using MsmField = decltype(A::x);

// managed path with points in normal form: to Montgomery form in place
template <class A> __global__ void __launch_bounds__(128) msm_to_montgomery_kernel(A *pts, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || pts[i].infinity)
    return;
  zk::fp_to_montgomery(pts[i].x, pts[i].x);
  zk::fp_to_montgomery(pts[i].y, pts[i].y);
}

// 1. window digits; pair (w, i) at w * n + i
__global__ void __launch_bounds__(128) msm_digits_kernel(const Scalar *scalars, uint32_t n, int c,
                                                         uint32_t *keys, uint32_t *vals) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const int W = zk::num_windows(c);
  const uint32_t B = 1u << (c - 1), nb = (uint32_t)W * B;
  int32_t d[zk::SCALAR_BITS / 4 + 1];
  uint64_t k[5];
#pragma unroll
  for (int j = 0; j < 5; j++) k[j] = scalars[i].limb[j];
  zk::signed_digits(d, k, c);
  for (int w = 0; w < W; w++) {
    uint32_t key = nb, val = i;
    if (d[w] != 0) {
      key = (uint32_t)w * B + (uint32_t)(d[w] < 0 ? -d[w] : d[w]) - 1;
      val |= d[w] < 0 ? MSM_NEG : 0;
    }
    keys[(size_t)w * n + i] = key;
    vals[(size_t)w * n + i] = val;
  }
}

// 3a. [start, end) of every non-empty bucket in the sorted keys (start and
// end are zeroed by the caller)
__global__ void msm_bucket_bounds_kernel(const uint32_t *keys, uint32_t count, uint32_t nb, uint32_t *start,
                                         uint32_t *end) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= count)
    return;
  const uint32_t key = keys[j];
  if (key >= nb)
    return;
  if (j == 0 || keys[j - 1] != key)
    start[key] = j;
  if (j + 1 == count || keys[j + 1] != key)
    end[key] = j + 1;
}

// 3b. tasks per bucket, ceil(size / task); entry nb is 0 so the exclusive
// scan's last entry is the task total
__global__ void msm_task_count_kernel(const uint32_t *start, const uint32_t *end, uint32_t nb, uint32_t task,
                                      uint32_t *ntasks) {
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > nb)
    return;
  ntasks[b] = b == nb ? 0 : (end[b] - start[b] + task - 1) / task;
}

// the bucket whose task range [toff[b], toff[b + 1]) holds task t
__device__ __forceinline__ uint32_t msm_task_bucket(const uint32_t *toff, uint32_t nb, uint32_t t) {
  uint32_t lo = 0, hi = nb;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (toff[mid + 1] <= t)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}

// 3c. one thread sums one task's points (mixed additions, negated for a
// negative digit; points flagged infinity are skipped)
template <class A>
__global__ void __launch_bounds__(128)
    msm_accumulate_kernel(const A *pts, const uint32_t *vals, const uint32_t *start, const uint32_t *end,
                          const uint32_t *toff, uint32_t nb, uint32_t task, uint32_t max_tasks,
                          zk::Xyzz<MsmField<A>> *partial, uint32_t *task_bucket) {
  using F = MsmField<A>;
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= max_tasks || t >= toff[nb])
    return;
  const uint32_t b = msm_task_bucket(toff, nb, t);
  const uint32_t first = start[b] + (t - toff[b]) * task;
  const uint32_t last = min(first + task, end[b]);
  zk::Xyzz<F> acc;
  zk::xyzz_set_identity(acc);
  for (uint32_t j = first; j < last; j++) {
    const uint32_t v = vals[j];
    const A &p = pts[v & ~MSM_NEG];
    if (p.infinity)
      continue;
    F y = p.y;
    if (v & MSM_NEG)
      zk::fp_neg(y, y);
    zk::xyzz_add_affine(acc, p.x, y);
  }
  partial[t] = acc;
  task_bucket[t] = b;
}

// 3d. one tree pass: task k of a bucket adds in task k + step when k is a
// multiple of 2 step; after the passes a bucket's sum is its first task's
template <class F>
__global__ void __launch_bounds__(128)
    msm_bucket_tree_kernel(zk::Xyzz<F> *partial, const uint32_t *task_bucket, const uint32_t *toff, uint32_t nb,
                           uint32_t max_tasks, uint32_t step) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= max_tasks || t >= toff[nb])
    return;
  const uint32_t b = task_bucket[t];
  const uint32_t k = t - toff[b], count = toff[b + 1] - toff[b];
  if (k % (2 * step) != 0 || k + step >= count)
    return;
  zk::Xyzz<F> acc = partial[t];
  zk::xyzz_add(acc, partial[t + step]);
  partial[t] = acc;
}

// 4. segment s of window w covers buckets [s L, (s + 1) L): from the top,
// running += B_j and total += running, so total = sum_j (j - s L + 1) B_j
template <class F>
__global__ void __launch_bounds__(128)
    msm_bucket_reduce_kernel(const zk::Xyzz<F> *partial, const uint32_t *toff, uint32_t W, uint32_t B,
                             uint32_t L, zk::Xyzz<F> *seg_total, zk::Xyzz<F> *seg_run) {
  const uint32_t S = B / L, g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= W * S)
    return;
  const uint32_t w = g / S, s = g % S;
  zk::Xyzz<F> run, total;
  zk::xyzz_set_identity(run);
  zk::xyzz_set_identity(total);
  for (int j = (int)L - 1; j >= 0; j--) {
    const uint32_t b = w * B + s * L + (uint32_t)j;
    if (toff[b + 1] != toff[b])
      zk::xyzz_add(run, partial[toff[b]]);
    zk::xyzz_add(total, run);
  }
  seg_total[g] = total;
  seg_run[g] = run;
}

// 5a. window w's sum, one block of S threads per window: thread s forms
// total_s + (s L) run_s by double-and-add (at most c - 1 doublings), then a
// shared-memory tree adds the S terms.  A single thread walking the suffix
// sums instead would chain about 3 S dependent additions.
constexpr uint32_t MSM_MAX_SEGMENTS = 64;
template <class F>
__global__ void __launch_bounds__(MSM_MAX_SEGMENTS)
    msm_window_sum_kernel(const zk::Xyzz<F> *seg_total, const zk::Xyzz<F> *seg_run, uint32_t S, uint32_t L,
                          zk::Xyzz<F> *win) {
  __shared__ zk::Xyzz<F> terms[MSM_MAX_SEGMENTS];
  const uint32_t w = blockIdx.x, s = threadIdx.x;
  const uint32_t m = s * L;
  zk::Xyzz<F> acc;
  zk::xyzz_set_identity(acc);
  const zk::Xyzz<F> run = seg_run[w * S + s];
  for (int bit = 31 - __clz(m | 1); m != 0 && bit >= 0; bit--) {
    zk::xyzz_dbl(acc, acc);
    if ((m >> bit) & 1)
      zk::xyzz_add(acc, run);
  }
  zk::xyzz_add(acc, seg_total[w * S + s]);
  terms[s] = acc;
  __syncthreads();
  for (uint32_t half = S / 2; half > 0; half /= 2) {
    if (s < half) {
      acc = terms[s];
      zk::xyzz_add(acc, terms[s + half]);
      terms[s] = acc;
    }
    __syncthreads();
  }
  if (s == 0)
    win[w] = terms[0];
}

}  // namespace b200
