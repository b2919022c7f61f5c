// x2_shfl.cuh -- exchange 2 of the 16 x 4 x 16 transform through warp shuffles.
//
// Exchange 2 (pass-2 layout <-> pass-3 layout, negacyclic_fft.cuh) only moves
// data inside a warp.  Through shared memory it costs 16 STS.128 + 16 LDS.128
// per thread = 128 wavefronts per warp and direction, about a third of the
// shared-memory traffic of a CMUX step, plus a second 32 KiB exchange buffer
// per CTA.  With the pass-2 work assigned as  lane p + 8 m  <->  (sub-problem
// 8 w + p, quarter m)  (exchange-1 layout x1t_*), the exchange is a 4 x 4 block
// transpose between lanes p + 8 m (pass-2 side) and lanes 4 p + a (pass-3
// side), done register to register with SHFL: no shared memory, no barrier.
//
//   forward  (pass 2 -> pass 3):  v'[4 p + a][4 m + bl] = v[p + 8 m][4 bl + a]
//   inverse  (pass 3 -> pass 2):  v'[p + 8 m][4 bl + a] = v[4 p + a][4 m + bl]
//
// Each direction is four rounds of 16 shuffles (one complex = two doubles per
// block index).  In round r the reading lane picks the partner whose block
// index is its own XOR r, so every register index of a SHFL is a compile-time
// constant; the lane-dependent part is an XOR permutation of four values
// before the rounds (sender side) and after them (receiver side), two stages
// of conditional swaps each (selects, no local memory).
//
// The CPU emulator (tests/emu) replays the same rounds over a 32-lane model of
// the warp; the GPU tests (forward-transform golden through the C ABI,
// bit-identity against the shared-memory variant) pin it to the hardware.
#pragma once
#include "hd.cuh"

namespace b200 {

// x[i * S] <- x[(i ^ s) * S] for i = 0..3, s in 0..3 (two conditional-swap stages)
template <int S>
B200_HD void xor_perm4(cplx *x, int s) {
  if (s & 1) {
    cplx t = x[0];
    x[0] = x[S];
    x[S] = t;
    t = x[2 * S];
    x[2 * S] = x[3 * S];
    x[3 * S] = t;
  }
  if (s & 2) {
    cplx t = x[0];
    x[0] = x[2 * S];
    x[2 * S] = t;
    t = x[S];
    x[S] = x[3 * S];
    x[3 * S] = t;
  }
}

// forward: sender side, block bl sends v[4 bl + ((lane >> 3) ^ r)] in round r
B200_HD void x2s_fwd_pre(cplx v[16], int lane) {
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
    xor_perm4<1>(&v[4 * bl], lane >> 3);
}
B200_HD int x2s_fwd_src(int lane, int r) { return (lane >> 2) + 8 * ((lane & 3) ^ r); }
// forward: receiver side, y[4 r + bl] holds value 4 ((lane & 3) ^ r) + bl
B200_HD void x2s_fwd_post(cplx y[16], int lane) {
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
    xor_perm4<4>(&y[bl], lane & 3);
}
// inverse: sender side, round r sends block (lane & 3) ^ r
B200_HD void x2s_inv_pre(cplx v[16], int lane) {
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
    xor_perm4<4>(&v[bl], lane & 3);
}
B200_HD int x2s_inv_src(int lane, int r) { return 4 * (lane & 7) + ((lane >> 3) ^ r); }
// inverse: receiver side, y[4 r + bl] belongs to v[4 bl + ((lane >> 3) ^ r)]
B200_HD void x2s_inv_post(const cplx y[16], cplx v[16], int lane) {
#pragma unroll
  for (int bl = 0; bl < 4; bl++) {
    cplx z[4] = {y[bl], y[4 + bl], y[8 + bl], y[12 + bl]};
    xor_perm4<1>(z, lane >> 3);
#pragma unroll
    for (int c = 0; c < 4; c++)
      v[4 * bl + c] = z[c];
  }
}

// ---------------------------------------------------------------------------
// Half-warp variant (x2h_*) for the lane-pair layout of the N = 2048 kernel
// (x1h_* in negacyclic_fft.cuh): lanes 0-15 of a warp belong to polynomial 0,
// lanes 16-31 to polynomial 1, and each half holds 4 sub-problems.  Pass-2
// half-lane p + 4 m <-> (sub-problem 4 w + p, quarter m), pass-3 half-lane
// 4 p + a; the same 4 x 4 block transposes as above, inside each half:
//
//   forward  (pass 2 -> pass 3):  v'[4 p + a][4 m + bl] = v[p + 4 m][4 bl + a]
//   inverse  (pass 3 -> pass 2):  v'[p + 4 m][4 bl + a] = v[4 p + a][4 m + bl]
//
// The receiver side of the forward and the sender side of the inverse use
// lane & 3 as before (x2s_fwd_post / x2s_inv_pre); only the quarter index m
// and the partner lanes change.
// ---------------------------------------------------------------------------
B200_HD void x2h_fwd_pre(cplx v[16], int lane) {
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
    xor_perm4<1>(&v[4 * bl], (lane >> 2) & 3);
}
B200_HD int x2h_fwd_src(int lane, int r) {
  return (lane & 16) | (((lane >> 2) & 3) + 4 * ((lane & 3) ^ r));
}
B200_HD int x2h_inv_src(int lane, int r) {
  return (lane & 16) | (4 * (lane & 3) + (((lane >> 2) & 3) ^ r));
}
B200_HD void x2h_inv_post(const cplx y[16], cplx v[16], int lane) {
#pragma unroll
  for (int bl = 0; bl < 4; bl++) {
    cplx z[4] = {y[bl], y[4 + bl], y[8 + bl], y[12 + bl]};
    xor_perm4<1>(z, (lane >> 2) & 3);
#pragma unroll
    for (int c = 0; c < 4; c++)
      v[4 * bl + c] = z[c];
  }
}

#if defined(__CUDACC__)
__device__ __forceinline__ cplx shfl_cplx(cplx x, int src) {
  return cmake(__shfl_sync(0xffffffffu, x.re, src), __shfl_sync(0xffffffffu, x.im, src));
}
__device__ __forceinline__ cplx shfl_xor_cplx(cplx x, int mask) {
  return cmake(__shfl_xor_sync(0xffffffffu, x.re, mask),
               __shfl_xor_sync(0xffffffffu, x.im, mask));
}
__device__ __forceinline__ void x2h_fwd(cplx v[16]) {
  const int lane = threadIdx.x & 31;
  x2h_fwd_pre(v, lane);
  cplx y[16];
#pragma unroll
  for (int r = 0; r < 4; r++)
#pragma unroll
    for (int bl = 0; bl < 4; bl++)
      y[4 * r + bl] = shfl_cplx(v[4 * bl + r], x2h_fwd_src(lane, r));
  x2s_fwd_post(y, lane);
#pragma unroll
  for (int b = 0; b < 16; b++)
    v[b] = y[b];
}
__device__ __forceinline__ void x2h_inv(cplx v[16]) {
  const int lane = threadIdx.x & 31;
  x2s_inv_pre(v, lane);
  cplx y[16];
#pragma unroll
  for (int r = 0; r < 4; r++)
#pragma unroll
    for (int bl = 0; bl < 4; bl++)
      y[4 * r + bl] = shfl_cplx(v[4 * r + bl], x2h_inv_src(lane, r));
  x2h_inv_post(y, v, lane);
}
__device__ __forceinline__ void x2s_fwd(cplx v[16]) {
  const int lane = threadIdx.x & 31;
  x2s_fwd_pre(v, lane);
  cplx y[16];
#pragma unroll
  for (int r = 0; r < 4; r++)
#pragma unroll
    for (int bl = 0; bl < 4; bl++)
      y[4 * r + bl] = shfl_cplx(v[4 * bl + r], x2s_fwd_src(lane, r));
  x2s_fwd_post(y, lane);
#pragma unroll
  for (int b = 0; b < 16; b++)
    v[b] = y[b];
}
__device__ __forceinline__ void x2s_inv(cplx v[16]) {
  const int lane = threadIdx.x & 31;
  x2s_inv_pre(v, lane);
  cplx y[16];
#pragma unroll
  for (int r = 0; r < 4; r++)
#pragma unroll
    for (int bl = 0; bl < 4; bl++)
      y[4 * r + bl] = shfl_cplx(v[4 * r + bl], x2s_inv_src(lane, r));
  x2s_inv_post(y, v, lane);
}
#else
// host model of one warp: v[lane][16], the shuffles of a round read the
// senders' registers after every lane has run its sender-side permutation
static inline void x2s_fwd_warp(cplx (*v)[16]) {
  for (int lane = 0; lane < 32; lane++)
    x2s_fwd_pre(v[lane], lane);
  cplx y[32][16];
  for (int lane = 0; lane < 32; lane++)
    for (int r = 0; r < 4; r++)
      for (int bl = 0; bl < 4; bl++)
        y[lane][4 * r + bl] = v[x2s_fwd_src(lane, r)][4 * bl + r];
  for (int lane = 0; lane < 32; lane++) {
    x2s_fwd_post(y[lane], lane);
    for (int b = 0; b < 16; b++)
      v[lane][b] = y[lane][b];
  }
}
static inline void x2s_inv_warp(cplx (*v)[16]) {
  for (int lane = 0; lane < 32; lane++)
    x2s_inv_pre(v[lane], lane);
  cplx y[32][16];
  for (int lane = 0; lane < 32; lane++)
    for (int r = 0; r < 4; r++)
      for (int bl = 0; bl < 4; bl++)
        y[lane][4 * r + bl] = v[x2s_inv_src(lane, r)][4 * r + bl];
  for (int lane = 0; lane < 32; lane++)
    x2s_inv_post(y[lane], v[lane], lane);
}
static inline void x2h_fwd_warp(cplx (*v)[16]) {
  for (int lane = 0; lane < 32; lane++)
    x2h_fwd_pre(v[lane], lane);
  cplx y[32][16];
  for (int lane = 0; lane < 32; lane++)
    for (int r = 0; r < 4; r++)
      for (int bl = 0; bl < 4; bl++)
        y[lane][4 * r + bl] = v[x2h_fwd_src(lane, r)][4 * bl + r];
  for (int lane = 0; lane < 32; lane++) {
    x2s_fwd_post(y[lane], lane);
    for (int b = 0; b < 16; b++)
      v[lane][b] = y[lane][b];
  }
}
static inline void x2h_inv_warp(cplx (*v)[16]) {
  for (int lane = 0; lane < 32; lane++)
    x2s_inv_pre(v[lane], lane);
  cplx y[32][16];
  for (int lane = 0; lane < 32; lane++)
    for (int r = 0; r < 4; r++)
      for (int bl = 0; bl < 4; bl++)
        y[lane][4 * r + bl] = v[x2h_inv_src(lane, r)][4 * r + bl];
  for (int lane = 0; lane < 32; lane++)
    x2h_inv_post(y[lane], v[lane], lane);
}
#endif

} // namespace b200
