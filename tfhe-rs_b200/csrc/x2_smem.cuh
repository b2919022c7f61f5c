// x2_smem.cuh -- exchange 2 of the lane-pair layout through the calling warp's
// own rows of the exchange-1 buffer.
//
// In the lane-pair layout (x1h_* in negacyclic_fft.cuh, x2h_* in x2_shfl.cuh)
// warp w's pass-2 accesses stay in rows 4 w .. 4 w + 3 of each xa[g] buffer:
// from the forward x1h_load_p2 to the inverse x1h_store_p2 those 256 complex
// slots per polynomial belong to warp w alone, and both exchange-2 transposes
// of a CMUX step fall inside that window.  So exchange 2 can go through them:
// 16 STS.128 + 16 LDS.128 per thread and direction, ordered by __syncwarp(),
// with no shuffles, no lane-dependent selects and no y[16] temporaries.  The
// register contents it leaves are exactly those of x2h_fwd / x2h_inv:
//
//   forward  (pass 2 -> pass 3):  v'[4 p + a][4 m + bl] = v[p + 4 m][4 bl + a]
//   inverse  (pass 3 -> pass 2):  v'[p + 4 m][4 bl + a] = v[4 p + a][4 m + bl]
//
// (half-lane indices i = lane & 15; each half-warp uses its own buffer xa[g]).
//
// Slot of element (pass-3 half-lane i3 = 4 p + a, register b = 4 m + bl)
// inside the warp's 256-slot region:
//
//   x2m_slot = 64 bl + 32 (m >> 1) + 8 a + ((4 (m & 1) + p) ^ 2 a)
//
// The 16-byte bank group is slot & 7 = (p0, p1 ^ a0, m0 ^ a1).  A pass-2
// quarter-warp (fixed a, bl; p = 0..3, m & 1 = 0..1) and a pass-3 quarter-warp
// (fixed m, bl; a = 0..3, p & 1 = 0..1) both cover all 8 groups, so every
// STS.128 / LDS.128 of both directions is conflict-free
// (emu_x2m_conflict_audit).  The compile-time register index enters the slot
// additively except through a (pass-2 side, 4 lane bases) and m & 1 (pass-3
// side, 2 lane bases): every access is one base register plus an immediate.
#pragma once
#include "hd.cuh"

namespace b200 {

B200_HD int x2m_slot(int i3, int b) {
  const int p = i3 >> 2, a = i3 & 3, m = b >> 2, bl = b & 3;
  return 64 * bl + 32 * (m >> 1) + 8 * a + ((4 * (m & 1) + p) ^ (2 * a));
}

// pass-2 side: half-lane i = p + 4 m holds v[4 bl + a] = element (4 p + a, 4 m + bl)
B200_HD void x2m_store_p2(cplx *rows, int i, const cplx v[16]) {
  const int p = i & 3, m = i >> 2;
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
#pragma unroll
    for (int a = 0; a < 4; a++)
      rows[x2m_slot(4 * p + a, 4 * m + bl)] = v[4 * bl + a];
}
B200_HD void x2m_load_p2(const cplx *rows, int i, cplx v[16]) {
  const int p = i & 3, m = i >> 2;
#pragma unroll
  for (int bl = 0; bl < 4; bl++)
#pragma unroll
    for (int a = 0; a < 4; a++)
      v[4 * bl + a] = rows[x2m_slot(4 * p + a, 4 * m + bl)];
}
// pass-3 side: half-lane i holds v[b] = element (i, b)
B200_HD void x2m_store_p3(cplx *rows, int i, const cplx v[16]) {
#pragma unroll
  for (int b = 0; b < 16; b++)
    rows[x2m_slot(i, b)] = v[b];
}
B200_HD void x2m_load_p3(const cplx *rows, int i, cplx v[16]) {
#pragma unroll
  for (int b = 0; b < 16; b++)
    v[b] = rows[x2m_slot(i, b)];
}

#if defined(__CUDACC__)
// `rows` = xa[g] + 256 w: the calling warp's rows of its half-warp's buffer.
// The first __syncwarp orders the stores after the other lanes' earlier reads
// of the same slots (x1h_load_p2, or the forward exchange's loads), the
// second the loads after the stores.
__device__ __forceinline__ void x2m_fwd(cplx *rows, cplx v[16]) {
  const int i = threadIdx.x & 15;
  __syncwarp();
  x2m_store_p2(rows, i, v);
  __syncwarp();
  x2m_load_p3(rows, i, v);
}
__device__ __forceinline__ void x2m_inv(cplx *rows, cplx v[16]) {
  const int i = threadIdx.x & 15;
  __syncwarp();
  x2m_store_p3(rows, i, v);
  __syncwarp();
  x2m_load_p2(rows, i, v);
}
#else
// host model of one warp: v[lane][16]; lanes 0-15 use buffer 0, 16-31 buffer 1
static inline void x2m_fwd_warp(cplx (*v)[16]) {
  cplx rows[2][256];
  for (int lane = 0; lane < 32; lane++)
    x2m_store_p2(rows[lane >> 4], lane & 15, v[lane]);
  for (int lane = 0; lane < 32; lane++)
    x2m_load_p3(rows[lane >> 4], lane & 15, v[lane]);
}
static inline void x2m_inv_warp(cplx (*v)[16]) {
  cplx rows[2][256];
  for (int lane = 0; lane < 32; lane++)
    x2m_store_p3(rows[lane >> 4], lane & 15, v[lane]);
  for (int lane = 0; lane < 32; lane++)
    x2m_load_p2(rows[lane >> 4], lane & 15, v[lane]);
}
#endif

} // namespace b200
