// pbs_n2048.cuh -- sm_90a classic PBS kernel for (N = 2048, k = 1, l = 1),
// i.e. PARAM_MESSAGE_2_CARRY_2_KS_PBS and friends (any n, any base_log <= 31).
//
// Replaces, on the reference side,
//   host_programmable_bootstrap / device_programmable_bootstrap_* kernels
//   (backends/tfhe-cuda-backend/cuda/src/pbs/programmable_bootstrap_classic.cuh)
// and restates the CPU path
//   FourierLweBootstrapKeyView::bootstrap (fft64/crypto/bootstrap.rs:480-520).
//
// Design (v1): one persistent CTA per LWE, 128 threads, 2 CTAs per SM.
//   * GLWE accumulator (2 x 2048 u64) lives in shared memory for the whole
//     918-step blind rotation; nothing but the final LWE goes back to HBM.
//   * each 64-thread group runs a register-resident 1024-point twist-free
//     negacyclic transform (16 x 4 x 16) with two swizzled smem exchanges;
//     pass-2/3 twiddles are loop invariant and stay in registers.
//   * the Fourier BSK is read with 128-bit L2-only loads (ld.global.cg), one
//     32 KiB contiguous block per (GGSW, column) per step, pre-permuted at
//     key-conversion time so that lane t reads element t.
#pragma once
#include "pbs_n2048_lanepair.cuh"
#include "pbs_n2048_phases.cuh"
#include "tma_bulk.cuh"
#include "x2_shfl.cuh"
#include "x2_smem.cuh"

#include <cuda_runtime.h>

namespace b200 {

// pass-1 twiddles (levels 1-4) are the same for every thread: constant bank,
// so after unrolling they are immediate c[bank][offset] operands of the DFMAs.
// Filled once per device by device_tables().
__constant__ cplx c_fft1024_pass1[15];

struct P22Smem {
  uint64_t acc[2][P22_N];       // 32 KiB
  cplx xa[2][P22_M];            // 32 KiB  exchange 1 / spectrum share
  cplx xb[2][P22_M];            // 32 KiB  exchange 2
  uint16_t a_hat[1024 + 8];     // switched mask (n <= 1024 for this kernel)
  uint32_t b_hat;
  unsigned long long red_half[4];
  long long red_dbl[4];
};

__device__ __forceinline__ void group_barrier(int g) {
  // named barrier 1+g over the 64 threads of the group
  asm volatile("bar.sync %0, 64;" ::"r"(g + 1) : "memory");
}

// Exchange 2 (pass-2 <-> pass-3 layout, x2_* in negacyclic_fft.cuh) only moves
// data between the 4 adjacent lanes 4q..4q+3 that share a sub-problem q: a
// warp-level barrier orders it (round 1 used the 64-thread named barrier and
// made each warp wait for its partner warp twice per transform pair).
// B200_X2_GROUP_BARRIER restores the named barrier for A/B builds.
__device__ __forceinline__ void x2_sync(int g) {
#ifdef B200_X2_GROUP_BARRIER
  group_barrier(g);
#else
  (void)g;
  __syncwarp();
#endif
}

// The spectrum store of a step overwrites the exchange-1 buffer of the group
// (xa_g, all 1024 slots) while the group's OTHER warp may, in principle, still
// be reading its exchange-1 values out of it: with exchange 2 warp-local (in
// shared memory or through shuffles) nothing else orders the two.  A split barrier does, at no
// cost: each warp signals "my exchange-1 loads are done" right after them
// (bar.arrive, non-blocking) and waits for the partner's signal just before the
// spectrum store (bar.sync on the partner's barrier; 1,500 cycles later it has
// long completed).  Barriers 3 + 2g + w: 32 arrivals + 32 waiters = 64.
__device__ __forceinline__ void spec_guard_arrive(int g, int t) {
  asm volatile("bar.arrive %0, 64;" ::"r"(3 + 2 * g + (t >> 5)) : "memory");
}
__device__ __forceinline__ void spec_guard_wait(int g, int t) {
  asm volatile("bar.sync %0, 64;" ::"r"(3 + 2 * g + (1 - (t >> 5))) : "memory");
}

// Split replacement of the CTA barrier that followed the MAC.  What that barrier
// protected: (a) xa_g, read by the OTHER group as `xa_other` during its MAC, is
// next written by group g in the inverse exchange 1, ~1,000 cycles later;
// (b) the key ring, next written by the TMA copy of the following step.  So the
// other group signals "my MAC is done" (bar.arrive, non-blocking) and group g
// waits for that signal only just before its inverse exchange-1 store; thread 0
// issues the next copy after the group barrier of that exchange (every thread of
// its own group is then past its MAC and has seen the other group's signal).
// The two groups of a CTA no longer meet after the MAC.  Barriers 7 + g: 64
// arrivals (group 1 - g) + 64 waiters (group g) = 128.
__device__ __forceinline__ void mac_done_arrive(int g) {
  asm volatile("bar.arrive %0, 128;" ::"r"(7 + (1 - g)) : "memory");
}
__device__ __forceinline__ void mac_done_wait(int g) {
  asm volatile("bar.sync %0, 128;" ::"r"(7 + g) : "memory");
}
// The same split for the barrier BEFORE the MAC (SPLIT = 2): a group signals "my
// spectrum is stored" and only waits for the other group's signal after its
// own-row products, which need nothing from the other group.  Barriers 9 + g.
__device__ __forceinline__ void spec_ready_arrive(int g) {
  asm volatile("bar.arrive %0, 128;" ::"r"(9 + (1 - g)) : "memory");
}
__device__ __forceinline__ void spec_ready_wait(int g) {
  asm volatile("bar.sync %0, 128;" ::"r"(9 + g) : "memory");
}

struct LdcgLoader {
  __device__ __forceinline__ cplx operator()(const cplx *p) const {
    return ldcg_cplx(p);
  }
};

// grid = num_samples, block = 128, dynamic smem = sizeof(P22Smem)
__global__ void __launch_bounds__(128, 2)
pbs_n2048_k1_l1_kernel(uint64_t *__restrict__ lwe_out,
                       const uint64_t *__restrict__ out_idx,
                       const uint64_t *__restrict__ luts,
                       const uint64_t *__restrict__ lut_idx,
                       const uint64_t *__restrict__ lwe_in,
                       const uint64_t *__restrict__ in_idx,
                       const cplx *__restrict__ bsk,
                       const Fft1024Tables *__restrict__ tables, uint32_t n,
                       uint32_t base_log, uint32_t num_many_lut,
                       uint32_t lut_stride, int centered_ms) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  P22Smem &sm = *reinterpret_cast<P22Smem *>(smem_raw);
  const int tid = threadIdx.x;
  const int g = tid >> 6;       // group = polynomial / output column
  const int t = tid & 63;       // thread inside the group
  const uint32_t s = blockIdx.x;
  const uint32_t log_mod = 12;  // log2(2N)

  // ---- prologue: modulus switch (a4/a5), acc = LUT * X^{-b_hat} -----------
  const uint64_t *ct = lwe_in + in_idx[s] * (uint64_t)(n + 1);
  CenteredMsSums sums;
  for (uint32_t i = tid; i < n; i += 128) {
    const uint64_t a = ct[i];
    sm.a_hat[i] = (uint16_t)modulus_switch_u64(a, log_mod);
    if (centered_ms)
      sums.add(a, log_mod);
  }
  if (centered_ms)
    centered_ms_publish_warp(sums, sm.red_half, sm.red_dbl);
  __syncthreads();
  if (tid == 0)
    sm.b_hat = ms_b_hat(ct[n], centered_ms, sm.red_half, sm.red_dbl, 4, log_mod);
  __syncthreads();
  rotate_lut(&sm.acc[0][0], P22_N, luts + lut_idx[s] * (uint64_t)(2 * P22_N), 2,
             P22_N, sm.b_hat, tid, 128, SameWord());

  // loop-invariant twiddles -> registers
  cplx tw2[3], tw3[15];
  {
#pragma unroll
    for (int e = 0; e < 3; e++)
      tw2[e] = tables->pass2[t >> 2][e];
#pragma unroll
    for (int e = 0; e < 15; e++)
      tw3[e] = tables->pass3[t][e];
  }
  __syncthreads();

  uint64_t *acc_g = sm.acc[g];
  cplx *xa_g = sm.xa[g];
  cplx *xb_g = sm.xb[g];
  const cplx *xa_other = sm.xa[1 - g];

  // ---- blind rotation: n CMUX steps (a14) -----------------------------
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t a = sm.a_hat[i];
    if (a == 0)
      continue; // uniform across the CTA
    cplx v[16];
    p22_load_digits(acc_g, t, a, base_log, v);
    radix16_fwd(v, c_fft1024_pass1);
    x1_store_p1(xa_g, t, v);
    group_barrier(g);
    x1_load_p2(xa_g, t, v);
    pass2_fwd(v, tw2);
    x2_store_p2(xb_g, t, v);
    x2_sync(g);
    x2_load_p3(xb_g, t, v);
    radix16_fwd(v, tw3);
    spec_store(xa_g, t, v);
    __syncthreads();
    p22_mac(v, xa_other, bsk + ((size_t)i * 2 + g) * (2 * P22_M), t, g,
            LdcgLoader());
    __syncthreads();
    radix16_inv(v, tw3);
    x2_store_p3(xb_g, t, v);
    x2_sync(g);
    x2_load_p2(xb_g, t, v);
    pass2_inv(v, tw2);
    x1_store_p2(xa_g, t, v);
    group_barrier(g);
    x1_load_p1(xa_g, t, v);
    radix16_inv(v, c_fft1024_pass1);
    p22_acc_update(acc_g, t, v);
    group_barrier(g);
  }
  __syncthreads();

  // ---- epilogue: sample extract (a16), optional many-LUT --------------
  sample_extract_many_lut(lwe_out, out_idx[s], gridDim.x, num_many_lut, lut_stride,
                          &sm.acc[0][0], P22_N, 1, P22_N, tid, 128, SameWord());
}

// ---------------------------------------------------------------------------
// v3 (shipped): v1's two-buffer / 2-CTA structure with a 32-bit running
// accumulator and an explicit software prefetch of the bootstrap key.  A profile
// of v1 on the hardware it was first tuned on showed 30 % of all stall samples in the MAC phase (long_scoreboard on the
// L2-resident key) and 23 % in the u64 rotate/decompose phase.  Experiments
// that were measured and dropped: 3 CTAs/SM at 168
// registers with or without prefetch (spills, exposed L2 latency), one template
// instance per thread group (I-cache), int->double on the fp64 pipe, L1
// prefetch of the other-row key values.  80 KiB smem, 255 regs, 2 CTAs / SM.
// ---------------------------------------------------------------------------
struct P22SmemV3 {
  cplx xa[2][P22_M];        // 32 KiB
  cplx xb[2][P22_M];        // 32 KiB
  uint32_t acc[2][P22_N];   // 16 KiB
  uint16_t a_hat[1024 + 8];
  uint32_t b_hat;
  unsigned long long red_half[4];
  long long red_dbl[4];
};

// MAC_MODE 3 only (launches of at most one CTA per SM): the 64 KiB Fourier key
// block of a step -- [column][row][16][64] complex, contiguous in the engine's
// layout -- is staged into a 2-slot shared-memory ring by cp.async.bulk (TMA) a
// whole step ahead; see tma_bulk.cuh.
struct P22SmemV3Tma {
  P22SmemV3 base;
  cplx ring[2][4][P22_M]; // 128 KiB
  unsigned long long bar[2];
};

// MAC_MODE 0 (round 1): own-row key values prefetched after the last forward
// pass, own spectrum kept in registers across the share barrier, other-row key
// values requested only after the own-row products have freed their registers:
// their L2 latency is exposed (the MAC phase was 16-18 % of a CMUX step in a
// per-phase clock profile, for 128 DP ops).
// MAC_MODE 1 (round 2): the own spectrum is written to shared memory anyway, so
// it is NOT kept in registers: all 32 key values of (GGSW i, column g) are
// requested right after the spectrum store and stay in flight across the
// barrier; the MAC then reads both spectra from shared memory.  +16 LDS.128 per
// thread and step, no exposed second L2 round trip.
// DIG_MODE 0: round-1 rotate + decompose; 1: p22v4_load_digits / acc_update.
// X2_MODE 0: exchange 2 through shared memory (warp-local); 1: through warp
// shuffles (x2_shfl.cuh),
// with the matching pass-2 thread assignment and exchange-1 swizzle (x1t_*).
template <int MAC_MODE, int DIG_MODE, int X2_MODE = 0>
__device__ __forceinline__ void
p22v3_blind_rotate(P22SmemV3 &sm, const cplx *__restrict__ bsk, int g, int t,
                   uint32_t n, uint32_t base_log, const cplx (&tw2)[3],
                   const cplx (&tw3)[15]) {
  uint32_t *acc_g = sm.acc[g];
  cplx *xa_g = sm.xa[g];
  cplx *xb_g = sm.xb[g];
  const cplx *xa_other = sm.xa[1 - g];
  // (GGSW i, column g) block = [row][b][t]; own row = g, other row = 1 - g
  const cplx *bsk_own = bsk + (size_t)g * (2 * P22_M) + (size_t)g * P22_M + t;
  const cplx *bsk_oth = bsk + (size_t)g * (2 * P22_M) + (size_t)(1 - g) * P22_M;
  uint32_t own[32]; // this thread's accumulator words, see p22v4_load_digits
  if constexpr (DIG_MODE != 0)
    p22v4_own_init(acc_g, t, own);
  [[maybe_unused]] P22SmemV3Tma *smt = nullptr;
  [[maybe_unused]] auto tma_issue = [&](uint32_t i) {
    if constexpr (MAC_MODE == 3) {
      unsigned long long *bar = &smt->bar[i & 1];
      mbar_arrive_expect_tx(bar, 4u * P22_M * (uint32_t)sizeof(cplx));
#pragma unroll
      for (int q = 0; q < 4; q++)
        tma_bulk_g2s(&smt->ring[i & 1][q][0],
                     bsk + (size_t)i * (4 * P22_M) + (size_t)q * P22_M,
                     P22_M * (uint32_t)sizeof(cplx), bar);
    }
  };
  if constexpr (MAC_MODE == 3) {
    smt = reinterpret_cast<P22SmemV3Tma *>(&sm);
    if (threadIdx.x == 0) {
      mbar_init(&smt->bar[0], 1);
      mbar_init(&smt->bar[1], 1);
      mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0 && n > 0)
      tma_issue(0);
  }
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t a = sm.a_hat[i];
    if constexpr (MAC_MODE == 3) {
      if (threadIdx.x == 0 && i + 1 < n)
        tma_issue(i + 1); // its last readers are behind the barrier after MAC i - 1
    } else {
      if (a == 0)
        continue;
    }
    const size_t step = (size_t)i * (4 * P22_M);
    cplx v[16], b_own[16];
    if constexpr (DIG_MODE == 0)
      p22v3_load_digits(acc_g, t, a, base_log, v);
    else
      p22v4_load_digits(acc_g, t, a, base_log, own, v);
    radix16_fwd(v, c_fft1024_pass1);
    if constexpr (X2_MODE == 1) {
      x1t_store_p1(xa_g, t, v);
      group_barrier(g);
      x1t_load_p2(xa_g, t, v);
      pass2_fwd(v, tw2);
      spec_guard_arrive(g, t);
      x2s_fwd(v);
    } else {
      x1_store_p1(xa_g, t, v);
      group_barrier(g);
      x1_load_p2(xa_g, t, v);
      pass2_fwd(v, tw2);
      spec_guard_arrive(g, t);
      x2_store_p2(xb_g, t, v);
      x2_sync(g); // exchange 2 stays inside groups of 4 adjacent lanes
      x2_load_p3(xb_g, t, v);
    }
    radix16_fwd(v, tw3);
    if constexpr (MAC_MODE == 0) {
      // own-row key values: requested here (after the last forward pass, so the
      // 64 registers are not live across it), consumed after
      // the share barrier
#pragma unroll
      for (int b = 0; b < 16; b++)
        b_own[b] = ldcg_cplx(bsk_own + step + b * 64);
      spec_guard_wait(g, t);
      spec_store(xa_g, t, v);
      __syncthreads();
      p22v3_mac(v, b_own, xa_other, bsk_oth + step, t, LdcgLoader());
    } else if constexpr (MAC_MODE == 3) {
      spec_guard_wait(g, t);
      spec_store(xa_g, t, v);
      __syncthreads();
      mbar_wait_parity(&smt->bar[i & 1], (i >> 1) & 1u);
      const cplx *k_own = &smt->ring[i & 1][2 * g + g][0];
      const cplx *k_oth = &smt->ring[i & 1][2 * g + (1 - g)][0];
#pragma unroll
      for (int b = 0; b < 16; b++)
        v[b] = cfma(xa_other[b * 64 + t], k_oth[b * 64 + t],
                    cmul(v[b], k_own[b * 64 + t]));
    } else if constexpr (MAC_MODE == 2) {
      // as mode 0, plus the first half of the other-row key values requested
      // before the barrier (232 live registers there) and the second half as
      // soon as the first own-row products have freed their registers
      cplx b_oth[16];
#pragma unroll
      for (int b = 0; b < 16; b++)
        b_own[b] = ldcg_cplx(bsk_own + step + b * 64);
#pragma unroll
      for (int b = 0; b < 8; b++)
        b_oth[b] = ldcg_cplx(bsk_oth + step + b * 64 + t);
      spec_guard_wait(g, t);
      spec_store(xa_g, t, v);
      __syncthreads();
#pragma unroll
      for (int b = 0; b < 8; b++)
        v[b] = cmul(v[b], b_own[b]);
#pragma unroll
      for (int b = 8; b < 16; b++)
        b_oth[b] = ldcg_cplx(bsk_oth + step + b * 64 + t);
#pragma unroll
      for (int b = 8; b < 16; b++)
        v[b] = cmul(v[b], b_own[b]);
#pragma unroll
      for (int b = 0; b < 16; b++)
        v[b] = cfma(xa_other[b * 64 + t], b_oth[b], v[b]);
    } else {
      spec_guard_wait(g, t);
      spec_store(xa_g, t, v);
      cplx b_oth[16];
#pragma unroll
      for (int b = 0; b < 16; b++)
        b_own[b] = ldcg_cplx(bsk_own + step + b * 64);
#pragma unroll
      for (int b = 0; b < 16; b++)
        b_oth[b] = ldcg_cplx(bsk_oth + step + b * 64 + t);
      __syncthreads();
#pragma unroll
      for (int b = 0; b < 16; b++)
        v[b] = cfma(xa_other[b * 64 + t], b_oth[b],
                    cmul(xa_g[b * 64 + t], b_own[b]));
    }
    __syncthreads();
    radix16_inv(v, tw3);
    if constexpr (X2_MODE == 1) {
      x2s_inv(v);
      pass2_inv(v, tw2);
      x1t_store_p2(xa_g, t, v);
      group_barrier(g);
      x1t_load_p1(xa_g, t, v);
    } else {
      x2_store_p3(xb_g, t, v);
      x2_sync(g);
      x2_load_p2(xb_g, t, v);
      pass2_inv(v, tw2);
      x1_store_p2(xa_g, t, v);
      group_barrier(g);
      x1_load_p1(xa_g, t, v);
    }
    radix16_inv(v, c_fft1024_pass1);
    if constexpr (DIG_MODE == 0)
      p22v2_acc_update(acc_g, t, v);
    else
      p22v4_acc_update(acc_g, t, v, own);
    group_barrier(g);
  }
}

template <int MAC_MODE, int DIG_MODE, int X2_MODE = 0>
__global__ void __launch_bounds__(128, 2)
pbs_n2048_k1_l1_v3_kernel(uint64_t *__restrict__ lwe_out,
                          const uint64_t *__restrict__ out_idx,
                          const uint64_t *__restrict__ luts,
                          const uint64_t *__restrict__ lut_idx,
                          const uint64_t *__restrict__ lwe_in,
                          const uint64_t *__restrict__ in_idx,
                          const cplx *__restrict__ bsk,
                          const Fft1024Tables *__restrict__ tables, uint32_t n,
                          uint32_t base_log, uint32_t num_many_lut,
                          uint32_t lut_stride, int centered_ms) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  P22SmemV3 &sm = *reinterpret_cast<P22SmemV3 *>(smem_raw);
  const int tid = threadIdx.x;
  const int g = tid >> 6;
  const int t = tid & 63;
  const uint32_t s = blockIdx.x;
  const uint32_t log_mod = 12;

  const uint64_t *ct = lwe_in + in_idx[s] * (uint64_t)(n + 1);
  CenteredMsSums sums;
  for (uint32_t i = tid; i < n; i += 128) {
    const uint64_t a = ct[i];
    sm.a_hat[i] = (uint16_t)modulus_switch_u64(a, log_mod);
    if (centered_ms)
      sums.add(a, log_mod);
  }
  if (centered_ms)
    centered_ms_publish_warp(sums, sm.red_half, sm.red_dbl);
  __syncthreads();
  if (tid == 0)
    sm.b_hat = ms_b_hat(ct[n], centered_ms, sm.red_half, sm.red_dbl, 4, log_mod);
  __syncthreads();
  rotate_lut(&sm.acc[0][0], P22_N, luts + lut_idx[s] * (uint64_t)(2 * P22_N), 2,
             P22_N, sm.b_hat, tid, 128, Torus64To32());
  cplx tw2[3], tw3[15];
#pragma unroll
  for (int e = 0; e < 3; e++)
    tw2[e] = tables->pass2[X2_MODE == 1 ? x1t_q(t) : (t >> 2)][e];
#pragma unroll
  for (int e = 0; e < 15; e++)
    tw3[e] = tables->pass3[t][e];
  __syncthreads();

  p22v3_blind_rotate<MAC_MODE, DIG_MODE, X2_MODE>(sm, bsk, g, t, n, base_log, tw2, tw3);
  __syncthreads();
  sample_extract_many_lut(lwe_out, out_idx[s], gridDim.x, num_many_lut, lut_stride,
                          &sm.acc[0][0], P22_N, 1, P22_N, tid, 128, Torus32To64());
}

// ---------------------------------------------------------------------------
// v6: the v3 arithmetic, bit for bit, with two data paths that take load off
// the shared-memory pipe and the register file:
//   * exchange 2 of every transform goes through warp shuffles (x2_shfl.cuh):
//     -1,024 shared-memory wavefronts per CMUX step and no second exchange
//     buffer, which frees 32 KiB of shared memory per CTA;
//   * that space holds a ONE-slot ring for the Fourier key block of a step
//     (64 KiB = [column][row][16][64] complex, contiguous in the engine's
//     layout), filled by the TMA unit (cp.async.bulk + mbarrier, tma_bulk.cuh)
//     a whole step ahead: the copy for step i + 1 is issued right after the MAC
//     of step i has released the slot and lands during the inverse transform.
//     No key value waits in a register: the L2 round trips that v3 exposes
//     twice per step leave the critical path, at two CTAs per SM (the TMA
//     variant 7 of v3 needs 208 KiB and runs one CTA per SM).
// 112 KiB shared memory per CTA, 2 CTAs / SM.
// Steps with a_hat = 0 are executed (they add exactly zero) so that the copy
// pipeline stays uniform.
// ---------------------------------------------------------------------------
// RING = number of 16 KiB key blocks the ring holds (4: whole block of a step,
// 2: the two "other" rows, 1: unused placeholder); STAGE_A: the switched mask is
// staged in shared memory (2 KiB) -- otherwise step i recomputes a_hat[i] from
// the input LWE word, loaded one step ahead: with the 64 KiB ring the 2 KiB
// would push the CTA over half an SM's shared memory.
template <int RING, bool STAGE_A>
struct P22SmemV6 {
  cplx xa[2][P22_M];        // 32 KiB  exchange 1 / spectrum share
  cplx ring[RING][P22_M];   // key blocks of one step
  uint32_t acc[2][P22_ACC_STRIDE]; // 16 KiB + 128 B
  uint16_t a_hat[STAGE_A ? 1024 + 8 : 4];
  uint32_t b_hat;
  unsigned long long red_half[4];
  long long red_dbl[4];
  unsigned long long bar;
};
// two CTAs per SM: 2 x (sizeof + 1 KiB reserved) <= 228 KiB
static_assert(sizeof(P22SmemV6<4, false>) <= 115712, "v6 must fit two CTAs per SM");
static_assert(sizeof(P22SmemV6<2, true>) <= 115712, "v6 hybrid must fit two CTAs per SM");

// Experiment knob (B200_P22_STAGGER=<cycles>, default 0): every second CTA that
// arrives on an SM starts that many cycles late, so that the two resident CTAs
// of an SM -- which run the same code at the same speed and would otherwise keep
// whatever phase relation they were launched with -- sit half a CMUX step apart.
__constant__ uint32_t c_p22_stagger;
__device__ uint32_t g_p22_sm_arrivals[512];

// Thread 0: the other-row key blocks of step i into the ring (KEY_MODE 2).
__device__ __forceinline__ void p22_ring_issue(cplx *ring, unsigned long long *bar,
                                               const cplx *bsk, uint32_t i) {
  mbar_arrive_expect_tx(bar, P22_RING_BYTES);
  tma_bulk_g2s(ring, p22_ring_src(bsk, i), P22_RING_BYTES, bar);
}

// What p22_lanepair_loop runs between its phases: nothing in the kernel; the
// phase-clock tool passes a probe that reads the clock.
struct P22NoProbe {
  __device__ __forceinline__ void begin() {}
  __device__ __forceinline__ void lap(int) {}
};

// The blind rotation of the lane-pair layout (pbs_n2048_lanepair.cuh): the
// pieces of each CMUX step in order, with the barriers, the warp exchanges and
// the key wait between them.  The MAC takes the other polynomial's value from
// lane l ^ 16 with one shuffle: no spectrum store, no barrier between the
// polynomials before or after it.  Exchange 2 goes through this warp's rows of
// xa[g] (X2 = 1, x2m_*) or stays inside each half-warp as shuffles (X2 = 0,
// x2h_*).  The values and the order of every operation are those of the other
// v6 instances, so the results are bit-identical.  Expects the ring copy of
// step 0 issued and the accumulator, a_hat and the barrier set up.
template <int X2, typename Probe>
__device__ __forceinline__ void
p22_lanepair_loop(P22SmemV6<2, true> &sm, const cplx *bsk, uint32_t n,
                  uint32_t base_log, const cplx *tw2, const cplx *tw3, Probe &probe) {
  const P22LanePair lp(threadIdx.x, sm.acc, sm.xa, sm.ring, bsk, c_fft1024_pass1, tw2, tw3);
  uint32_t own[32];
  lp.own_init(own);
  uint32_t a_next = n > 0 ? sm.a_hat[0] : 0;
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t a = a_next; // read a step ahead: every address of the step hangs on it
    a_next = sm.a_hat[i + 1];  // a_hat has 8 words of padding
    cplx v[16];
    probe.begin();
    lp.digits(a, base_log, own, v);                                     probe.lap(0);
    lp.fwd_pass1(v);                                                    probe.lap(1);
    lp.x1_fwd_store(v); __syncthreads(); lp.x1_fwd_load(v);             probe.lap(2);
    lp.fwd_pass2(v);                                                    probe.lap(3);
    if constexpr (X2 == 1) x2m_fwd(lp.x2_rows, v); else x2h_fwd(v);     probe.lap(4);
    lp.fwd_pass3(v);                                                    probe.lap(5);
    cplx b_own[16];
    lp.own_row_load(i, b_own); mbar_wait_parity(&sm.bar, i & 1u);       probe.lap(6);
    lp.mac(v, b_own, [](int, cplx x) { return shfl_xor_cplx(x, 16); }); probe.lap(7);
    lp.inv_pass3(v);                                                    probe.lap(8);
    if constexpr (X2 == 1) x2m_inv(lp.x2_rows, v); else x2h_inv(v);     probe.lap(9);
    lp.inv_pass2(v);                                                    probe.lap(10);
    // the forward exchange-1 loads (or the exchange-2 loads) of this warp read
    // the same slots (rows 4 w .. 4 w + 3 of xa[g]); no other warp touches them
    // in between
    __syncwarp();
    lp.x1_inv_store(v);
    __syncthreads();
    if (threadIdx.x == 0 && i + 1 < n)
      p22_ring_issue(&sm.ring[0][0], &sm.bar, bsk, i + 1); // every warp is past its MAC
    lp.x1_inv_load(v);                                                  probe.lap(11);
    lp.inv_pass1(v);                                                    probe.lap(12);
    lp.acc_update(v, own); __syncthreads();                             probe.lap(13);
  }
}

// KEY_MODE 0: key block through the TMA ring; 1: v3's register prefetch
// (own row after the last forward pass, other row after the own products) --
// the A/B partner that isolates the effect of the ring; 2: own row through
// registers, other row (the one v3 waits for) through the ring.
// X2 (lane-pair layout only): exchange 2 through the warp's own rows of xa[g]
// (1, x2m_*, x2_smem.cuh) or through half-warp shuffles (0, x2h_*).
template <int KEY_MODE, bool STAGE_A, int CVT = 0, int SPLIT_POST = 0, int X2 = 1>
__global__ void __launch_bounds__(128, 2)
pbs_n2048_k1_l1_v6_kernel(uint64_t *__restrict__ lwe_out,
                          const uint64_t *__restrict__ out_idx,
                          const uint64_t *__restrict__ luts,
                          const uint64_t *__restrict__ lut_idx,
                          const uint64_t *__restrict__ lwe_in,
                          const uint64_t *__restrict__ in_idx,
                          const cplx *__restrict__ bsk,
                          const Fft1024Tables *__restrict__ tables, uint32_t n,
                          uint32_t base_log, uint32_t num_many_lut,
                          uint32_t lut_stride, int centered_ms) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int RING = KEY_MODE == 0 ? 4 : KEY_MODE == 2 ? 2 : 1;
  // The shipped two-CTA instance runs the lane-pair layout (p22_lanepair_loop).
  constexpr bool LANE_PAIR = KEY_MODE == 2 && STAGE_A && CVT == 2 && SPLIT_POST == 1;
  using Smem = P22SmemV6<RING, STAGE_A>;
  Smem &sm = *reinterpret_cast<Smem *>(smem_raw);
  const int tid = threadIdx.x;
  const int g = LANE_PAIR ? p22lp_g(tid) : tid >> 6;
  const int t = LANE_PAIR ? p22lp_t(tid) : tid & 63;
  const uint32_t s = blockIdx.x;
  const uint32_t log_mod = 12;

  if (c_p22_stagger) {
    if (tid == 0) {
      uint32_t smid;
      asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
      if (atomicAdd(&g_p22_sm_arrivals[smid & 511], 1u) & 1u) {
        const long long until = clock64() + (long long)c_p22_stagger;
        while (clock64() < until)
          __nanosleep(100);
      }
    }
    __syncthreads();
  }
  if (tid == 0) {
    mbar_init(&sm.bar, 1);
    mbar_fence_init();
  }
  const uint64_t *ct = lwe_in + in_idx[s] * (uint64_t)(n + 1);
  CenteredMsSums sums;
  if (centered_ms || STAGE_A) {
    for (uint32_t i = tid; i < n; i += 128) {
      const uint64_t a = ct[i];
      if constexpr (STAGE_A)
        sm.a_hat[i] = (uint16_t)modulus_switch_u64(a, log_mod);
      if (centered_ms)
        sums.add(a, log_mod);
    }
  }
  if (centered_ms)
    centered_ms_publish_warp(sums, sm.red_half, sm.red_dbl);
  __syncthreads();
  auto tma_issue = [&](uint32_t i) {
    if constexpr (KEY_MODE == 2) {
      p22_ring_issue(&sm.ring[0][0], &sm.bar, bsk, i); // other rows only
    } else {
      mbar_arrive_expect_tx(&sm.bar, 4u * P22_M * (uint32_t)sizeof(cplx));
#pragma unroll
      for (int q = 0; q < 4; q++)
        tma_bulk_g2s(&sm.ring[q][0],
                     bsk + (size_t)i * (4 * P22_M) + (size_t)q * P22_M,
                     P22_M * (uint32_t)sizeof(cplx), &sm.bar);
    }
  };
  if (tid == 0) {
    if (KEY_MODE != 1 && n > 0)
      tma_issue(0);
    sm.b_hat = ms_b_hat(ct[n], centered_ms, sm.red_half, sm.red_dbl, 4, log_mod);
  }
  __syncthreads();
  rotate_lut(&sm.acc[0][0], P22_ACC_STRIDE, luts + lut_idx[s] * (uint64_t)(2 * P22_N),
             2, P22_N, sm.b_hat, tid, 128, Torus64To32());
  cplx tw2[3], tw3[15];
#pragma unroll
  for (int e = 0; e < 3; e++)
    tw2[e] = tables->pass2[LANE_PAIR ? x1h_q(t) : x1t_q(t)][e];
#pragma unroll
  for (int e = 0; e < 15; e++)
    tw3[e] = tables->pass3[t][e];
  __syncthreads();

  if constexpr (LANE_PAIR) {
    P22NoProbe probe;
    p22_lanepair_loop<X2>(sm, bsk, n, base_log, tw2, tw3, probe);
  } else {
    uint32_t *acc_g = sm.acc[g];
    cplx *xa_g = sm.xa[g];
    [[maybe_unused]] const cplx *xa_other = sm.xa[1 - g];
    // ring slot of block 2c + r: RING = 4 -> 2c + r; RING = 2 -> blocks 1, 2 at 0, 1
    [[maybe_unused]] const cplx *k_own = &sm.ring[RING == 4 ? 2 * g + g : 0][0];
    const cplx *k_oth = &sm.ring[RING == 4 ? 2 * g + (1 - g) : RING == 2 ? g : 0][0];
    const cplx *bsk_own = bsk + (size_t)g * (2 * P22_M) + (size_t)g * P22_M + t;
    [[maybe_unused]] const cplx *bsk_oth =
        bsk + (size_t)g * (2 * P22_M) + (size_t)(1 - g) * P22_M;
    uint32_t own[32];
    p22v4_own_init(acc_g, t, own);
    [[maybe_unused]] uint64_t ct_next = (!STAGE_A && n > 0) ? ct[0] : 0;
    [[maybe_unused]] uint32_t a_next = (STAGE_A && n > 0) ? sm.a_hat[0] : 0;
    for (uint32_t i = 0; i < n; i++) {
      uint32_t a;
      if constexpr (STAGE_A) {
        a = a_next; // read a step ahead: every address of the step hangs on it
        a_next = sm.a_hat[i + 1]; // a_hat has 8 words of padding
      } else {
        a = modulus_switch_u64(ct_next, log_mod) & (2 * P22_N - 1);
        if (i + 1 < n)
          ct_next = ct[i + 1];
      }
      if constexpr (KEY_MODE == 1) {
        if (a == 0)
          continue;
      }
      cplx v[16];
      p22v4_load_digits<CVT>(acc_g, t, a, base_log, own, v);
      radix16_fwd(v, c_fft1024_pass1);
      x1t_store_p1(xa_g, t, v);
      group_barrier(g);
      x1t_load_p2(xa_g, t, v);
      pass2_fwd(v, tw2);
      spec_guard_arrive(g, t);
      x2s_fwd(v);
      radix16_fwd(v, tw3);
      if constexpr (KEY_MODE == 0) {
        spec_guard_wait(g, t);
        spec_store(xa_g, t, v);
        __syncthreads();
        mbar_wait_parity(&sm.bar, i & 1u);
#pragma unroll
        for (int b = 0; b < 16; b++)
          v[b] = cfma(xa_other[b * 64 + t], k_oth[b * 64 + t],
                      cmul(v[b], k_own[b * 64 + t]));
        if constexpr (SPLIT_POST) {
          mac_done_arrive(g);
        } else {
          __syncthreads();
          if (tid == 0 && i + 1 < n)
            tma_issue(i + 1); // every reader of the slot is behind the barrier
        }
      } else if constexpr (KEY_MODE == 2) {
        // own row through registers (requested here, consumed after the share
        // barrier), other row from the ring: half the ring traffic of mode 0
        const size_t step = (size_t)i * (4 * P22_M);
        cplx b_own[16];
#pragma unroll
        for (int b = 0; b < 16; b++)
          b_own[b] = ldcg_cplx(bsk_own + step + b * 64);
        spec_guard_wait(g, t);
        spec_store(xa_g, t, v);
        if constexpr (SPLIT_POST == 2) {
          spec_ready_arrive(g);
#pragma unroll
          for (int b = 0; b < 16; b++)
            v[b] = cmul(v[b], b_own[b]); // same operation order as below
          spec_ready_wait(g);
          mbar_wait_parity(&sm.bar, i & 1u);
#pragma unroll
          for (int b = 0; b < 16; b++)
            v[b] = cfma(xa_other[b * 64 + t], k_oth[b * 64 + t], v[b]);
        } else {
        __syncthreads();
        mbar_wait_parity(&sm.bar, i & 1u);
#pragma unroll
        for (int b = 0; b < 16; b++)
          v[b] = cfma(xa_other[b * 64 + t], k_oth[b * 64 + t],
                      cmul(v[b], b_own[b]));
        }
        if constexpr (SPLIT_POST) {
          mac_done_arrive(g);
        } else {
          __syncthreads();
          if (tid == 0 && i + 1 < n)
            tma_issue(i + 1);
        }
      } else {
        const size_t step = (size_t)i * (4 * P22_M);
        cplx b_own[16];
#pragma unroll
        for (int b = 0; b < 16; b++)
          b_own[b] = ldcg_cplx(bsk_own + step + b * 64);
        spec_guard_wait(g, t);
        spec_store(xa_g, t, v);
        __syncthreads();
        p22v3_mac(v, b_own, xa_other, bsk_oth + step, t, LdcgLoader());
        __syncthreads();
      }
      radix16_inv(v, tw3);
      x2s_inv(v);
      pass2_inv(v, tw2);
      if constexpr (SPLIT_POST && KEY_MODE != 1)
        mac_done_wait(g); // the other group has read this group's spectrum
      x1t_store_p2(xa_g, t, v);
      group_barrier(g);
      if constexpr (SPLIT_POST && KEY_MODE != 1) {
        if (tid == 0 && i + 1 < n)
          tma_issue(i + 1); // both groups are past their MAC: the slot is free
      }
      x1t_load_p1(xa_g, t, v);
      radix16_inv(v, c_fft1024_pass1);
      p22v4_acc_update(acc_g, t, v, own);
      group_barrier(g);
    }
  }
  __syncthreads();
  sample_extract_many_lut(lwe_out, out_idx[s], gridDim.x, num_many_lut, lut_stride,
                          &sm.acc[0][0], P22_ACC_STRIDE, 1, P22_N, tid, 128,
                          Torus32To64());
}

// ---------------------------------------------------------------------------
// BSK conversion for this kernel: standard-domain u64 polynomial (i, r, c)
// -> spectrum scaled by 2^-64 / M, stored at [(i*2 + c)*2 + r][b][t].
// grid = n * 4 polynomials (source order [i][r][c]), block = 64.
// Replaces cuda_convert_lwe_programmable_bootstrap_key_64_async's
// batch_FFT16x4x16_classical_specialized
// (cuda/src/pbs/bootstrapping_key.cuh:141-250, fft/bnsmfft.cuh:612).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(64)
bsk_convert_n2048_k1_l1_kernel(cplx *__restrict__ dst,
                               const uint64_t *__restrict__ src,
                               const Fft1024Tables *__restrict__ tables) {
  __shared__ cplx xa[P22_M];
  __shared__ cplx xb[P22_M];
  const int t = threadIdx.x;
  const uint32_t poly = blockIdx.x; // = (i*2 + r)*2 + c
  const uint32_t i = poly >> 2, r = (poly >> 1) & 1, c = poly & 1;
  const uint64_t *p = src + (size_t)poly * P22_N;
  const double scale = 2.27373675443232059478759765625e-13; // 2^-42 = 2^-64 / 1024 * 2^32 (see scaled_double_to_torus32)
  cplx v[16];
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    const uint32_t j = 64u * j1 + t;
    v[j1] = cmake(ll_to_double((int64_t)p[j]) * scale,
                  ll_to_double((int64_t)p[j + P22_M]) * scale);
  }
  radix16_fwd(v, c_fft1024_pass1);
  x1_store_p1(xa, t, v);
  __syncthreads();
  x1_load_p2(xa, t, v);
  pass2_fwd(v, &tables->pass2[t >> 2][0]);
  x2_store_p2(xb, t, v);
  __syncthreads();
  x2_load_p3(xb, t, v);
  radix16_fwd(v, tables->pass3[t]);
  cplx *out = dst + (((size_t)i * 2 + c) * 2 + r) * P22_M;
  spec_store(out, t, v);
}

} // namespace b200
