// pbs_n8192.cuh -- sm_90a register-FFT classic PBS for (N = 8192, k = 1,
// l = 2): PARAM_MESSAGE_3_CARRY_3_KS_PBS (n = 1077, log B = 15;
// tfhe/src/shortint/parameters/v1_0/classic/tuniform/p_fail_2_minus_128/
// ks_pbs.rs:67-77).  The working set of this shape (two 8192-coefficient
// accumulators, four 4096-point spectra per step, 512 KiB of Fourier key per
// step) does not fit one SM's shared memory: round 1 and the reference's CUDA
// backend run it on kernels that keep all of it in global memory.  Here the
// accumulators, the exchanges and the key stream stay on chip and only the
// parked spectra go off chip, to a per-thread area that stays in L2:
//
//   * one LWE per CTA, 256 threads, one CTA per SM, persistent grid (all
//     resident CTAs walk the 565 MB key together: it is read from HBM once per
//     round of the grid);
//   * 4096-point transform = 16 x 16 x 16 (negacyclic_fft.cuh, xg_* / xq_*):
//     three register passes, exchange 1 across the CTA through a 64 KiB
//     shared-memory buffer, exchange 2 inside a half-warp in that half-warp's own
//     region of the same buffer;
//   * the (k+1) l = 4 forward transforms of a step run one after the other; each
//     spectrum (16 values = 256 bytes per thread) is PARKED in a per-thread
//     area of a global workspace -- 256 threads x 4 spectra x 256 bytes =
//     256 KiB per CTA, 33 MiB for a grid of 132 CTAs, sized to fit the 50 MiB
//     L2 next to the key stream (L2-only accesses; whether it stays resident is
//     not measured, only the kernel's speed against the generic workspace kernel
//     is, see DESIGN.md section 4) -- and fetched back by the Fourier MAC, which is thread-local: thread t3 owns
//     slots 16 t3 .. 16 t3 + 15 of every spectrum and of both output columns;
//   * u32 running accumulator (top 32 bits) in shared memory, as in the other
//     register kernels.  With l * log B = 30 the decomposition drops only TWO
//     bits of that word, so an exact tie is hit by a quarter of all values: the
//     reference's round-half-up (harmless on its 64-bit word, where a tie has
//     probability 2^-34) would bias every coefficient by +2^-33 here -- measured
//     10x the oracle's output noise on PARAM_MESSAGE_3_CARRY_3.  The tie goes
//     to EVEN instead, exactly as in the multi-bit kernels (digits_u32,
//     pbs_multibit_n2048_phases.cuh) and under the same switch
//     (b200_set_multibit_tie_rule(1) restores round-half-up).
// Fourier key layout: [i][level slot][row r][column c][b < 16][t3 < 256]
// complex128, value at slot pos = 16 t3 + b, pre-scaled by 2^-64 / 4096 * 2^32.
#pragma once
#include "pbs_n8192_phases.cuh"          // sizes, key layout, rotate + decompose (host + device)
#include "pbs_n2048.cuh"                 // ldcg_cplx, phases
#include "pbs_n512.cuh"                  // ldnc_cplx
#include "tma_bulk.cuh"

#include <cuda_runtime.h>

namespace b200 {


__constant__ cplx c_fft4096_pass1[15];

struct N8192Smem {
  cplx xbuf[P8K_M];          // 64 KiB  exchanges 1 and 2
  uint32_t acc[2][P8K_N];    // 64 KiB
  uint16_t a_hat[2048 + 8];
  uint32_t b_hat;
  unsigned long long red_half;
  long long red_dbl;
};

// Park area of a CTA: [slot < 4][value < 16][thread < 256] complex, so that a
// warp's access to one value is 512 contiguous bytes.  L2-only accesses: the
// area is re-read within a step, by the thread that wrote it.
constexpr size_t P8K_PARK_PER_CTA = 4 * 16 * 256;
__device__ __forceinline__ cplx *n8192_park_area(cplx *park, int t) {
  return park + (size_t)blockIdx.x * P8K_PARK_PER_CTA + t;
}
__device__ __forceinline__ cplx *park_slot(cplx *pk, uint32_t slot) { return pk + (size_t)slot * (16 * 256); }
__device__ __forceinline__ void park16(cplx *slot, const cplx v[16]) {
#pragma unroll
  for (int b = 0; b < 16; b++)
    __stcg(reinterpret_cast<double2 *>(slot + b * 256), make_double2(v[b].re, v[b].im));
}
__device__ __forceinline__ void fetch16(const cplx *slot, cplx v[16]) {
#pragma unroll
  for (int b = 0; b < 16; b++) {
    const double2 x = __ldcg(reinterpret_cast<const double2 *>(slot + b * 256));
    v[b] = cmake(x.x, x.y);
  }
}
// 16 words (packed digits) in the first four values of a slot
__device__ __forceinline__ void park_words16(cplx *slot, const uint32_t (&r)[16]) {
#pragma unroll
  for (int q = 0; q < 4; q++)
    __stcg(reinterpret_cast<uint4 *>(slot + q * 256), make_uint4(r[4 * q], r[4 * q + 1], r[4 * q + 2], r[4 * q + 3]));
}
__device__ __forceinline__ void fetch_words16(const cplx *slot, uint32_t (&r)[16]) {
#pragma unroll
  for (int q = 0; q < 4; q++) {
    const uint4 x = __ldcg(reinterpret_cast<const uint4 *>(slot + q * 256));
    r[4 * q] = x.x;
    r[4 * q + 1] = x.y;
    r[4 * q + 2] = x.z;
    r[4 * q + 3] = x.w;
  }
}

// digits of level slot `lvl` of ct1 = acc * X^a - acc for polynomial `acc_p`:
// thread t holds complex coefficients j = 256*j1 + t (re <- j, im <- j + 4096)
__device__ __forceinline__ void n8192_load_digits(const uint32_t *acc_p, int t,
                                                  uint32_t a, uint32_t base_log,
                                                  uint32_t lvl, bool ties_even,
                                                  cplx v[16]) {
  const uint32_t d = a & (P8K_N - 1);
  const bool neg0 = (a >> 13) != 0u; // a >= N
  const uint32_t base4 = ((uint32_t)t - d) * 4u;
  const unsigned char *accb = reinterpret_cast<const unsigned char *>(acc_p);
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    const uint32_t j = 256u * j1 + (uint32_t)t;
    const uint32_t ub0 = base4 + 1024u * j1;     // 4 * (j - d)
    const uint32_t ub1 = ub0 + 4u * P8K_M;       // 4 * (j + M - d)
    const uint32_t ib0 = ub0 & (4u * P8K_N - 4u);
    const uint32_t r0 = *reinterpret_cast<const uint32_t *>(accb + ib0);
    const uint32_t r1 =
        *reinterpret_cast<const uint32_t *>(accb + (ib0 ^ (4u * P8K_M)));
    const bool n0 = ((int32_t)ub0 < 0) != neg0;
    const bool n1 = ((int32_t)ub1 < 0) != neg0;
    const uint32_t x0 = (n0 ? 0u - r0 : r0) - acc_p[j];
    const uint32_t x1 = (n1 ? 0u - r1 : r1) - acc_p[j + P8K_M];
    int32_t d0[2], d1[2];
    digits_u32<2>(x0, base_log, 2, d0, ties_even);
    digits_u32<2>(x1, base_log, 2, d1, ties_even);
    v[j1] = cmake(int_to_double(lvl ? d0[1] : d0[0]),
                  int_to_double(lvl ? d1[1] : d1[0]));
  }
}

// forward transform of v (pass-1 layout) -> pass-3 layout, thread t
__device__ __forceinline__ void n8192_forward(cplx v[16], cplx *xbuf, int t,
                                              const Fft4096Tables *tables) {
  radix16_fwd(v, c_fft4096_pass1);
  __syncthreads(); // every half-warp is done with its region (previous exchange 2)
  xg_store_p1(xbuf, t, v);
  __syncthreads();
  xg_load_p2(xbuf, t, v);
  {
    cplx tw[15];
#pragma unroll
    for (int e = 0; e < 15; e++)
      tw[e] = ldnc_cplx(&tables->pass2[t >> 4][e]);
    radix16_fwd(v, tw);
  }
  cplx *hw = xbuf + (t >> 4) * 256; // this half-warp's region
  __syncwarp();
  xq_store_p1(hw, t & 15, v);
  __syncwarp();
  xq_load_p2(hw, t & 15, v);
  {
    cplx tw[15];
#pragma unroll
    for (int e = 0; e < 15; e++)
      tw[e] = ldnc_cplx(&tables->pass3[t][e]);
    radix16_fwd(v, tw);
  }
}

// inverse transform: pass-3 layout -> pass-1 layout (unnormalised: the 1/M is in the key)
__device__ __forceinline__ void n8192_inverse(cplx v[16], cplx *xbuf, int t,
                                              const Fft4096Tables *tables) {
  {
    cplx tw[15];
#pragma unroll
    for (int e = 0; e < 15; e++)
      tw[e] = ldnc_cplx(&tables->pass3[t][e]);
    radix16_inv(v, tw);
  }
  cplx *hw = xbuf + (t >> 4) * 256;
  __syncthreads(); // the buffer is free (exchange-1 loads of the previous transform)
  xq_store_p2(hw, t & 15, v);
  __syncwarp();
  xq_load_p1(hw, t & 15, v);
  {
    cplx tw[15];
#pragma unroll
    for (int e = 0; e < 15; e++)
      tw[e] = ldnc_cplx(&tables->pass2[t >> 4][e]);
    radix16_inv(v, tw);
  }
  __syncwarp();
  xg_store_p2(xbuf, t, v); // into this half-warp's own region
  __syncthreads();
  xg_load_p1(xbuf, t, v);
  radix16_inv(v, c_fft4096_pass1);
}

// persistent grid, block = 256, one CTA per SM
__global__ void __launch_bounds__(256, 1)
pbs_n8192_k1_l2_kernel(uint64_t *__restrict__ lwe_out,
                       const uint64_t *__restrict__ out_idx,
                       const uint64_t *__restrict__ luts,
                       const uint64_t *__restrict__ lut_idx,
                       const uint64_t *__restrict__ lwe_in,
                       const uint64_t *__restrict__ in_idx,
                       const cplx *__restrict__ bsk,
                       const Fft4096Tables *__restrict__ tables, uint32_t n,
                       uint32_t base_log, uint32_t num_samples,
                       uint32_t num_many_lut, uint32_t lut_stride,
                       int centered_ms, int ties_even, cplx *__restrict__ park) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  N8192Smem &sm = *reinterpret_cast<N8192Smem *>(smem_raw);
  const int t = threadIdx.x;
  const uint32_t log_mod = 14; // log2(2N)

  cplx *const pk = n8192_park_area(park, t);

  for (uint32_t s = blockIdx.x; s < num_samples; s += gridDim.x) {
    // ---- prologue: modulus switch, acc = LUT * X^{-b_hat} -------------------
    const uint64_t *ct = lwe_in + in_idx[s] * (uint64_t)(n + 1);
    if (t == 0) {
      sm.red_half = 0;
      sm.red_dbl = 0;
    }
    __syncthreads();
    {
      CenteredMsSums sums;
      for (uint32_t i = t; i < n; i += 256) {
        const uint64_t a = ct[i];
        sm.a_hat[i] = (uint16_t)modulus_switch_u64(a, log_mod);
        if (centered_ms)
          sums.add(a, log_mod);
      }
      if (centered_ms)
        centered_ms_publish_atomic(sums, &sm.red_half, &sm.red_dbl);
    }
    __syncthreads();
    if (t == 0)
      sm.b_hat = ms_b_hat(ct[n], centered_ms, &sm.red_half, &sm.red_dbl, 1, log_mod);
    __syncthreads();
    rotate_lut(&sm.acc[0][0], P8K_N, luts + lut_idx[s] * (uint64_t)(2 * P8K_N), 2,
               P8K_N, sm.b_hat, t, 256, Torus64To32());
    __syncthreads();

    // ---- blind rotation ---------------------------------------------------------
    for (uint32_t i = 0; i < n; i++) {
      const uint32_t a = sm.a_hat[i];
      if (a == 0)
        continue; // uniform across the CTA
      // forward: spectrum index sp = 2 lvl + r, parked in slot sp
#pragma unroll 1
      for (uint32_t sp = 0; sp < 4; sp++) {
        const uint32_t lvl = sp >> 1, r = sp & 1;
        cplx v[16];
        n8192_load_digits(sm.acc[r], t, a, base_log, lvl, ties_even != 0, v);
        n8192_forward(v, sm.xbuf, t, tables);
        park16(park_slot(pk, sp), v);
      }
      // per output column: Fourier MAC (thread-local), inverse, accumulate
      // key block (i, level slot, row, column): [b][t3]
      const cplx *key_i = bsk + (size_t)i * (8 * P8K_M) + t;
#pragma unroll 1
      for (uint32_t c = 0; c < 2; c++) {
        cplx out[16];
        cplx kbuf[3][8];
        auto key_chunk = [&](int ch, cplx (&dst)[8]) {
          // ch = 2 sp + half; block index = (lvl * 2 + r) * 2 + c = 2 sp + c
          const int sp = ch >> 1, hb = (ch & 1) * 8;
          const cplx *kb = key_i + (size_t)(2 * sp + c) * P8K_M;
#pragma unroll
          for (int b = 0; b < 8; b++)
            dst[b] = ldcg_cplx(kb + (hb + b) * 256);
        };
        key_chunk(0, kbuf[0]);
        key_chunk(1, kbuf[1]);
#pragma unroll
        for (int sp = 0; sp < 4; sp++) {
          cplx f[16];
          fetch16(park_slot(pk, sp), f);
#pragma unroll
          for (int h = 0; h < 2; h++) {
            const int ch = 2 * sp + h;
            if (ch + 2 < 8)
              key_chunk(ch + 2, kbuf[(ch + 2) % 3]);
#pragma unroll
            for (int b = 0; b < 8; b++)
              out[8 * h + b] = sp == 0 ? cmul(f[8 * h + b], kbuf[ch % 3][b])
                                       : cfma(f[8 * h + b], kbuf[ch % 3][b], out[8 * h + b]);
          }
        }
        n8192_inverse(out, sm.xbuf, t, tables);
        // acc[c] += result; the other column still needs the OLD acc[c]? no:
        // the spectra of this step are already parked, nothing reads acc again
        // before the next step
        uint32_t *acc_c = sm.acc[c];
#pragma unroll
        for (int j1 = 0; j1 < 16; j1++) {
          const uint32_t j = 256u * j1 + (uint32_t)t;
          acc_c[j] += scaled_double_to_torus32(out[j1].re);
          acc_c[j + P8K_M] += scaled_double_to_torus32(out[j1].im);
        }
      }
      __syncthreads(); // accumulator complete before the next step's rotated reads
    }
    __syncthreads();

    // ---- epilogue: sample extract, optional many-LUT ---------------------------
    sample_extract_many_lut(lwe_out, out_idx[s], num_samples, num_many_lut, lut_stride,
                            &sm.acc[0][0], P8K_N, 1, P8K_N, t, 256, Torus32To64());
    __syncthreads(); // the working set is reused by the next sample
  }
}

// ===========================================================================
// Second generation (the default): same arithmetic and results, three
// scheduling changes relative to the first one:
//   * the Fourier key streams through a TMA ring in shared memory (5 slots of
//     16 KiB = 4 slot rows x 256 threads), refilled by thread 0 one chunk behind
//     the consumers and running ahead through the transforms, instead of
//     per-thread 128-bit loads that exposed the L2 latency inside the MAC;
//   * each accumulator polynomial is rotated and decomposed ONCE per step: the
//     level-1 digits wait, packed two per word, in the park slot that will
//     hold that level's spectrum;
//   * pass-2 / pass-3 twiddles are requested while the values are in flight
//     through the exchange buffers (their registers are dead there).
// ===========================================================================
#define P8K_SLOTS 5
#define P8K_CHUNK 1024 // complex values per ring slot: 4 rows [b] x 256 threads

struct N8192SmemV2 {
  cplx xbuf[P8K_M];                 // 64 KiB  exchanges 1 and 2
  uint32_t acc[2][P8K_N];           // 64 KiB
  cplx ring[P8K_SLOTS][P8K_CHUNK];  // 80 KiB  Fourier key chunks
  uint16_t a_hat[2048 + 8];
  unsigned long long full[P8K_SLOTS];
  unsigned long long empty[P8K_SLOTS];
  uint32_t b_hat;
  unsigned long long red_half;
  long long red_dbl;
};

__device__ __forceinline__ void n8192_load_tw(const cplx *row, cplx tw[15]) {
#pragma unroll
  for (int e = 0; e < 15; e++)
    tw[e] = ldnc_cplx(row + e);
}

// twiddle rows are requested one pass AHEAD of their use (the tables do not fit
// the L1 left beside 217 KiB of shared memory: an L2 round trip is about one
// radix-16 pass long)
__device__ __forceinline__ void n8192_forward_v2(cplx v[16], cplx *xbuf, int t,
                                                 const Fft4096Tables *tables) {
  cplx tw2[15], tw3[15];
  n8192_load_tw(&tables->pass2[t >> 4][0], tw2);
  radix16_fwd(v, c_fft4096_pass1);
  __syncthreads(); // every half-warp is done with its region (previous exchange 2)
  xg_store_p1(xbuf, t, v);
  __syncthreads();
  xg_load_p2(xbuf, t, v);
  n8192_load_tw(&tables->pass3[t][0], tw3);
  radix16_fwd(v, tw2);
  cplx *hw = xbuf + (t >> 4) * 256;
  __syncwarp();
  xq_store_p1(hw, t & 15, v);
  __syncwarp();
  xq_load_p2(hw, t & 15, v);
  radix16_fwd(v, tw3);
}

// tw3: pass-3 twiddles of this thread, already loaded by the caller
__device__ __forceinline__ void n8192_inverse_v2(cplx v[16], cplx tw3[15], cplx *xbuf,
                                                 int t, const Fft4096Tables *tables) {
  cplx tw2[15];
  n8192_load_tw(&tables->pass2[t >> 4][0], tw2);
  radix16_inv(v, tw3);
  cplx *hw = xbuf + (t >> 4) * 256;
  __syncthreads(); // the buffer is free (exchange-1 loads of the previous transform)
  xq_store_p2(hw, t & 15, v);
  __syncwarp();
  xq_load_p1(hw, t & 15, v);
  radix16_inv(v, tw2);
  __syncwarp();
  xg_store_p2(xbuf, t, v);
  __syncthreads();
  xg_load_p1(xbuf, t, v);
  radix16_inv(v, c_fft4096_pass1);
}

// ALL_ARRIVE (debug instance for compute-sanitizer racecheck): every consumer
// thread arrives on the slot's `empty` barrier itself instead of lane 0 after a
// __syncwarp -- the tool follows a direct arrive -> wait edge but not the
// reads -> __syncwarp -> lane-0 arrive chain of the shipped instance.
template <bool ALL_ARRIVE>
__global__ void __launch_bounds__(256, 1)
pbs_n8192_k1_l2_v2_kernel(uint64_t *__restrict__ lwe_out,
                          const uint64_t *__restrict__ out_idx,
                          const uint64_t *__restrict__ luts,
                          const uint64_t *__restrict__ lut_idx,
                          const uint64_t *__restrict__ lwe_in,
                          const uint64_t *__restrict__ in_idx,
                          const cplx *__restrict__ bsk,
                          const Fft4096Tables *__restrict__ tables, uint32_t n,
                          uint32_t base_log, uint32_t num_samples,
                          uint32_t num_many_lut, uint32_t lut_stride,
                          int centered_ms, int ties_even,
                          uint32_t stagger_cycles, cplx *__restrict__ park) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  N8192SmemV2 &sm = *reinterpret_cast<N8192SmemV2 *>(smem_raw);
  const int t = threadIdx.x;
  const uint32_t log_mod = 14; // log2(2N)

  if (t == 0) {
    for (int s = 0; s < P8K_SLOTS; s++) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], ALL_ARRIVE ? 256 : 8); // one arrival per warp
    }
    mbar_fence_init();
  }
  __syncthreads();
  cplx *const pk = n8192_park_area(park, t);

  // experiment knob (B200_N8192_STAGGER, default 0): CTA b starts b / grid of
  // `stagger_cycles` late, so that the CTAs sit in different phases of a step
  // and their key reads do not hit the L2 at the same moment.  Measured: no
  // effect between 0 and 240 k cycles -- the
  // key path is not what bounds the step.
  if (stagger_cycles) {
    const long long until =
        clock64() + (long long)((unsigned long long)blockIdx.x * stagger_cycles / gridDim.x);
    while (clock64() < until)
      __nanosleep(200);
  }

  // ring state.  Consumers (all threads, uniform): slot / parity of the next
  // chunk.  Producer (thread 0): step and chunk-in-step of the next chunk to
  // request, its slot, and the parity of the release it must see first.
  uint32_t c_slot = 0, c_par = 0;
  uint32_t p_slot = 0, p_par = 1, p_step = 0, p_idx = 0;
  // a fresh mbarrier passes a wait on parity 1: the first round needs no release
  auto produce = [&]() {
    if (p_step >= n)
      return;
    mbar_wait_parity(&sm.empty[p_slot], p_par);
    const uint32_t c = p_idx >> 4, sp = (p_idx >> 2) & 3, q4 = p_idx & 3;
    const cplx *src = bsk + n8192_key_offset(p_step, sp >> 1, sp & 1, c, 4 * q4, 0);
    mbar_arrive_expect_tx(&sm.full[p_slot], P8K_CHUNK * sizeof(cplx));
    tma_bulk_g2s(&sm.ring[p_slot][0], src, P8K_CHUNK * sizeof(cplx), &sm.full[p_slot]);
    if (++p_slot == P8K_SLOTS) {
      p_slot = 0;
      p_par ^= 1u;
    }
    if (++p_idx == 32) {
      p_idx = 0;
      do
        p_step++;
      while (p_step < n && sm.a_hat[p_step] == 0);
    }
  };

  for (uint32_t s = blockIdx.x; s < num_samples; s += gridDim.x) {
    // ---- prologue: modulus switch, acc = LUT * X^{-b_hat} -------------------
    const uint64_t *ct = lwe_in + in_idx[s] * (uint64_t)(n + 1);
    if (t == 0) {
      sm.red_half = 0;
      sm.red_dbl = 0;
    }
    __syncthreads();
    {
      CenteredMsSums sums;
      for (uint32_t i = t; i < n; i += 256) {
        const uint64_t a = ct[i];
        sm.a_hat[i] = (uint16_t)modulus_switch_u64(a, log_mod);
        if (centered_ms)
          sums.add(a, log_mod);
      }
      if (centered_ms)
        centered_ms_publish_atomic(sums, &sm.red_half, &sm.red_dbl);
    }
    __syncthreads();
    if (t == 0) {
      // the key of the first steps starts to stream under the rest of the prologue
      p_step = 0;
      p_idx = 0;
      while (p_step < n && sm.a_hat[p_step] == 0)
        p_step++;
      for (int f = 0; f < P8K_SLOTS; f++)
        produce();
      sm.b_hat = ms_b_hat(ct[n], centered_ms, &sm.red_half, &sm.red_dbl, 1, log_mod);
    }
    __syncthreads();
    rotate_lut(&sm.acc[0][0], P8K_N, luts + lut_idx[s] * (uint64_t)(2 * P8K_N), 2,
               P8K_N, sm.b_hat, t, 256, Torus64To32());
    __syncthreads();

    // ---- blind rotation ---------------------------------------------------------
    bool first_chunk = true; // of this sample: the ring is full, nothing to refill yet
    for (uint32_t i = 0; i < n; i++) {
      const uint32_t a = sm.a_hat[i];
      if (a == 0)
        continue; // uniform across the CTA
      // forward: spectrum sp = 2 lvl + r is parked in slot sp
#pragma unroll 1
      for (uint32_t r = 0; r < 2; r++) {
        cplx v[16];
        {
          uint32_t packed[16];
          n8192_load_digits2(sm.acc[r], t, a, base_log, ties_even != 0, v, packed);
          park_words16(park_slot(pk, 2 + r), packed);
        }
        n8192_forward_v2(v, sm.xbuf, t, tables);
        park16(park_slot(pk, r), v);
        {
          uint32_t packed[16];
          fetch_words16(park_slot(pk, 2 + r), packed);
          n8192_unpack_digits(packed, v);
        }
        n8192_forward_v2(v, sm.xbuf, t, tables);
        park16(park_slot(pk, 2 + r), v);
      }
      // per output column: Fourier MAC (thread-local, key from the ring),
      // inverse, accumulate
#pragma unroll 1
      for (uint32_t c = 0; c < 2; c++) {
        cplx out[16];
        cplx tw3[15];
#pragma unroll
        for (int sp = 0; sp < 4; sp++) {
          cplx f[16];
          fetch16(park_slot(pk, sp), f);
          if (sp == 3)
            n8192_load_tw(&tables->pass3[t][0], tw3);
#pragma unroll
          for (int q4 = 0; q4 < 4; q4++) {
            mbar_wait_parity(&sm.full[c_slot], c_par);
            const cplx *ks = &sm.ring[c_slot][t];
#pragma unroll
            for (int bq = 0; bq < 4; bq++) {
              const cplx kv = ks[bq * 256];
              out[4 * q4 + bq] = sp == 0 ? cmul(f[4 * q4 + bq], kv)
                                         : cfma(f[4 * q4 + bq], kv, out[4 * q4 + bq]);
            }
            if (ALL_ARRIVE) {
              // the loads above are still in flight when a bare arrive issues
              mbar_arrive_after_reads(&sm.empty[c_slot]);
            } else {
              // no fence: in the compiled kernel lane 0's arrive issues after
              // the warp's DMULs that wait on these loads, so they are done.
              // That is the schedule, not a guarantee of the source;
              // tests/test_gpu_replay_words.py would see a late read.
              __syncwarp();
              if ((t & 31) == 0)
                mbar_arrive(&sm.empty[c_slot]);
            }
            if (++c_slot == P8K_SLOTS) {
              c_slot = 0;
              c_par ^= 1u;
            }
            if (t == 0) {
              if (!first_chunk)
                produce(); // refills the slot released one chunk ago
            }
            first_chunk = false;
          }
        }
        n8192_inverse_v2(out, tw3, sm.xbuf, t, tables);
        uint32_t *acc_c = sm.acc[c];
#pragma unroll
        for (int j1 = 0; j1 < 16; j1++) {
          const uint32_t j = 256u * j1 + (uint32_t)t;
          acc_c[j] += scaled_double_to_torus32(out[j1].re);
          acc_c[j + P8K_M] += scaled_double_to_torus32(out[j1].im);
        }
      }
      __syncthreads(); // accumulator complete before the next step's rotated reads
    }
    __syncthreads();

    // ---- epilogue: sample extract, optional many-LUT ---------------------------
    sample_extract_many_lut(lwe_out, out_idx[s], num_samples, num_many_lut, lut_stride,
                            &sm.acc[0][0], P8K_N, 1, P8K_N, t, 256, Torus32To64());
    __syncthreads(); // the working set is reused by the next sample
  }
}

// ---------------------------------------------------------------------------
// BSK conversion: standard-domain u64 polynomial, source order
// [i][level slot][row r][column c][N] -> spectrum scaled by 2^-64 / 4096 * 2^32
// at [i][level slot][r][c][b][t3].  grid = #polynomials, block = 256.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
bsk_convert_n8192_kernel(cplx *__restrict__ dst, const uint64_t *__restrict__ src,
                         const Fft4096Tables *__restrict__ tables) {
  extern __shared__ __align__(16) unsigned char conv_smem[]; // 64 KiB (dynamic: above the static limit)
  cplx *xbuf = reinterpret_cast<cplx *>(conv_smem);
  const int t = threadIdx.x;
  const uint64_t *p = src + (size_t)blockIdx.x * P8K_N;
  const double scale = P8K_KEY_SCALE; // 2^-44
  cplx v[16];
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    const uint32_t j = 256u * j1 + t;
    v[j1] = cmake(ll_to_double((int64_t)p[j]) * scale,
                  ll_to_double((int64_t)p[j + P8K_M]) * scale);
  }
  n8192_forward(v, xbuf, t, tables);
  // blockIdx.x = ((i * 2 + level slot) * 2 + r) * 2 + c: the source order
  const uint32_t poly = blockIdx.x;
#pragma unroll
  for (int b = 0; b < 16; b++)
    dst[n8192_key_offset(poly >> 3, (poly >> 2) & 1, (poly >> 1) & 1, poly & 1, b, t)] = v[b];
}

} // namespace b200
