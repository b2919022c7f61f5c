// pbs_multibit_n2048.cuh -- sm_90a multi-bit PBS kernel for (N = 2048, k = 1,
// l <= 2, grouping factor <= 4), e.g. PARAM_MULTI_BIT_GROUP_3_MESSAGE_2_CARRY_2 and
// PARAM_GPU_MULTI_BIT_GROUP_4_MESSAGE_2_CARRY_2 (the reference's GPU default).
//
// Replaces the reference's keybundle + accumulate kernel pairs
// (backends/tfhe-cuda-backend/cuda/src/pbs/programmable_bootstrap_multibit.cuh:
// 30-430, _cg_multibit, _tbc_multibit), which materialise the per-sample key
// bundle in HBM.  Here one persistent CTA per LWE keeps
//   * the GLWE accumulator in REGISTERS (32 u32 words per thread: the
//     multi-bit loop has no rotation, every thread only ever touches its own
//     coefficients; and the accumulator is re-assigned, not accumulated, each
//     step, so 32 bits carry no error build-up),
//   * the l*(k+1) digit spectra in shared memory,
// and folds the bundle into the Fourier MAC (pbs_multibit_n2048_phases.cuh),
// streaming the 2^g GGSWs of the step with coalesced 128-bit L2 loads.
//
// Fourier key layout for this kernel (complex128):
//   [group][column c][slot b < 16][level idx][row r][ggsw s][t < 64]
#pragma once
#include "pbs_multibit_n2048_phases.cuh"
#include "pbs_n2048.cuh"
#include "tma_bulk.cuh"

namespace b200 {

struct MbSmem {
  cplx sp[2][2][P22_M]; // [level idx][row] parked spectra            64 KiB
  cplx xa[2][P22_M];    // per-group exchange buffer / MAC staging    32 KiB
  cplx zeta[16];
  uint32_t degs[16];
  uint32_t b_hat;
};

__host__ __device__ inline size_t mb_key_row(uint32_t grp, uint32_t c,
                                             uint32_t b, uint32_t lvl,
                                             uint32_t r, uint32_t s,
                                             uint32_t l, uint32_t nggsw) {
  return ((((((size_t)grp * 2 + c) * 16 + b) * l + lvl) * 2 + r) * nggsw + s) *
         64;
}

// tables re-read (not kept live) around the MAC: the registers they would hold
// carry the double-buffered key rows there.  volatile: one load per call.
__device__ __forceinline__ cplx mb_ld_table(const cplx *p) {
  cplx v;
  asm volatile("ld.global.nc.v2.f64 {%0, %1}, [%2];"
               : "=d"(v.re), "=d"(v.im)
               : "l"(p));
  return v;
}

struct MbSlotRows {
  const cplx *key_c; // rows of (grp, c, slot 0)
  size_t slot_stride;
  __device__ __forceinline__ const cplx *operator()(int b) const {
    return key_c + (size_t)b * slot_stride;
  }
};
struct MbOutSlot {
  cplx *xa_g;
  int t;
  __device__ __forceinline__ void operator()(int b, cplx v) const {
    xa_g[b * 64 + t] = v;
  }
};

// ---------------------------------------------------------------------------
// Low-latency mode (launches of at most one CTA per SM): the fused kernel above
// spends 2^g * l * 2 key rows per spectrum slot in every step of the ONE CTA
// that owns an LWE -- fine when two CTAs per SM keep the machine busy, pure
// latency when a handful do.  For small batches the bundle
//   bundle[s][grp] = sum_sigma GGSW_{grp,sigma} * X^{deg_sigma(s, grp)}
// is instead built for ALL groups at once by a grid that covers the whole GPU
// (mb_bundle_kernel: steps x 2 columns x 4 slot quads CTAs, key rows streamed
// once per chunk of samples) into a stream-ordered workspace, and the
// sequential part (pbs_multibit_seq_kernel) only does
// the n/g external products against its per-sample bundle: 2*l key rows per
// slot instead of 2^g*l*2.  Same split as the reference's keybundle +
// accumulate kernel pairs (programmable_bootstrap_multibit.cuh:30-430), with
// the bundle in this engine's spectrum order.
//
// bundle layout: [sample][group][level idx][column c][row r][b < 16][t < 64]
// ---------------------------------------------------------------------------
__host__ __device__ inline size_t mb_bundle_row(uint32_t s, uint32_t grp,
                                                uint32_t lvl, uint32_t c,
                                                uint32_t r, uint32_t steps,
                                                uint32_t l) {
  return (((((size_t)s * steps + grp) * l + lvl) * 2 + c) * 2 + r) * P22_M;
}

constexpr int MB_BUNDLE_CHUNK = 16; // samples whose degrees are staged together

// grid = (n/g groups, 2 columns, 4 slot quads), block = 256: thread (b, t) owns
// one spectrum slot of one (group, column).  When the 2^g * l * 2 key values of
// a slot fit in registers (<= 32 complex: every reference set except g = 4 with
// l = 2) they are loaded ONCE per launch and every sample's bundle entry is a
// short chain of table look-ups and complex FMAs on them: the key is streamed
// once whatever the batch, the only per-sample traffic is the 2*l values written.
template <int GROUPING, int L>
__global__ void __launch_bounds__(256)
mb_bundle_kernel(cplx *__restrict__ bundle, const cplx *__restrict__ bsk,
                 const cplx *__restrict__ root,
                 const cplx *__restrict__ mono_tab,
                 const uint64_t *__restrict__ lwe_in,
                 const uint64_t *__restrict__ in_idx, uint32_t n,
                 uint32_t num_samples) {
  constexpr uint32_t nggsw = 1u << GROUPING;
  constexpr int S = MB_BUNDLE_CHUNK;
  constexpr bool KEY_IN_REGS = nggsw * L * 2 <= 32;
  __shared__ cplx zeta[16];
  __shared__ uint32_t degs[S][nggsw];
  const int tid = threadIdx.x;
  const int t = tid & 63;
  const uint32_t b = 4 * blockIdx.z + (tid >> 6);
  const uint32_t grp = blockIdx.x, c = blockIdx.y;
  const uint32_t steps = gridDim.x;
  const uint32_t rb = mb_bitrev4(b);
  if (tid < 16)
    zeta[tid] = root[(256u * tid) & (2 * P22_N - 1)];
  const cplx *rows = bsk + mb_key_row(grp, c, b, 0, 0, 0, L, nggsw) + t;
  auto key = [&](uint32_t sigma, int lvl, int r) {
    return ldcg_cplx(rows + ((size_t)(lvl * 2 + r) * nggsw + sigma) * 64);
  };
  cplx kreg[KEY_IN_REGS ? nggsw : 1][L][2];
  if constexpr (KEY_IN_REGS) {
#pragma unroll
    for (uint32_t sigma = 0; sigma < nggsw; sigma++)
#pragma unroll
      for (int lvl = 0; lvl < L; lvl++)
#pragma unroll
        for (int r = 0; r < 2; r++)
          kreg[sigma][lvl][r] = key(sigma, lvl, r);
  }
  for (uint32_t s0 = 0; s0 < num_samples; s0 += S) {
    __syncthreads();
    for (uint32_t w = tid; w < S * nggsw; w += 256) {
      const uint32_t ss = w / nggsw, sigma = w % nggsw;
      if (s0 + ss < num_samples && sigma) {
        const uint64_t *ct = lwe_in + in_idx[s0 + ss] * (uint64_t)(n + 1);
        uint64_t sum = 0;
#pragma unroll
        for (uint32_t u = 0; u < GROUPING; u++)
          if ((sigma >> (GROUPING - 1 - u)) & 1u)
            sum += ct[grp * GROUPING + u];
        degs[ss][sigma] = modulus_switch_u64(sum, 12);
      }
    }
    __syncthreads();
    const uint32_t cnt = min((uint32_t)S, num_samples - s0);
    for (uint32_t ss = 0; ss < cnt; ss++) {
      cplx acc[L][2];
      mb_bundle_entry<nggsw, L>(
          [&](uint32_t sigma, int lvl, int r) {
            if constexpr (KEY_IN_REGS)
              return kreg[sigma][lvl][r];
            else
              return key(sigma, lvl, r);
          },
          [&](uint32_t deg) { return mono_tab[(size_t)deg * 64 + t]; }, zeta,
          degs[ss], rb, acc);
#pragma unroll
      for (int lvl = 0; lvl < L; lvl++)
#pragma unroll
        for (int r = 0; r < 2; r++)
          bundle[mb_bundle_row(s0 + ss, grp, lvl, c, r, steps, L) + b * 64 + t] =
              acc[lvl][r];
    }
  }
}

template <int GROUPING, int L>
__global__ void __launch_bounds__(128, 2)
pbs_multibit_n2048_k1_kernel(uint64_t *__restrict__ lwe_out,
                             const uint64_t *__restrict__ out_idx,
                             const uint64_t *__restrict__ luts,
                             const uint64_t *__restrict__ lut_idx,
                             const uint64_t *__restrict__ lwe_in,
                             const uint64_t *__restrict__ in_idx,
                             const cplx *__restrict__ bsk,
                             const Fft1024Tables *__restrict__ tables,
                             const cplx *__restrict__ root,
                             const cplx *__restrict__ mono_tab, uint32_t n,
                             uint32_t base_log, uint32_t num_many_lut,
                             uint32_t lut_stride, int ties_even) {
  constexpr uint32_t grouping = GROUPING;
  constexpr uint32_t l = L;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  MbSmem &sm = *reinterpret_cast<MbSmem *>(smem_raw);
  const int tid = threadIdx.x;
  const int g = tid >> 6;
  const int t = tid & 63;
  const uint32_t s_idx = blockIdx.x;
  const uint32_t log_mod = 12;
  constexpr uint32_t nggsw = 1u << GROUPING;
  const uint32_t steps = n / grouping;
  const uint64_t *ct = lwe_in + in_idx[s_idx] * (uint64_t)(n + 1);

  if (tid == 0)
    sm.b_hat = modulus_switch_u64(ct[n], log_mod);
  if (tid < 16)
    sm.zeta[tid] = root[(256u * tid) & (2 * P22_N - 1)];
  __syncthreads();

  // accumulator: this thread's 32 coefficients of polynomial g of LUT*X^-b_hat
  uint32_t acc_lo[16], acc_hi[16];
  {
    const uint64_t *lut =
        luts + lut_idx[s_idx] * (uint64_t)(2 * P22_N) + (size_t)g * P22_N;
    const uint32_t b_hat = sm.b_hat;
#pragma unroll
    for (int j1 = 0; j1 < 16; j1++) {
      const uint32_t j = 64u * j1 + (uint32_t)t;
      acc_lo[j1] = torus64_to_32(rot_div_coeff(lut, P22_N, j, b_hat));
      acc_hi[j1] = torus64_to_32(rot_div_coeff(lut, P22_N, j + P22_M, b_hat));
    }
  }
  const cplx *tw2_src = &tables->pass2[t >> 2][0];
  const cplx *tw3_src = &tables->pass3[t][0];

  cplx *xa_g = sm.xa[g];
  const cplx *sp = &sm.sp[0][0][0];

  for (uint32_t grp = 0; grp < steps; grp++) {
    // degrees of the rotated GGSWs (selection bit of mask element u is bit
    // g-1-u of s), standard modulus switch of the selected sum
    if (tid >= 1 && tid < (int)nggsw) {
      uint64_t sum = 0;
#pragma unroll
      for (uint32_t u = 0; u < grouping; u++)
        if (((uint32_t)tid >> (grouping - 1 - u)) & 1u)
          sum += ct[grp * grouping + u];
      sm.degs[tid] = modulus_switch_u64(sum, log_mod);
    }
    cplx v[16];
    {
      cplx tw2[3], tw3[15];
#pragma unroll
      for (int e = 0; e < 3; e++)
        tw2[e] = mb_ld_table(tw2_src + e);
#pragma unroll
      for (int e = 0; e < 15; e++)
        tw3[e] = mb_ld_table(tw3_src + e);
#pragma unroll
      for (uint32_t lvl = 0; lvl < l; lvl++) {
        mb_load_digits(acc_lo, acc_hi, base_log, l, lvl, v, ties_even != 0);
        radix16_fwd(v, c_fft1024_pass1);
        x1_store_p1(xa_g, t, v);
        group_barrier(g);
        x1_load_p2(xa_g, t, v);
        group_barrier(g);
        pass2_fwd(v, tw2);
        x2_store_p2(xa_g, t, v);
        x2_sync(g); // exchange 2 is local to 4 adjacent lanes
        x2_load_p3(xa_g, t, v);
        group_barrier(g);
        radix16_fwd(v, tw3);
        spec_store(&sm.sp[lvl][g][0], t, v);
      }
    }
    __syncthreads();

    // Fourier MAC with the bundle folded in; results staged in xa_g
    {
      cplx mono_base[nggsw - 1];
#pragma unroll
      for (uint32_t s = 1; s < nggsw; s++)
        mono_base[s - 1] = mono_tab[(size_t)sm.degs[s] * 64 + t];
      MbSlotRows rows{bsk + mb_key_row(grp, g, 0, 0, 0, 0, l, nggsw),
                      (size_t)l * 2 * nggsw * 64};
      mb_mac_step<(int)nggsw, L>(sp, mono_base, sm.zeta, sm.degs, t,
                                 LdcgLoader(), rows, MbOutSlot{xa_g, t});
    }
    __syncthreads(); // every read of sp / degs done before the next step
#pragma unroll
    for (int b = 0; b < 16; b++)
      v[b] = xa_g[b * 64 + t];
    group_barrier(g);
    {
      cplx tw2[3], tw3[15];
#pragma unroll
      for (int e = 0; e < 3; e++)
        tw2[e] = mb_ld_table(tw2_src + e);
#pragma unroll
      for (int e = 0; e < 15; e++)
        tw3[e] = mb_ld_table(tw3_src + e);
      radix16_inv(v, tw3);
      x2_store_p3(xa_g, t, v);
      x2_sync(g);
      x2_load_p2(xa_g, t, v);
      group_barrier(g);
      pass2_inv(v, tw2);
      x1_store_p2(xa_g, t, v);
      group_barrier(g);
      x1_load_p1(xa_g, t, v);
      radix16_inv(v, c_fft1024_pass1);
    }
    mb_acc_assign(acc_lo, acc_hi, v);
    group_barrier(g);
  }

  // epilogue: spill the accumulator to shared memory once, sample extract
  __syncthreads();
  uint32_t *acc_s = reinterpret_cast<uint32_t *>(&sm.sp[0][0][0]);
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    acc_s[g * P22_N + 64 * j1 + t] = acc_lo[j1];
    acc_s[g * P22_N + 64 * j1 + t + P22_M] = acc_hi[j1];
  }
  __syncthreads();
  sample_extract_many_lut(lwe_out, out_idx[s_idx], gridDim.x, num_many_lut, lut_stride,
                          acc_s, P22_N, 1, P22_N, tid, 128, Torus32To64());
}

// ---------------------------------------------------------------------------
// Sequential part of the low-latency mode: one CTA per LWE (one per SM), the
// n/g external products against the per-sample bundle written by
// mb_bundle_kernel.  Built for latency: accumulator in registers, pass-2/3
// twiddles in registers for the whole loop, two exchange buffers (one named
// barrier per exchange), the bundle rows of a step requested before the share
// barrier in chunks of 16 values, double buffered, MAC results straight into the
// transform registers.  6 barriers per step for l = 1.
// ---------------------------------------------------------------------------
struct MbSeqSmem {
  cplx sp[2][2][P22_M]; // [level idx][row] parked spectra            64 KiB
  cplx xa[2][P22_M];    // exchange 1                                 32 KiB
  cplx xb[2][P22_M];    // exchange 2                                 32 KiB
  uint32_t b_hat;
};
// TMA variant (l = 1): the 64 KiB bundle block of a step -- [column][row][1024]
// complex, contiguous -- is brought into a 2-slot shared-memory ring by
// cp.async.bulk a whole step ahead (one elected thread, mbarrier complete_tx),
// so no key value is ever waited for and no register holds one across the
// share barrier; the MAC reads spectra and key from shared memory.
struct MbSeqSmemTma {
  cplx ring[2][4][P22_M]; // [slot][column * 2 + row]                 128 KiB
  cplx sp[1][2][P22_M];   //                                           32 KiB
  cplx xa[2][P22_M];      //                                           32 KiB
  cplx xb[2][P22_M];      //                                           32 KiB
  unsigned long long bar[2];
  uint32_t b_hat;
};

template <int L, bool TMA = false>
__global__ void __launch_bounds__(128, 1)
pbs_multibit_seq_kernel(uint64_t *__restrict__ lwe_out,
                        const uint64_t *__restrict__ out_idx,
                        const uint64_t *__restrict__ luts,
                        const uint64_t *__restrict__ lut_idx,
                        const uint64_t *__restrict__ lwe_in,
                        const uint64_t *__restrict__ in_idx,
                        const cplx *__restrict__ bundle,
                        const Fft1024Tables *__restrict__ tables, uint32_t n,
                        uint32_t steps, uint32_t base_log,
                        uint32_t num_many_lut, uint32_t lut_stride,
                        int ties_even) {
  static_assert(!TMA || L == 1, "the bulk-copy ring is sized for l = 1");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using Smem = typename std::conditional<TMA, MbSeqSmemTma, MbSeqSmem>::type;
  Smem &sm = *reinterpret_cast<Smem *>(smem_raw);
  const int tid = threadIdx.x;
  const int g = tid >> 6;
  const int t = tid & 63;
  const uint32_t s_idx = blockIdx.x;
  const uint64_t *ct = lwe_in + in_idx[s_idx] * (uint64_t)(n + 1);
  [[maybe_unused]] auto tma_issue = [&](uint32_t grp) {
    if constexpr (TMA) {
      // 4 x 16 KiB: [column][row] of (sample, group grp)
      const cplx *src = bundle + mb_bundle_row(s_idx, grp, 0, 0, 0, steps, 1);
      unsigned long long *bar = &sm.bar[grp & 1];
      mbar_arrive_expect_tx(bar, 4u * P22_M * (uint32_t)sizeof(cplx));
#pragma unroll
      for (int q = 0; q < 4; q++)
        tma_bulk_g2s(&sm.ring[grp & 1][q][0], src + (size_t)q * P22_M,
                     P22_M * (uint32_t)sizeof(cplx), bar);
    }
  };
  if (tid == 0) {
    sm.b_hat = modulus_switch_u64(ct[n], 12);
    if constexpr (TMA) {
      mbar_init(&sm.bar[0], 1);
      mbar_init(&sm.bar[1], 1);
      mbar_fence_init();
    }
  }
  __syncthreads();
  if constexpr (TMA)
    if (tid == 0)
      tma_issue(0);
  uint32_t acc_lo[16], acc_hi[16];
  {
    const uint64_t *lut =
        luts + lut_idx[s_idx] * (uint64_t)(2 * P22_N) + (size_t)g * P22_N;
    const uint32_t b_hat = sm.b_hat;
#pragma unroll
    for (int j1 = 0; j1 < 16; j1++) {
      const uint32_t j = 64u * j1 + (uint32_t)t;
      acc_lo[j1] = torus64_to_32(rot_div_coeff(lut, P22_N, j, b_hat));
      acc_hi[j1] = torus64_to_32(rot_div_coeff(lut, P22_N, j + P22_M, b_hat));
    }
  }
  cplx tw2[3], tw3[15];
#pragma unroll
  for (int e = 0; e < 3; e++)
    tw2[e] = tables->pass2[t >> 2][e];
#pragma unroll
  for (int e = 0; e < 15; e++)
    tw3[e] = tables->pass3[t][e];
  cplx *xa_g = sm.xa[g], *xb_g = sm.xb[g];
  const cplx *sp = &sm.sp[0][0][0];
  constexpr int CH_SLOTS = 8 / L;       // spectrum slots per chunk
  constexpr int CH_VALS = CH_SLOTS * L * 2; // = 16 key values per chunk
  constexpr int NCH = 16 / CH_SLOTS;

  for (uint32_t grp = 0; grp < steps; grp++) {
    cplx v[16];
    if constexpr (TMA) {
      // next step's block into the other slot: its last readers (the MAC of
      // step grp - 1) are behind the CTA barrier that ended that MAC
      if (tid == 0 && grp + 1 < steps)
        tma_issue(grp + 1);
    }
#pragma unroll
    for (uint32_t lvl = 0; lvl < (uint32_t)L; lvl++) {
      mb_load_digits(acc_lo, acc_hi, base_log, L, lvl, v, ties_even != 0);
      radix16_fwd(v, c_fft1024_pass1);
      x1_store_p1(xa_g, t, v);
      group_barrier(g);
      x1_load_p2(xa_g, t, v);
      pass2_fwd(v, tw2);
      x2_store_p2(xb_g, t, v);
      x2_sync(g);
      x2_load_p3(xb_g, t, v);
      radix16_fwd(v, tw3);
      spec_store(&sm.sp[lvl][g][0], t, v);
    }
    if constexpr (TMA) {
      __syncthreads();
      mbar_wait_parity(&sm.bar[grp & 1], (grp >> 1) & 1u);
      const cplx *k0 = &sm.ring[grp & 1][2 * g][0], *k1 = &sm.ring[grp & 1][2 * g + 1][0];
      // the same two-FMA chain from zero as the register-prefetch branch below:
      // the multi-bit accumulator is RE-ASSIGNED from f64 every step, so one
      // differently rounded product can flip a digit of the next step and the
      // outputs then differ by a fresh encryption of zero -- still correct, but
      // not the word-for-word agreement between the schedules that
      // test_reference_golden_keyset_on_gpu asserts
#pragma unroll
      for (int b = 0; b < 16; b++)
        v[b] = cfma(sp[(size_t)(16 + b) * 64 + t], k1[b * 64 + t],
                    cfma(sp[(size_t)b * 64 + t], k0[b * 64 + t],
                         cmake(0.0, 0.0)));
    } else {
    // column g of this sample's bundle for this step: [lvl][c][r][1024]
    const cplx *bun_c = bundle + mb_bundle_row(s_idx, grp, 0, (uint32_t)g, 0, steps, L);
    cplx kv[2][CH_VALS];
    auto issue = [&](int ch, cplx *dst) {
#pragma unroll
      for (int bb = 0; bb < CH_SLOTS; bb++)
#pragma unroll
        for (int lvl = 0; lvl < L; lvl++)
#pragma unroll
          for (int r = 0; r < 2; r++)
            dst[(bb * L + lvl) * 2 + r] =
                ldcg_cplx(bun_c + ((size_t)lvl * 4 + r) * P22_M +
                          (ch * CH_SLOTS + bb) * 64 + t);
    };
    issue(0, kv[0]); // in flight across the barrier
    issue(1, kv[1]);
    __syncthreads();
#pragma unroll
    for (int ch = 0; ch < NCH; ch++) {
#pragma unroll
      for (int bb = 0; bb < CH_SLOTS; bb++) {
        const int b = ch * CH_SLOTS + bb;
        cplx out = cmake(0.0, 0.0);
#pragma unroll
        for (int lvl = 0; lvl < L; lvl++)
#pragma unroll
          for (int r = 0; r < 2; r++)
            out = cfma(sp[((size_t)(lvl * 2 + r) * 16 + b) * 64 + t],
                       kv[ch & 1][(bb * L + lvl) * 2 + r], out);
        v[b] = out;
      }
      if (ch + 2 < NCH)
        issue(ch + 2, kv[ch & 1]);
    }
    }
    __syncthreads(); // every read of sp done before the next step overwrites it
    radix16_inv(v, tw3);
    x2_store_p3(xb_g, t, v);
    x2_sync(g);
    x2_load_p2(xb_g, t, v);
    pass2_inv(v, tw2);
    x1_store_p2(xa_g, t, v);
    group_barrier(g);
    x1_load_p1(xa_g, t, v);
    radix16_inv(v, c_fft1024_pass1);
    mb_acc_assign(acc_lo, acc_hi, v);
  }

  __syncthreads();
  uint32_t *acc_s = reinterpret_cast<uint32_t *>(&sm.sp[0][0][0]);
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++) {
    acc_s[g * P22_N + 64 * j1 + t] = acc_lo[j1];
    acc_s[g * P22_N + 64 * j1 + t + P22_M] = acc_hi[j1];
  }
  __syncthreads();
  sample_extract_many_lut(lwe_out, out_idx[s_idx], gridDim.x, num_many_lut, lut_stride,
                          acc_s, P22_N, 1, P22_N, tid, 128, Torus32To64());
}

// key conversion into the layout above.  grid = #source polynomials
// ([ggsw = grp*2^g + s][level idx][row r][col c][N]), block = 64.
__global__ void __launch_bounds__(64)
bsk_convert_multibit_n2048_kernel(cplx *__restrict__ dst,
                                  const uint64_t *__restrict__ src,
                                  const Fft1024Tables *__restrict__ tables,
                                  uint32_t l, uint32_t grouping) {
  __shared__ cplx xa[P22_M];
  __shared__ cplx xb[P22_M];
  const int t = threadIdx.x;
  const uint32_t nggsw = 1u << grouping;
  uint32_t poly = blockIdx.x;
  const uint32_t c = poly & 1;
  poly >>= 1;
  const uint32_t r = poly & 1;
  poly >>= 1;
  const uint32_t lvl = poly % l;
  poly /= l;
  const uint32_t s = poly & (nggsw - 1), grp = poly >> grouping;
  const uint64_t *p = src + (size_t)blockIdx.x * P22_N;
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
#pragma unroll
  for (int b = 0; b < 16; b++)
    dst[mb_key_row(grp, c, b, lvl, r, s, l, nggsw) + t] = v[b];
}

} // namespace b200
