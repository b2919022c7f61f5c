// pbs_n2048_lanepair.cuh -- the CMUX step of the lane-pair layout of the
// N = 2048 classic PBS (the shipped two-CTA instance,
// pbs_n2048_k1_l1_v6_kernel<2, true, 2, 1, X2>) as per-thread pieces.  The
// kernel's loop (p22_lanepair_loop, pbs_n2048.cuh), the phase-clock tool
// (tools/micro/phase_clocks.cu) and the CPU replay (tests/emu/emu_lanepair.cpp)
// all run these pieces, so they run the same step.
//
// Thread map: lane l of warp w runs thread t = 16 w + (l & 15) of polynomial
// g = l >> 4, so lanes l and l ^ 16 hold the same spectrum slots 16 t + b of the
// two polynomials after the forward transform.
//
// The step is cut wherever a thread needs another thread's data: the CTA
// barriers around exchange 1 (x1h_*), exchange 2 in both directions (a warp
// exchange: x2m_* through the warp's own rows, or x2h_* shuffles), the MAC's
// partner value from lane l ^ 16, the wait for the ring's key block, and the
// barrier after the accumulator update.  The pieces are named after the phases
// of the step, as the phase-clock tool prints them (DESIGN §10); the caller
// runs what lies between them.
#pragma once
#include "pbs_n2048_phases.cuh"
#include "x2_shfl.cuh"
#include "x2_smem.cuh"

#include <stddef.h>

namespace b200 {

// The rows of acc are 16 words apart modulo the 32 banks: in the lane-pair
// layout a warp reads and writes the same 16 coefficients of both polynomials,
// and the two halves then hit disjoint banks.
constexpr int P22_ACC_STRIDE = P22_N + 16;

B200_HD int p22lp_g(int tid) { return (tid >> 4) & 1; }
B200_HD int p22lp_t(int tid) { return ((tid >> 5) << 4) | (tid & 15); }

// Key block of step i: [column c][row r][16][64] complex, blocks 2c + r.  The
// other rows, blocks 1 (column 0, row 1) and 2 (column 1, row 0), are adjacent:
// one copy into the two-slot ring, where column g finds its other row in slot g.
constexpr uint32_t P22_RING_BYTES = 2u * P22_M * (uint32_t)sizeof(cplx);
B200_HD const cplx *p22_ring_src(const cplx *bsk, uint32_t i) {
  return bsk + (size_t)i * (4 * P22_M) + P22_M;
}

// L2-only 128-bit load of a key value (a plain load on the host)
B200_HD cplx ldcg_cplx(const cplx *p) {
#if defined(__CUDA_ARCH__)
  const double2 v = __ldcg(reinterpret_cast<const double2 *>(p));
  return cmake(v.x, v.y);
#else
  return *p;
#endif
}

// One thread of the step: where its data lives, and the phases it runs.
struct P22LanePair {
  int g, t;
  uint32_t *acc_g;     // accumulator row of polynomial g
  cplx *xa_g;          // exchange-1 buffer of polynomial g
  cplx *x2_rows;       // rows 4 w .. 4 w + 3 of xa_g: warp w's alone from
                       // x1_fwd_load to x1_inv_store
  const cplx *k_oth;   // ring slot of row 1 - g of column g
  const cplx *bsk_own; // row g of column g, element t, in the key block of step 0
  const cplx *pass1, *tw2, *tw3; // twiddles of the three passes

  // the two accumulator rows, exchange-1 buffers and ring slots
  B200_HD P22LanePair(int tid, uint32_t (*acc)[P22_ACC_STRIDE], cplx (*xa)[P22_M],
                      const cplx (*ring)[P22_M], const cplx *bsk, const cplx *pass1_,
                      const cplx *tw2_, const cplx *tw3_)
      : g(p22lp_g(tid)), t(p22lp_t(tid)), acc_g(acc[g]), xa_g(xa[g]),
        x2_rows(xa_g + 256 * (tid >> 5)), k_oth(ring[g]),
        bsk_own(bsk + (size_t)g * (2 * P22_M) + (size_t)g * P22_M + t), pass1(pass1_),
        tw2(tw2_), tw3(tw3_) {}

  B200_HD void own_init(uint32_t own[32]) const { p22v4_own_init(acc_g, t, own); }

  // digits (rotate + decompose)
  B200_HD void digits(uint32_t a, uint32_t base_log, const uint32_t own[32], cplx v[16]) const {
    p22v4_load_digits<2>(acc_g, t, a, base_log, own, v);
  }
  B200_HD void fwd_pass1(cplx v[16]) const { radix16_fwd(v, pass1); }
  // exchange 1, either side of a CTA barrier
  B200_HD void x1_fwd_store(const cplx v[16]) const { x1h_store_p1(xa_g, t, v); }
  B200_HD void x1_fwd_load(cplx v[16]) const { x1h_load_p2(xa_g, t, v); }
  B200_HD void fwd_pass2(cplx v[16]) const { pass2_fwd(v, tw2); }
  // (exchange 2)
  B200_HD void fwd_pass3(cplx v[16]) const { radix16_fwd(v, tw3); }
  // own-row key load of step i (the other row arrives in the ring)
  B200_HD void own_row_load(uint32_t i, cplx b_own[16]) const {
    const size_t step = (size_t)i * (4 * P22_M);
#pragma unroll
    for (int b = 0; b < 16; b++)
      b_own[b] = ldcg_cplx(bsk_own + step + b * 64);
  }
  // MAC of output column g: F_other * B[1 - g][g] + F_g * B[g][g], where
  // partner(b, v[b]) returns lane l ^ 16's v[b] from before the MAC
  template <typename Partner>
  B200_HD void mac(cplx v[16], const cplx b_own[16], Partner partner) const {
#pragma unroll
    for (int b = 0; b < 16; b++) {
      const cplx o = partner(b, v[b]);
      v[b] = cfma(o, k_oth[b * 64 + t], cmul(v[b], b_own[b]));
    }
  }
  B200_HD void inv_pass3(cplx v[16]) const { radix16_inv(v, tw3); }
  // (inverse exchange 2)
  B200_HD void inv_pass2(cplx v[16]) const { pass2_inv(v, tw2); }
  // inverse exchange 1, either side of a CTA barrier
  B200_HD void x1_inv_store(const cplx v[16]) const { x1h_store_p2(xa_g, t, v); }
  B200_HD void x1_inv_load(cplx v[16]) const { x1h_load_p1(xa_g, t, v); }
  B200_HD void inv_pass1(cplx v[16]) const { radix16_inv(v, pass1); }
  B200_HD void acc_update(const cplx v[16], uint32_t own[32]) const {
    p22v4_acc_update(acc_g, t, v, own);
  }
};

} // namespace b200
