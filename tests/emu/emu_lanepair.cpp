// emu_lanepair.cpp -- CPU replay of the lane-pair layout of the N = 2048
// classic PBS kernel (pbs_n2048_k1_l1_v6_kernel<2, true, 2, 1>).
//
// TEST INFRASTRUCTURE ONLY.  Same B200_HD phase functions as the kernel
// (tfhe-rs_b200/csrc/*.cuh), compiled with g++: 4 warps x 32 lanes, lane l of
// warp w runs thread t = 16 w + (l & 15) of polynomial l >> 4.  Every barrier
// of the kernel is one loop over the 128 threads; the shuffles (half-warp
// exchange 2 and the MAC's partner lane l ^ 16) read the registers of the
// other lanes after every lane has reached them.  The accumulator rows sit
// P22_ACC_STRIDE words apart as in P22SmemV6.
// Compare it with emu_p22.cpp only when both are built with
// -ffp-contract=off: otherwise g++ fuses products and sums wherever the shape
// of the surrounding code lets it, differently in the two files.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../tfhe-rs_b200/csrc/pbs_n2048_phases.cuh"
#include "../../tfhe-rs_b200/csrc/x2_shfl.cuh"

namespace {

constexpr int ACC_STRIDE = P22_N + 16; // P22_ACC_STRIDE of pbs_n2048.cuh

struct Lane {
  cplx v[16];
  uint32_t own[32];
};

int lane_g(int tid) { return (tid >> 4) & 1; }
int lane_t(int tid) { return ((tid >> 5) << 4) | (tid & 15); }

const Fft1024Tables *tables() {
  static Fft1024Tables tb;
  static bool init = false;
  if (!init) {
    b200_fill_fft1024_tables(&tb);
    init = true;
  }
  return &tb;
}

// one warp-wide register exchange: f(warp registers [32][16])
template <typename F> void per_warp(std::vector<Lane> &R, F f) {
  for (int w = 0; w < 4; w++) {
    cplx W[32][16];
    for (int l = 0; l < 32; l++)
      std::memcpy(W[l], R[32 * w + l].v, sizeof(W[l]));
    f(W);
    for (int l = 0; l < 32; l++)
      std::memcpy(R[32 * w + l].v, W[l], sizeof(W[l]));
  }
}

} // namespace

extern "C" {

// one LWE, same arguments as emu_pbs_p22_v3 (tests/emu/emu_p22.cpp); bsk in
// the layout of emu_bsk_convert_p22.  Runs every step, a_hat = 0 included,
// as the kernel does.
void emu_pbs_p22_lanepair(const double *bsk_, const uint64_t *lut, const uint64_t *ct,
                          uint32_t n, uint32_t base_log, int centered_ms,
                          uint32_t num_many_lut, uint32_t lut_stride, uint32_t count,
                          uint64_t *out_base) {
  const cplx *bsk = reinterpret_cast<const cplx *>(bsk_);
  const Fft1024Tables *tb = tables();
  const uint32_t log_mod = 12;
  std::vector<uint32_t> acc(2 * ACC_STRIDE);
  std::vector<cplx> xa(2 * P22_M);
  std::vector<uint16_t> a_hat(n);
  CenteredMsSums sums;
  for (uint32_t i = 0; i < n; i++) {
    a_hat[i] = (uint16_t)modulus_switch_u64(ct[i], log_mod);
    sums.add(ct[i], log_mod);
  }
  const uint32_t b_hat = ms_b_hat(ct[n], centered_ms, &sums.half, &sums.dbl, 1, log_mod);
  rotate_lut(acc.data(), ACC_STRIDE, lut, 2, P22_N, b_hat, 0, 1, Torus64To32());
  std::vector<Lane> R(128);
  auto acc_of = [&](int tid) { return acc.data() + lane_g(tid) * ACC_STRIDE; };
  auto xa_of = [&](int tid) { return xa.data() + lane_g(tid) * P22_M; };
  for (int tid = 0; tid < 128; tid++)
    p22v4_own_init(acc_of(tid), lane_t(tid), R[tid].own);
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t a = a_hat[i];
    for (int tid = 0; tid < 128; tid++) {
      cplx *v = R[tid].v;
      p22v4_load_digits<2>(acc_of(tid), lane_t(tid), a, base_log, R[tid].own, v);
      radix16_fwd(v, tb->pass1);
      x1h_store_p1(xa_of(tid), lane_t(tid), v);
    }
    for (int tid = 0; tid < 128; tid++) {
      x1h_load_p2(xa_of(tid), lane_t(tid), R[tid].v);
      pass2_fwd(R[tid].v, &tb->pass2[x1h_q(lane_t(tid))][0]);
    }
    per_warp(R, [](cplx (*W)[16]) { b200::x2h_fwd_warp(W); });
    for (int tid = 0; tid < 128; tid++)
      radix16_fwd(R[tid].v, tb->pass3[lane_t(tid)]);
    // MAC: column g = F_other * B[1 - g][g] + F_g * B[g][g], F_other from lane l ^ 16
    for (int w = 0; w < 4; w++) {
      cplx V[32][16];
      for (int l = 0; l < 32; l++)
        std::memcpy(V[l], R[32 * w + l].v, sizeof(V[l]));
      for (int l = 0; l < 32; l++) {
        const int tid = 32 * w + l, g = lane_g(tid), t = lane_t(tid);
        const cplx *bsk_ig = bsk + ((size_t)i * 2 + g) * (2 * P22_M);
        for (int b = 0; b < 16; b++) {
          const cplx k_own = bsk_ig[(g * 16 + b) * 64 + t];
          const cplx k_oth = bsk_ig[((1 - g) * 16 + b) * 64 + t];
          R[tid].v[b] = cfma(V[l ^ 16][b], k_oth, cmul(V[l][b], k_own));
        }
      }
    }
    for (int tid = 0; tid < 128; tid++)
      radix16_inv(R[tid].v, tb->pass3[lane_t(tid)]);
    per_warp(R, [](cplx (*W)[16]) { b200::x2h_inv_warp(W); });
    for (int tid = 0; tid < 128; tid++) {
      pass2_inv(R[tid].v, &tb->pass2[x1h_q(lane_t(tid))][0]);
      x1h_store_p2(xa_of(tid), lane_t(tid), R[tid].v);
    }
    for (int tid = 0; tid < 128; tid++) {
      x1h_load_p1(xa_of(tid), lane_t(tid), R[tid].v);
      radix16_inv(R[tid].v, tb->pass1);
      p22v4_acc_update(acc_of(tid), lane_t(tid), R[tid].v, R[tid].own);
    }
  }
  sample_extract_many_lut(out_base, 0, count, num_many_lut, lut_stride, acc.data(),
                          ACC_STRIDE, 1, P22_N, 0, 1, Torus32To64());
}

// Bank-conflict audit of the lane-pair layout.
// which = 0: exchange 1 (x1h_*), 128-bit accesses, every quarter-warp of every
//            access pattern: the worst number of distinct slots that share a
//            16-byte bank group (1 = conflict-free);
// which = 1: accumulator (32-bit) at row stride `acc_stride` words: the rotated
//            reads of rotate + decompose for every rotation, and the own-word
//            reads and writes; per warp, the worst number of distinct words
//            that share a bank (1 = conflict-free).
int emu_lanepair_conflict_audit(int which, int acc_stride) {
  int worst = 1;
  // distinct slots of `lanes` lanes per bank (group) slot % groups
  auto count = [&](const int *slot, int lanes, int groups) {
    int hist[32] = {0};
    for (int y = 0; y < lanes; y++) {
      bool dup = false;
      for (int z = 0; z < y; z++)
        dup = dup || slot[z] == slot[y];
      if (!dup && ++hist[slot[y] % groups] > worst)
        worst = hist[slot[y] % groups];
    }
  };
  if (which == 0) {
    // slot index in complex units: 16 bytes = 4 banks, 8 groups of 4 banks
    for (int w = 0; w < 4; w++)
      for (int quarter = 0; quarter < 4; quarter++)
        for (int reg = 0; reg < 16; reg++) {
          int p1[8], p2[8];
          for (int j = 0; j < 8; j++) {
            const int t = lane_t(32 * w + 8 * quarter + j);
            p1[j] = x1h_slot(reg, t);
            p2[j] = x1h_slot(x1h_q(t), 16 * (reg & 3) + 4 * x1h_bh(t) + (reg >> 2));
          }
          count(p1, 8, 8);
          count(p2, 8, 8);
        }
    return worst;
  }
  for (int w = 0; w < 4; w++)
    for (int j1 = 0; j1 < 16; j1++) {
      int own0[32], own1[32];
      for (int l = 0; l < 32; l++) {
        const int tid = 32 * w + l, base = lane_g(tid) * acc_stride, j = 64 * j1 + lane_t(tid);
        own0[l] = base + j;
        own1[l] = base + j + P22_M;
      }
      count(own0, 32, 32);
      count(own1, 32, 32);
      for (int d = 0; d < P22_N; d++) {
        int r0[32], r1[32];
        for (int l = 0; l < 32; l++) {
          const int tid = 32 * w + l, base = lane_g(tid) * acc_stride;
          const int i0 = (64 * j1 + lane_t(tid) - d) & (P22_N - 1);
          r0[l] = base + i0;
          r1[l] = base + (i0 ^ P22_M);
        }
        count(r0, 32, 32);
        count(r1, 32, 32);
      }
    }
  return worst;
}

} // extern "C"
