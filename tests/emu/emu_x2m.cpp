// emu_x2m.cpp -- CPU replay of exchange 2 through the warp's own rows
// (x2m_*, tfhe-rs_b200/csrc/x2_smem.cuh) in the lane-pair layout of the
// N = 2048 classic PBS kernel (pbs_n2048_k1_l1_v6_kernel<2, true, 2, 1, 1>).
//
// TEST INFRASTRUCTURE ONLY.  The same B200_HD phase functions as the kernel,
// compiled with g++, over 4 warps x 32 lanes as in emu_lanepair.cpp (lane l of
// warp w runs thread t = 16 w + (l & 15) of polynomial l >> 4).  The pass-2
// window of the step runs warp after warp, and exchange 2 goes through the
// warp's rows of the shared exchange-1 buffer: a slot outside those rows would
// corrupt the next warp's exchange-1 loads (forward) or the previous warp's
// exchange-1 stores (inverse), and the replay would no longer match.
// Build with -ffp-contract=off to compare with emu_p22.cpp / emu_lanepair.cpp.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../tfhe-rs_b200/csrc/pbs_n2048_phases.cuh"
#include "../../tfhe-rs_b200/csrc/x2_shfl.cuh"
#include "../../tfhe-rs_b200/csrc/x2_smem.cuh"

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

uint64_t splitmix(uint64_t &s) {
  uint64_t z = (s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

} // namespace

extern "C" {

// x2m_*_warp against x2h_*_warp on one warp of random doubles (random bit
// patterns, NaNs excluded): the number of (lane, register) words that differ.
int emu_x2m_register_check(uint64_t seed) {
  int bad = 0;
  for (int dir = 0; dir < 2; dir++) {
    cplx a[32][16], b[32][16];
    for (int l = 0; l < 32; l++)
      for (int r = 0; r < 16; r++) {
        uint64_t x = splitmix(seed) & ~(1ull << 62), y = splitmix(seed) & ~(1ull << 62);
        std::memcpy(&a[l][r].re, &x, 8);
        std::memcpy(&a[l][r].im, &y, 8);
      }
    std::memcpy(b, a, sizeof(a));
    if (dir == 0) {
      b200::x2h_fwd_warp(a);
      b200::x2m_fwd_warp(b);
    } else {
      b200::x2h_inv_warp(a);
      b200::x2m_inv_warp(b);
    }
    for (int l = 0; l < 32; l++)
      for (int r = 0; r < 16; r++)
        bad += std::memcmp(&a[l][r], &b[l][r], sizeof(cplx)) != 0;
  }
  return bad;
}

// one LWE, same arguments as emu_pbs_p22_lanepair (emu_lanepair.cpp)
void emu_pbs_p22_lanepair_x2m(const double *bsk_, const uint64_t *lut, const uint64_t *ct,
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
  // the rows 4 w .. 4 w + 3 of the lane's buffer (x2_rows of the kernel)
  auto rows_of = [&](int tid) { return xa_of(tid) + 256 * (tid >> 5); };
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
    for (int w = 0; w < 4; w++) {
      for (int tid = 32 * w; tid < 32 * w + 32; tid++) {
        x1h_load_p2(xa_of(tid), lane_t(tid), R[tid].v);
        pass2_fwd(R[tid].v, &tb->pass2[x1h_q(lane_t(tid))][0]);
      }
      for (int tid = 32 * w; tid < 32 * w + 32; tid++)
        b200::x2m_store_p2(rows_of(tid), tid & 15, R[tid].v);
      for (int tid = 32 * w; tid < 32 * w + 32; tid++)
        b200::x2m_load_p3(rows_of(tid), tid & 15, R[tid].v);
    }
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
    for (int w = 0; w < 4; w++) {
      for (int tid = 32 * w; tid < 32 * w + 32; tid++) {
        radix16_inv(R[tid].v, tb->pass3[lane_t(tid)]);
        b200::x2m_store_p3(rows_of(tid), tid & 15, R[tid].v);
      }
      for (int tid = 32 * w; tid < 32 * w + 32; tid++)
        b200::x2m_load_p2(rows_of(tid), tid & 15, R[tid].v);
      for (int tid = 32 * w; tid < 32 * w + 32; tid++) {
        pass2_inv(R[tid].v, &tb->pass2[x1h_q(lane_t(tid))][0]);
        x1h_store_p2(xa_of(tid), lane_t(tid), R[tid].v);
      }
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

// Bank-conflict audit of exchange 2 through the warp's rows: every quarter-warp
// of every 128-bit access (pass-2 side: the forward stores and inverse loads;
// pass-3 side: the forward loads and inverse stores), the worst number of
// distinct slots sharing a 16-byte bank group (1 = conflict-free).
// swizzled = 0 audits the plain map 16 i3 + b instead, to show the audit sees
// conflicts.  Returns -1 if a map is not a bijection on the warp's 256 slots.
int emu_x2m_conflict_audit(int swizzled) {
  auto slot = [&](int i3, int b) { return swizzled ? b200::x2m_slot(i3, b) : 16 * i3 + b; };
  bool seen[256] = {false};
  for (int i3 = 0; i3 < 16; i3++)
    for (int b = 0; b < 16; b++) {
      const int s = slot(i3, b);
      if (s < 0 || s >= 256 || seen[s])
        return -1;
      seen[s] = true;
    }
  int worst = 1;
  auto count = [&](const int *s) {
    int hist[8] = {0};
    for (int y = 0; y < 8; y++)
      if (++hist[s[y] & 7] > worst)
        worst = hist[s[y] & 7];
  };
  for (int quarter = 0; quarter < 2; quarter++) // the two quarters of a half-warp
    for (int reg = 0; reg < 16; reg++) {
      int s2[8], s3[8];
      const int bl = reg >> 2, a = reg & 3;
      for (int j = 0; j < 8; j++) {
        const int i = 8 * quarter + j, p = i & 3, m = i >> 2;
        s2[j] = slot(4 * p + a, 4 * m + bl); // v[4 bl + a] of half-lane p + 4 m
        s3[j] = slot(i, reg);                // v[b] of half-lane i
      }
      count(s2);
      count(s3);
    }
  return worst;
}

} // extern "C"
