// emu_lanepair.cpp -- CPU replay of the lane-pair layout of the N = 2048
// classic PBS kernel (pbs_n2048_k1_l1_v6_kernel<2, true, 2, 1, X2>), with
// exchange 2 through half-warp shuffles (X2 = 0, x2h_*) or through the warp's
// own rows of the exchange-1 buffer (X2 = 1, x2m_*).
//
// TEST INFRASTRUCTURE ONLY.  The replay runs the kernel's per-thread pieces
// (P22LanePair, tfhe-rs_b200/csrc/pbs_n2048_lanepair.cuh), compiled with g++,
// over 4 warps x 32 lanes; the thread map, the twiddle rows, the own-row key
// pointer and the ring's key offsets all come from there.  Every CTA barrier of
// the kernel is one loop over the 128 threads.  The window between the two
// exchange-1 barriers runs warp after warp: exchange 2 goes through the host
// model of the warp exchange, and the MAC reads lane l ^ 16's registers from
// before the MAC.  With X2 = 1 a slot outside the warp's rows would corrupt the
// next warp's exchange-1 loads or the previous warp's exchange-1 stores, and the
// replay would no longer match.  The accumulator rows sit P22_ACC_STRIDE words
// apart as in P22SmemV6.
// Compare it with emu_p22.cpp only when both are built with
// -ffp-contract=off: otherwise g++ fuses products and sums wherever the shape
// of the surrounding code lets it, differently in the two files.
#include <cstdint>
#include <cstring>
#include <memory>
#include <vector>

#include "../../tfhe-rs_b200/csrc/pbs_n2048_lanepair.cuh"

using namespace b200;

namespace {

// filled once, thread-safely: the replay is called from several threads at once
const Fft1024Tables *tables() {
  static const Fft1024Tables *tb = [] {
    Fft1024Tables *t = new Fft1024Tables;
    b200_fill_fft1024_tables(t);
    return t;
  }();
  return tb;
}

uint64_t splitmix(uint64_t &s) {
  uint64_t z = (s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// The CTA's shared memory and registers
struct Cta {
  uint32_t acc[2][P22_ACC_STRIDE];
  cplx xa[2][P22_M];
  cplx ring[2][P22_M];
  cplx v[128][16], b_own[128][16];
  uint32_t own[128][32];
};

// exchange 2 of warp w, both directions
template <int X2> void x2_fwd(Cta &c, const std::vector<P22LanePair> &T, int w) {
  if constexpr (X2 == 1) {
    for (int tid = 32 * w; tid < 32 * w + 32; tid++)
      x2m_store_p2(T[tid].x2_rows, tid & 15, c.v[tid]);
    for (int tid = 32 * w; tid < 32 * w + 32; tid++)
      x2m_load_p3(T[tid].x2_rows, tid & 15, c.v[tid]);
  } else {
    x2h_fwd_warp(c.v + 32 * w);
  }
}
template <int X2> void x2_inv(Cta &c, const std::vector<P22LanePair> &T, int w) {
  if constexpr (X2 == 1) {
    for (int tid = 32 * w; tid < 32 * w + 32; tid++)
      x2m_store_p3(T[tid].x2_rows, tid & 15, c.v[tid]);
    for (int tid = 32 * w; tid < 32 * w + 32; tid++)
      x2m_load_p2(T[tid].x2_rows, tid & 15, c.v[tid]);
  } else {
    x2h_inv_warp(c.v + 32 * w);
  }
}

// one LWE, same arguments as emu_pbs_p22_v3 (tests/emu/emu_p22.cpp); bsk in
// the layout of emu_bsk_convert_p22.  Runs every step, a_hat = 0 included,
// as the kernel does.
template <int X2>
void replay(const double *bsk_, const uint64_t *lut, const uint64_t *ct, uint32_t n,
            uint32_t base_log, int centered_ms, uint32_t num_many_lut, uint32_t lut_stride,
            uint32_t count, uint64_t *out_base) {
  const cplx *bsk = reinterpret_cast<const cplx *>(bsk_);
  const Fft1024Tables *tb = tables();
  const uint32_t log_mod = 12;
  auto cta = std::make_unique<Cta>();
  Cta &c = *cta;
  std::vector<uint16_t> a_hat(n);
  CenteredMsSums sums;
  for (uint32_t i = 0; i < n; i++) {
    a_hat[i] = (uint16_t)modulus_switch_u64(ct[i], log_mod);
    sums.add(ct[i], log_mod);
  }
  const uint32_t b_hat = ms_b_hat(ct[n], centered_ms, &sums.half, &sums.dbl, 1, log_mod);
  rotate_lut(&c.acc[0][0], P22_ACC_STRIDE, lut, 2, P22_N, b_hat, 0, 1, Torus64To32());
  std::vector<P22LanePair> T;
  for (int tid = 0; tid < 128; tid++) {
    const int t = p22lp_t(tid);
    T.emplace_back(tid, c.acc, c.xa, c.ring, bsk, tb->pass1, tb->pass2[x1h_q(t)], tb->pass3[t]);
    T[tid].own_init(c.own[tid]);
  }
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t a = a_hat[i];
    std::memcpy(c.ring, p22_ring_src(bsk, i), P22_RING_BYTES); // the TMA copy of step i
    for (int tid = 0; tid < 128; tid++) {
      T[tid].digits(a, base_log, c.own[tid], c.v[tid]);
      T[tid].fwd_pass1(c.v[tid]);
      T[tid].x1_fwd_store(c.v[tid]);
    }
    for (int w = 0; w < 4; w++) {
      for (int tid = 32 * w; tid < 32 * w + 32; tid++) {
        T[tid].x1_fwd_load(c.v[tid]);
        T[tid].fwd_pass2(c.v[tid]);
      }
      x2_fwd<X2>(c, T, w);
      for (int tid = 32 * w; tid < 32 * w + 32; tid++) {
        T[tid].fwd_pass3(c.v[tid]);
        T[tid].own_row_load(i, c.b_own[tid]);
      }
      cplx V[32][16]; // the warp's registers before the MAC
      std::memcpy(V, c.v + 32 * w, sizeof(V));
      for (int l = 0; l < 32; l++) {
        const int tid = 32 * w + l;
        T[tid].mac(c.v[tid], c.b_own[tid], [&](int b, cplx) { return V[l ^ 16][b]; });
        T[tid].inv_pass3(c.v[tid]);
      }
      x2_inv<X2>(c, T, w);
      for (int tid = 32 * w; tid < 32 * w + 32; tid++) {
        T[tid].inv_pass2(c.v[tid]);
        T[tid].x1_inv_store(c.v[tid]);
      }
    }
    for (int tid = 0; tid < 128; tid++) {
      T[tid].x1_inv_load(c.v[tid]);
      T[tid].inv_pass1(c.v[tid]);
      T[tid].acc_update(c.v[tid], c.own[tid]);
    }
  }
  sample_extract_many_lut(out_base, 0, count, num_many_lut, lut_stride, &c.acc[0][0],
                          P22_ACC_STRIDE, 1, P22_N, 0, 1, Torus32To64());
}

} // namespace

extern "C" {

void emu_pbs_p22_lanepair(const double *bsk, const uint64_t *lut, const uint64_t *ct,
                          uint32_t n, uint32_t base_log, int centered_ms,
                          uint32_t num_many_lut, uint32_t lut_stride, uint32_t count,
                          uint64_t *out_base) {
  replay<0>(bsk, lut, ct, n, base_log, centered_ms, num_many_lut, lut_stride, count, out_base);
}

void emu_pbs_p22_lanepair_x2m(const double *bsk, const uint64_t *lut, const uint64_t *ct,
                              uint32_t n, uint32_t base_log, int centered_ms,
                              uint32_t num_many_lut, uint32_t lut_stride, uint32_t count,
                              uint64_t *out_base) {
  replay<1>(bsk, lut, ct, n, base_log, centered_ms, num_many_lut, lut_stride, count, out_base);
}

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
      x2h_fwd_warp(a);
      x2m_fwd_warp(b);
    } else {
      x2h_inv_warp(a);
      x2m_inv_warp(b);
    }
    for (int l = 0; l < 32; l++)
      for (int r = 0; r < 16; r++)
        bad += std::memcmp(&a[l][r], &b[l][r], sizeof(cplx)) != 0;
  }
  return bad;
}

// Bank-conflict audit of exchange 2 through the warp's rows: every quarter-warp
// of every 128-bit access (pass-2 side: the forward stores and inverse loads;
// pass-3 side: the forward loads and inverse stores), the worst number of
// distinct slots sharing a 16-byte bank group (1 = conflict-free).
// swizzled = 0 audits the plain map 16 i3 + b instead, to show the audit sees
// conflicts.  Returns -1 if a map is not a bijection on the warp's 256 slots.
int emu_x2m_conflict_audit(int swizzled) {
  auto slot = [&](int i3, int b) { return swizzled ? x2m_slot(i3, b) : 16 * i3 + b; };
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
            const int t = p22lp_t(32 * w + 8 * quarter + j);
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
        const int tid = 32 * w + l, base = p22lp_g(tid) * acc_stride, j = 64 * j1 + p22lp_t(tid);
        own0[l] = base + j;
        own1[l] = base + j + P22_M;
      }
      count(own0, 32, 32);
      count(own1, 32, 32);
      for (int d = 0; d < P22_N; d++) {
        int r0[32], r1[32];
        for (int l = 0; l < 32; l++) {
          const int tid = 32 * w + l, base = p22lp_g(tid) * acc_stride;
          const int i0 = (64 * j1 + p22lp_t(tid) - d) & (P22_N - 1);
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
