// emu_p22.cpp -- CPU "CTA emulator" for the N=2048/k=1/l=1 PBS kernel.
//
// TEST INFRASTRUCTURE ONLY.  Compiles the very same B200_HD phase functions
// the sm_90a kernel inlines (tfhe-rs_b200/csrc/*.cuh) with g++ and replays a
// 128-thread block phase by phase (every barrier of the kernel = one loop over
// all threads here), so index math, swizzles, twiddle tables and rounding can
// be checked against the oracle without a GPU.  It is never used by the
// product path and is not a fallback.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../tfhe-rs_b200/csrc/pbs_multibit_n2048_phases.cuh"
#include "../../tfhe-rs_b200/csrc/pbs_generic_phases.cuh"
#include "../../tfhe-rs_b200/csrc/pbs_n8192_phases.cuh"
#include "../../tfhe-rs_b200/csrc/pbs_n512_phases.cuh"
#include "../../tfhe-rs_b200/csrc/x2_shfl.cuh"

// The tables are filled on first use by whichever thread gets there first: the
// replays are called from several threads at once (tests/
// test_gpu_replay_words.py), and a function-local static is initialised exactly
// once, before any thread sees it.
static const Fft1024Tables *tables() {
  static const Fft1024Tables *tb = [] {
    Fft1024Tables *t = new Fft1024Tables;
    b200_fill_fft1024_tables(t);
    return t;
  }();
  return tb;
}

struct Regs {
  cplx v[16];
  uint32_t own[32];
};

// forward transform of 1024 complex values with 64 emulated threads;
// output in slot order pos = 16*t + b
static void fwd1024(const cplx *in, cplx *out_pos) {
  const Fft1024Tables *tb = tables();
  std::vector<Regs> R(64);
  std::vector<cplx> xa(P22_M), xb(P22_M);
  for (int t = 0; t < 64; t++) {
    for (int j1 = 0; j1 < 16; j1++)
      R[t].v[j1] = in[64 * j1 + t];
    radix16_fwd(R[t].v, tb->pass1);
    x1_store_p1(xa.data(), t, R[t].v);
  }
  for (int t = 0; t < 64; t++) {
    x1_load_p2(xa.data(), t, R[t].v);
    pass2_fwd(R[t].v, &tb->pass2[t >> 2][0]);
    x2_store_p2(xb.data(), t, R[t].v);
  }
  for (int t = 0; t < 64; t++) {
    x2_load_p3(xb.data(), t, R[t].v);
    radix16_fwd(R[t].v, tb->pass3[t]);
    for (int b = 0; b < 16; b++)
      out_pos[fft1024_pos(t, b)] = R[t].v[b];
  }
}

static void inv1024(const cplx *in_pos, cplx *out) {
  const Fft1024Tables *tb = tables();
  std::vector<Regs> R(64);
  std::vector<cplx> xa(P22_M), xb(P22_M);
  for (int t = 0; t < 64; t++) {
    for (int b = 0; b < 16; b++)
      R[t].v[b] = in_pos[fft1024_pos(t, b)];
    radix16_inv(R[t].v, tb->pass3[t]);
    x2_store_p3(xb.data(), t, R[t].v);
  }
  for (int t = 0; t < 64; t++) {
    x2_load_p2(xb.data(), t, R[t].v);
    pass2_inv(R[t].v, &tb->pass2[t >> 2][0]);
    x1_store_p2(xa.data(), t, R[t].v);
  }
  for (int t = 0; t < 64; t++) {
    x1_load_p1(xa.data(), t, R[t].v);
    radix16_inv(R[t].v, tb->pass1);
    for (int j1 = 0; j1 < 16; j1++)
      out[64 * j1 + t] = R[t].v[j1];
  }
}

// the same two transforms with exchange 2 through the warp-shuffle rounds
// (x2_shfl.cuh) and the matching exchange-1 layout (x1t_*)
static void fwd1024_shfl(const cplx *in, cplx *out_pos) {
  const Fft1024Tables *tb = tables();
  std::vector<Regs> R(64);
  std::vector<cplx> xa(P22_M);
  cplx w[64][16];
  for (int t = 0; t < 64; t++) {
    for (int j1 = 0; j1 < 16; j1++)
      R[t].v[j1] = in[64 * j1 + t];
    radix16_fwd(R[t].v, tb->pass1);
    x1t_store_p1(xa.data(), t, R[t].v);
  }
  for (int t = 0; t < 64; t++) {
    x1t_load_p2(xa.data(), t, R[t].v);
    pass2_fwd(R[t].v, &tb->pass2[x1t_q(t)][0]);
    std::memcpy(w[t], R[t].v, sizeof(w[t]));
  }
  b200::x2s_fwd_warp(&w[0]);
  b200::x2s_fwd_warp(&w[32]);
  for (int t = 0; t < 64; t++) {
    std::memcpy(R[t].v, w[t], sizeof(w[t]));
    radix16_fwd(R[t].v, tb->pass3[t]);
    for (int b = 0; b < 16; b++)
      out_pos[fft1024_pos(t, b)] = R[t].v[b];
  }
}
static void inv1024_shfl(const cplx *in_pos, cplx *out) {
  const Fft1024Tables *tb = tables();
  std::vector<Regs> R(64);
  std::vector<cplx> xa(P22_M);
  cplx w[64][16];
  for (int t = 0; t < 64; t++) {
    for (int b = 0; b < 16; b++)
      R[t].v[b] = in_pos[fft1024_pos(t, b)];
    radix16_inv(R[t].v, tb->pass3[t]);
    std::memcpy(w[t], R[t].v, sizeof(w[t]));
  }
  b200::x2s_inv_warp(&w[0]);
  b200::x2s_inv_warp(&w[32]);
  for (int t = 0; t < 64; t++) {
    std::memcpy(R[t].v, w[t], sizeof(w[t]));
    pass2_inv(R[t].v, &tb->pass2[x1t_q(t)][0]);
    x1t_store_p2(xa.data(), t, R[t].v);
  }
  for (int t = 0; t < 64; t++) {
    x1t_load_p1(xa.data(), t, R[t].v);
    radix16_inv(R[t].v, tb->pass1);
    for (int j1 = 0; j1 < 16; j1++)
      out[64 * j1 + t] = R[t].v[j1];
  }
}

// M = 256 (N = 512) transform of the pbs_n512 kernel: 16 emulated threads
static const Fft256Tables *tables256() {
  static const Fft256Tables *tb = [] {
    Fft256Tables *t = new Fft256Tables;
    b200_fill_fft256_tables(t);
    return t;
  }();
  return tb;
}
static void fwd256(const cplx *in, cplx *out_pos) {
  const Fft256Tables *tb = tables256();
  std::vector<Regs> R(16);
  std::vector<cplx> xb(256);
  for (int u = 0; u < 16; u++) {
    for (int j1 = 0; j1 < 16; j1++)
      R[u].v[j1] = in[16 * j1 + u];
    radix16_fwd(R[u].v, tb->pass1);
    xq_store_p1(xb.data(), u, R[u].v);
  }
  for (int q = 0; q < 16; q++) {
    xq_load_p2(xb.data(), q, R[q].v);
    radix16_fwd(R[q].v, tb->pass2[q]);
    for (int b = 0; b < 16; b++)
      out_pos[16 * q + b] = R[q].v[b];
  }
}
static void inv256(const cplx *in_pos, cplx *out) {
  const Fft256Tables *tb = tables256();
  std::vector<Regs> R(16);
  std::vector<cplx> xb(256);
  for (int q = 0; q < 16; q++) {
    for (int b = 0; b < 16; b++)
      R[q].v[b] = in_pos[16 * q + b];
    radix16_inv(R[q].v, tb->pass2[q]);
    xq_store_p2(xb.data(), q, R[q].v);
  }
  for (int u = 0; u < 16; u++) {
    xq_load_p1(xb.data(), u, R[u].v);
    radix16_inv(R[u].v, tb->pass1);
    for (int j1 = 0; j1 < 16; j1++)
      out[16 * j1 + u] = R[u].v[j1];
  }
}

// M = 4096 (N = 8192) transform of the pbs_n8192 kernel: 256 emulated threads
static const Fft4096Tables *tables4096() {
  static const Fft4096Tables *tb = [] {
    Fft4096Tables *t = new Fft4096Tables;
    b200_fill_fft4096_tables(t);
    return t;
  }();
  return tb;
}
static void fwd4096(const cplx *in, cplx *out_pos) {
  const Fft4096Tables *tb = tables4096();
  std::vector<Regs> R(256);
  std::vector<cplx> buf(4096);
  for (int t = 0; t < 256; t++) {
    for (int j1 = 0; j1 < 16; j1++)
      R[t].v[j1] = in[256 * j1 + t];
    radix16_fwd(R[t].v, tb->pass1);
    xg_store_p1(buf.data(), t, R[t].v);
  }
  for (int t = 0; t < 256; t++) {
    xg_load_p2(buf.data(), t, R[t].v);
    radix16_fwd(R[t].v, tb->pass2[t >> 4]);
  }
  // exchange 2 inside each half-warp's region (after every thread's exchange-1 load: emulated phase order)
  for (int t = 0; t < 256; t++)
    xq_store_p1(buf.data() + (t >> 4) * 256, t & 15, R[t].v);
  for (int t = 0; t < 256; t++) {
    xq_load_p2(buf.data() + (t >> 4) * 256, t & 15, R[t].v);
    radix16_fwd(R[t].v, tb->pass3[t]);
    for (int b = 0; b < 16; b++)
      out_pos[16 * t + b] = R[t].v[b];
  }
}
static void inv4096(const cplx *in_pos, cplx *out) {
  const Fft4096Tables *tb = tables4096();
  std::vector<Regs> R(256);
  std::vector<cplx> buf(4096);
  for (int t = 0; t < 256; t++) {
    for (int b = 0; b < 16; b++)
      R[t].v[b] = in_pos[16 * t + b];
    radix16_inv(R[t].v, tb->pass3[t]);
    xq_store_p2(buf.data() + (t >> 4) * 256, t & 15, R[t].v);
  }
  for (int t = 0; t < 256; t++) {
    xq_load_p1(buf.data() + (t >> 4) * 256, t & 15, R[t].v);
    radix16_inv(R[t].v, tb->pass2[t >> 4]);
  }
  for (int t = 0; t < 256; t++)
    xg_store_p2(buf.data(), t, R[t].v);
  for (int t = 0; t < 256; t++) {
    xg_load_p1(buf.data(), t, R[t].v);
    radix16_inv(R[t].v, tb->pass1);
    for (int j1 = 0; j1 < 16; j1++)
      out[256 * j1 + t] = R[t].v[j1];
  }
}

extern "C" {

void emu_fft4096_fwd(const double *in, double *out) {
  fwd4096(reinterpret_cast<const cplx *>(in), reinterpret_cast<cplx *>(out));
}
void emu_fft4096_inv(const double *in, double *out) {
  inv4096(reinterpret_cast<const cplx *>(in), reinterpret_cast<cplx *>(out));
}

void emu_fft256_fwd(const double *in, double *out) {
  fwd256(reinterpret_cast<const cplx *>(in), reinterpret_cast<cplx *>(out));
}
void emu_fft256_inv(const double *in, double *out) {
  inv256(reinterpret_cast<const cplx *>(in), reinterpret_cast<cplx *>(out));
}

void emu_fft1024_fwd_shfl(const double *in, double *out) {
  fwd1024_shfl(reinterpret_cast<const cplx *>(in), reinterpret_cast<cplx *>(out));
}
void emu_fft1024_inv_shfl(const double *in, double *out) {
  inv1024_shfl(reinterpret_cast<const cplx *>(in), reinterpret_cast<cplx *>(out));
}

// forward transform test entry: in/out interleaved (re, im), out in slot order
void emu_fft1024_fwd(const double *in, double *out) {
  fwd1024(reinterpret_cast<const cplx *>(in), reinterpret_cast<cplx *>(out));
}
// unnormalised inverse (result = 1024 * original)
void emu_fft1024_inv(const double *in, double *out) {
  inv1024(reinterpret_cast<const cplx *>(in), reinterpret_cast<cplx *>(out));
}

// mirrors bsk_convert_n2048_k1_l1_kernel; src = n*4 polynomials [i][r][c][N]
void emu_bsk_convert_p22(const uint64_t *src, uint32_t n, double *dst_) {
  cplx *dst = reinterpret_cast<cplx *>(dst_);
  const double scale = 2.27373675443232059478759765625e-13; // 2^-42 = 2^-64 / 1024 * 2^32 (see scaled_double_to_torus32)
  std::vector<cplx> in(P22_M), out(P22_M);
  for (uint32_t poly = 0; poly < n * 4; poly++) {
    const uint32_t i = poly >> 2, r = (poly >> 1) & 1, c = poly & 1;
    const uint64_t *p = src + (size_t)poly * P22_N;
    for (int j = 0; j < P22_M; j++)
      in[j] = cmake(ll_to_double((int64_t)p[j]) * scale,
                    ll_to_double((int64_t)p[j + P22_M]) * scale);
    fwd1024(in.data(), out.data());
    cplx *o = dst + (((size_t)i * 2 + c) * 2 + r) * P22_M;
    for (int t = 0; t < 64; t++)
      for (int b = 0; b < 16; b++)
        o[b * 64 + t] = out[fft1024_pos(t, b)];
  }
}

struct HostLoader {
  cplx operator()(const cplx *p) const { return *p; }
};

// mirrors pbs_n2048_k1_l1_kernel for one sample
void emu_pbs_p22(const double *bsk_, const uint64_t *lut, const uint64_t *ct,
                 uint32_t n, uint32_t base_log, int centered_ms,
                 uint32_t num_many_lut, uint32_t lut_stride, uint32_t count,
                 uint64_t *out_base /* many-lut stride count*(N+1) */) {
  const cplx *bsk = reinterpret_cast<const cplx *>(bsk_);
  const Fft1024Tables *tb = tables();
  const uint32_t log_mod = 12;
  std::vector<uint64_t> acc(2 * P22_N);
  std::vector<cplx> xa(2 * P22_M), xb(2 * P22_M);
  std::vector<uint16_t> a_hat(n);
  // prologue
  CenteredMsSums sums;
  for (uint32_t i = 0; i < n; i++) {
    a_hat[i] = (uint16_t)modulus_switch_u64(ct[i], log_mod);
    sums.add(ct[i], log_mod);
  }
  const uint32_t b_hat = ms_b_hat(ct[n], centered_ms, &sums.half, &sums.dbl, 1, log_mod);
  rotate_lut(acc.data(), P22_N, lut, 2, P22_N, b_hat, 0, 1, SameWord());
  std::vector<Regs> R(128);
  std::vector<cplx> tw2(128 * 12), tw3(128 * 15);
  for (int tid = 0; tid < 128; tid++) {
    const int t = tid & 63;
    for (int e = 0; e < 3; e++)
      tw2[tid * 12 + e] = tb->pass2[t >> 2][e];
    for (int e = 0; e < 15; e++)
      tw3[tid * 15 + e] = tb->pass3[t][e];
  }
#define FOR_THREADS                                                            \
  for (int tid = 0; tid < 128; tid++) {                                        \
    const int g = tid >> 6, t = tid & 63;                                      \
    cplx *v = R[tid].v;                                                        \
    uint64_t *acc_g = acc.data() + g * P22_N;                                  \
    cplx *xa_g = xa.data() + g * P22_M;                                        \
    cplx *xb_g = xb.data() + g * P22_M;                                        \
    const cplx *xa_other = xa.data() + (1 - g) * P22_M;                        \
    (void)acc_g; (void)xa_g; (void)xb_g; (void)xa_other; (void)t; (void)v;
#define END_THREADS }
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t a = a_hat[i];
    if (a == 0)
      continue;
    FOR_THREADS
      p22_load_digits(acc_g, t, a, base_log, v);
      radix16_fwd(v, tb->pass1);
      x1_store_p1(xa_g, t, v);
    END_THREADS
    FOR_THREADS
      x1_load_p2(xa_g, t, v);
      pass2_fwd(v, &tw2[tid * 12]);
      x2_store_p2(xb_g, t, v);
    END_THREADS
    FOR_THREADS
      x2_load_p3(xb_g, t, v);
      radix16_fwd(v, &tw3[tid * 15]);
      spec_store(xa_g, t, v);
    END_THREADS
    FOR_THREADS
      p22_mac(v, xa_other, bsk + ((size_t)i * 2 + g) * (2 * P22_M), t, g,
              HostLoader());
    END_THREADS
    FOR_THREADS
      radix16_inv(v, &tw3[tid * 15]);
      x2_store_p3(xb_g, t, v);
    END_THREADS
    FOR_THREADS
      x2_load_p2(xb_g, t, v);
      pass2_inv(v, &tw2[tid * 12]);
      x1_store_p2(xa_g, t, v);
    END_THREADS
    FOR_THREADS
      x1_load_p1(xa_g, t, v);
      radix16_inv(v, tb->pass1);
      p22_acc_update(acc_g, t, v);
    END_THREADS
  }
  sample_extract_many_lut(out_base, 0, count, num_many_lut, lut_stride, acc.data(), P22_N,
                          1, P22_N, 0, 1, SameWord());
}

// mirrors pbs_n2048_k1_l1_v3_kernel (u32 accumulator, lean digits, prefetch MAC)
void emu_pbs_p22_v3(const double *bsk_, const uint64_t *lut, const uint64_t *ct,
                    uint32_t n, uint32_t base_log, int centered_ms,
                    uint32_t num_many_lut, uint32_t lut_stride, uint32_t count,
                    uint64_t *out_base) {
  const cplx *bsk = reinterpret_cast<const cplx *>(bsk_);
  const Fft1024Tables *tb = tables();
  const uint32_t log_mod = 12;
  std::vector<uint32_t> acc(2 * P22_N);
  std::vector<cplx> xa(2 * P22_M);
  std::vector<uint16_t> a_hat(n);
  CenteredMsSums sums;
  for (uint32_t i = 0; i < n; i++) {
    a_hat[i] = (uint16_t)modulus_switch_u64(ct[i], log_mod);
    sums.add(ct[i], log_mod);
  }
  const uint32_t b_hat = ms_b_hat(ct[n], centered_ms, &sums.half, &sums.dbl, 1, log_mod);
  rotate_lut(acc.data(), P22_N, lut, 2, P22_N, b_hat, 0, 1, Torus64To32());
  std::vector<Regs> R(128);
#define FOR_THREADS2                                                           \
  for (int tid = 0; tid < 128; tid++) {                                        \
    const int g = tid >> 6, t = tid & 63;                                      \
    cplx *v = R[tid].v;                                                        \
    uint32_t *acc_g = acc.data() + g * P22_N;                                  \
    cplx *xa_g = xa.data() + g * P22_M;                                        \
    const cplx *xa_other = xa.data() + (1 - g) * P22_M;                        \
    (void)acc_g; (void)xa_g; (void)xa_other; (void)t; (void)v;
  FOR_THREADS2
    p22v4_own_init(acc_g, t, R[tid].own);
  END_THREADS
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t a = a_hat[i];
    if (a == 0)
      continue;
    FOR_THREADS2
      // shipped phases (v4); must produce the digits of the round-1 phases bit for bit
      cplx v3[16];
      p22v3_load_digits(acc_g, t, a, base_log, v3);
      p22v4_load_digits(acc_g, t, a, base_log, R[tid].own, v);
      for (int q = 0; q < 16; q++)
        if (v3[q].re != v[q].re || v3[q].im != v[q].im) {
          std::fprintf(stderr, "emu: v4 digits differ from v3 (tid %d, q %d)\n", tid, q);
          std::abort();
        }
      radix16_fwd(v, tb->pass1);
      x1_store_p1(xa_g, t, v);
    END_THREADS
    FOR_THREADS2
      x1_load_p2(xa_g, t, v);
    END_THREADS
    FOR_THREADS2
      pass2_fwd(v, &tb->pass2[t >> 2][0]);
      x2_store_p2(xa_g, t, v);
    END_THREADS
    FOR_THREADS2
      x2_load_p3(xa_g, t, v);
    END_THREADS
    FOR_THREADS2
      radix16_fwd(v, tb->pass3[t]);
      spec_store(xa_g, t, v);
    END_THREADS
    FOR_THREADS2
      const cplx *bsk_ig = bsk + ((size_t)i * 2 + g) * (2 * P22_M);
      cplx b_own[16];
      for (int b = 0; b < 16; b++)
        b_own[b] = bsk_ig[(g * 16 + b) * 64 + t];
      p22v3_mac(v, b_own, xa_other, bsk_ig + (1 - g) * P22_M, t, HostLoader());
    END_THREADS
    FOR_THREADS2
      radix16_inv(v, tb->pass3[t]);
      x2_store_p3(xa_g, t, v);
    END_THREADS
    FOR_THREADS2
      x2_load_p2(xa_g, t, v);
    END_THREADS
    FOR_THREADS2
      pass2_inv(v, &tb->pass2[t >> 2][0]);
      x1_store_p2(xa_g, t, v);
    END_THREADS
    FOR_THREADS2
      x1_load_p1(xa_g, t, v);
      radix16_inv(v, tb->pass1);
      p22v4_acc_update(acc_g, t, v, R[tid].own);
    END_THREADS
  }
  sample_extract_many_lut(out_base, 0, count, num_many_lut, lut_stride, acc.data(), P22_N,
                          1, P22_N, 0, 1, Torus32To64());
}

// bank-conflict audit of the exchange layouts: for each of the 8 access
// patterns returns the worst number of distinct-address lanes of a quarter
// warp (8 consecutive threads) that share a 16-byte bank group (1 = free).
int emu_exchange_conflict_audit() {
  int worst = 1;
  auto audit = [&](auto slot_of) {
    for (int reg = 0; reg < 16; reg++)
      for (int quarter = 0; quarter < 8; quarter++) {
        int cnt[8] = {0};
        for (int l = 0; l < 8; l++)
          cnt[slot_of(8 * quarter + l, reg) & 7]++;
        for (int b = 0; b < 8; b++)
          if (cnt[b] > worst)
            worst = cnt[b];
      }
  };
  audit([](int t, int q) { return x1_slot(q, t); });                       // p1 side
  audit([](int t, int r) { return x1_slot(t >> 2, 16 * (r & 3) + 4 * (t & 3) + (r >> 2)); });
  audit([](int t, int r) { return x2_slot(4 * (t >> 2) + (r & 3), 4 * (t & 3) + (r >> 2)); });
  audit([](int t, int b) { return x2_slot(t, b); });                       // p3 side
  audit([](int t, int b) { return b * 64 + t; });                          // spectrum
  // exchange 1 of the shuffle variant (x1t_*)
  audit([](int t, int q) { return x1t_slot(q, t); });
  audit([](int t, int r) { return x1t_slot(x1t_q(t), 16 * (r & 3) + 4 * x1t_bh(t) + (r >> 2)); });
  // 16 x 16 exchange of the N = 512 kernel (two polynomials per warp, 16 lanes each)
  audit([](int t, int q) { return xq_slot(q, t & 15); });
  audit([](int t, int u) { return xq_slot(t & 15, u); });
  return worst;
}

} // extern "C"

// ---------------------------------------------------------------------------
// multi-bit fast kernel (pbs_multibit_n2048.cuh)
// ---------------------------------------------------------------------------
static size_t mb_key_row(uint32_t grp, uint32_t c, uint32_t b, uint32_t lvl,
                         uint32_t r, uint32_t s, uint32_t l, uint32_t nggsw) {
  return ((((((size_t)grp * 2 + c) * 16 + b) * l + lvl) * 2 + r) * nggsw + s) * 64;
}

// mirrors bsk_convert_multibit_n2048_kernel
extern "C" void emu_bsk_convert_mb(const uint64_t *src, uint32_t n, uint32_t l,
                        uint32_t grouping, double *dst_) {
  cplx *dst = reinterpret_cast<cplx *>(dst_);
  const uint32_t nggsw = 1u << grouping;
  const uint32_t polys = (n / grouping) * nggsw * l * 4;
  const double scale = 2.27373675443232059478759765625e-13; // 2^-42 = 2^-64 / 1024 * 2^32 (see scaled_double_to_torus32)
  std::vector<cplx> in(P22_M), out(P22_M);
  for (uint32_t idx = 0; idx < polys; idx++) {
    uint32_t poly = idx;
    const uint32_t c = poly & 1; poly >>= 1;
    const uint32_t r = poly & 1; poly >>= 1;
    const uint32_t lvl = poly % l; poly /= l;
    const uint32_t s = poly & (nggsw - 1), grp = poly >> grouping;
    const uint64_t *p = src + (size_t)idx * P22_N;
    for (int j = 0; j < P22_M; j++)
      in[j] = cmake(ll_to_double((int64_t)p[j]) * scale,
                    ll_to_double((int64_t)p[j + P22_M]) * scale);
    fwd1024(in.data(), out.data());
    for (int t = 0; t < 64; t++)
      for (int b = 0; b < 16; b++)
        dst[mb_key_row(grp, c, b, lvl, r, s, l, nggsw) + t] = out[fft1024_pos(t, b)];
  }
}


// LL = false: mirrors pbs_multibit_n2048_k1_kernel (bundle folded into the
// MAC, mb_mac_step); LL = true: the low-latency mode, mb_bundle_kernel's bundle
// of each step (mb_bundle_entry) then pbs_multibit_seq_kernel's MAC, 2 l terms
// per slot summed from zero in (level, row) order
template <int GROUPING, bool LL = false>
static void emu_pbs_mb_impl(const cplx *bsk, const uint64_t *lut,
                            const uint64_t *ct, uint32_t n, uint32_t base_log,
                            uint32_t l, uint32_t num_many_lut,
                            uint32_t lut_stride, uint32_t count,
                            uint64_t *out_base) {
  constexpr uint32_t nggsw = 1u << GROUPING, grouping = GROUPING;
  const Fft1024Tables *tb = tables();
  const uint32_t log_mod = 12;
  std::vector<cplx> root(4 * P22_M), tw(P22_M);
  b200_fill_generic_tables(10, tw.data(), root.data());
  cplx zeta[16];
  for (int m = 0; m < 16; m++)
    zeta[m] = root[(256u * m) & (2 * P22_N - 1)];
  const uint32_t b_hat = modulus_switch_u64(ct[n], log_mod);
  struct T { uint32_t lo[16], hi[16]; cplx v[16]; };
  std::vector<T> R(128);
  for (int tid = 0; tid < 128; tid++) {
    const int g = tid >> 6, t = tid & 63;
    const uint64_t *lp = lut + (size_t)g * P22_N;
    for (int j1 = 0; j1 < 16; j1++) {
      const uint32_t j = 64u * j1 + t;
      R[tid].lo[j1] = torus64_to_32(rot_div_coeff(lp, P22_N, j, b_hat));
      R[tid].hi[j1] = torus64_to_32(rot_div_coeff(lp, P22_N, j + P22_M, b_hat));
    }
  }
  std::vector<cplx> sp(4 * P22_M), xa(2 * P22_M);
  uint32_t degs[16] = {0};
#define MB_THREADS                                                             \
  for (int tid = 0; tid < 128; tid++) {                                        \
    const int g = tid >> 6, t = tid & 63;                                      \
    cplx *v = R[tid].v;                                                        \
    cplx *xa_g = xa.data() + g * P22_M;                                        \
    (void)g; (void)t; (void)v; (void)xa_g;
  for (uint32_t grp = 0; grp < n / grouping; grp++) {
    for (uint32_t s = 1; s < nggsw; s++) {
      uint64_t sum = 0;
      for (uint32_t u = 0; u < grouping; u++)
        if ((s >> (grouping - 1 - u)) & 1u)
          sum += ct[grp * grouping + u];
      degs[s] = modulus_switch_u64(sum, log_mod);
    }
    for (uint32_t lvl = 0; lvl < l; lvl++) {
      MB_THREADS
        mb_load_digits(R[tid].lo, R[tid].hi, base_log, l, lvl, v);
        radix16_fwd(v, tb->pass1);
        x1_store_p1(xa_g, t, v);
      END_THREADS
      MB_THREADS
        x1_load_p2(xa_g, t, v);
      END_THREADS
      MB_THREADS
        pass2_fwd(v, &tb->pass2[t >> 2][0]);
        x2_store_p2(xa_g, t, v);
      END_THREADS
      MB_THREADS
        x2_load_p3(xa_g, t, v);
      END_THREADS
      MB_THREADS
        radix16_fwd(v, tb->pass3[t]);
        spec_store(sp.data() + (size_t)(lvl * 2 + g) * P22_M, t, v);
      END_THREADS
    }
    if (LL) {
      // the bundle of this step, [lvl][c][r][b * 64 + t]
      std::vector<cplx> bun((size_t)l * 4 * P22_M);
      for (uint32_t c = 0; c < 2; c++)
        for (uint32_t b = 0; b < 16; b++)
          for (int t = 0; t < 64; t++) {
            const cplx *rows = bsk + mb_key_row(grp, c, b, 0, 0, 0, l, nggsw) + t;
            auto key = [&](uint32_t sigma, int lvl, int r) {
              return rows[((size_t)(lvl * 2 + r) * nggsw + sigma) * 64];
            };
            auto mono_row = [&](uint32_t deg) { return root[mb_base_exponent(deg, t)]; };
            auto put = [&](auto &acc) {
              for (uint32_t lvl = 0; lvl < l; lvl++)
                for (int r = 0; r < 2; r++)
                  bun[((lvl * 2 + c) * 2 + r) * P22_M + b * 64 + t] = acc[lvl][r];
            };
            if (l == 1) {
              cplx acc[1][2];
              mb_bundle_entry<(int)nggsw, 1>(key, mono_row, zeta, degs, mb_bitrev4(b), acc);
              put(acc);
            } else {
              cplx acc[2][2];
              mb_bundle_entry<(int)nggsw, 2>(key, mono_row, zeta, degs, mb_bitrev4(b), acc);
              put(acc);
            }
          }
      MB_THREADS
        for (int b = 0; b < 16; b++) {
          cplx out = cmake(0.0, 0.0);
          for (uint32_t lvl = 0; lvl < l; lvl++)
            for (int r = 0; r < 2; r++)
              out = cfma(sp[((size_t)(lvl * 2 + r) * 16 + b) * 64 + t],
                         bun[((lvl * 2 + g) * 2 + r) * P22_M + b * 64 + t], out);
          v[b] = out;
        }
      END_THREADS
    } else {
    MB_THREADS
      cplx mono_base[nggsw - 1];
      for (uint32_t s = 1; s < nggsw; s++)
        mono_base[s - 1] = root[mb_base_exponent(degs[s], t)];
      const cplx *key_c = bsk + mb_key_row(grp, g, 0, 0, 0, 0, l, nggsw);
      const size_t slot_stride = (size_t)l * 2 * nggsw * 64;
      auto slot_rows = [&](int b) { return key_c + (size_t)b * slot_stride; };
      auto out_slot = [&](int b, cplx val) { xa_g[b * 64 + t] = val; };
      if (l == 1)
        mb_mac_step<(int)nggsw, 1>(sp.data(), mono_base, zeta, degs, t, HostLoader(), slot_rows, out_slot);
      else
        mb_mac_step<(int)nggsw, 2>(sp.data(), mono_base, zeta, degs, t, HostLoader(), slot_rows, out_slot);
    END_THREADS
    MB_THREADS
      for (int b = 0; b < 16; b++)
        v[b] = xa_g[b * 64 + t];
    END_THREADS
    }
    MB_THREADS
      radix16_inv(v, tb->pass3[t]);
      x2_store_p3(xa_g, t, v);
    END_THREADS
    MB_THREADS
      x2_load_p2(xa_g, t, v);
    END_THREADS
    MB_THREADS
      pass2_inv(v, &tb->pass2[t >> 2][0]);
      x1_store_p2(xa_g, t, v);
    END_THREADS
    MB_THREADS
      x1_load_p1(xa_g, t, v);
      radix16_inv(v, tb->pass1);
      mb_acc_assign(R[tid].lo, R[tid].hi, v);
    END_THREADS
  }
  std::vector<uint32_t> acc(2 * P22_N);
  for (int tid = 0; tid < 128; tid++) {
    const int g = tid >> 6, t = tid & 63;
    for (int j1 = 0; j1 < 16; j1++) {
      acc[g * P22_N + 64 * j1 + t] = R[tid].lo[j1];
      acc[g * P22_N + 64 * j1 + t + P22_M] = R[tid].hi[j1];
    }
  }
  sample_extract_many_lut(out_base, 0, count, num_many_lut, lut_stride, acc.data(), P22_N,
                          1, P22_N, 0, 1, Torus32To64());
}

// mirrors the low-latency multi-bit mode (mb_bundle_kernel + pbs_multibit_seq_kernel)
extern "C" void emu_pbs_mb_ll(const double *bsk_, const uint64_t *lut, const uint64_t *ct,
                   uint32_t n, uint32_t base_log, uint32_t l, uint32_t grouping,
                   uint32_t num_many_lut, uint32_t lut_stride, uint32_t count,
                   uint64_t *out_base) {
  const cplx *bsk = reinterpret_cast<const cplx *>(bsk_);
  if (grouping == 2)
    emu_pbs_mb_impl<2, true>(bsk, lut, ct, n, base_log, l, num_many_lut, lut_stride, count, out_base);
  else if (grouping == 3)
    emu_pbs_mb_impl<3, true>(bsk, lut, ct, n, base_log, l, num_many_lut, lut_stride, count, out_base);
  else
    emu_pbs_mb_impl<4, true>(bsk, lut, ct, n, base_log, l, num_many_lut, lut_stride, count, out_base);
}

extern "C" void emu_pbs_mb(const double *bsk_, const uint64_t *lut, const uint64_t *ct,
                uint32_t n, uint32_t base_log, uint32_t l, uint32_t grouping,
                uint32_t num_many_lut, uint32_t lut_stride, uint32_t count,
                uint64_t *out_base) {
  const cplx *bsk = reinterpret_cast<const cplx *>(bsk_);
  if (grouping == 2)
    emu_pbs_mb_impl<2>(bsk, lut, ct, n, base_log, l, num_many_lut, lut_stride, count, out_base);
  else if (grouping == 3)
    emu_pbs_mb_impl<3>(bsk, lut, ct, n, base_log, l, num_many_lut, lut_stride, count, out_base);
  else
    emu_pbs_mb_impl<4>(bsk, lut, ct, n, base_log, l, num_many_lut, lut_stride, count, out_base);
}


// ---------------------------------------------------------------------------
// (N = 8192, k = 1, l = 2) register kernel (pbs_n8192.cuh): key conversion and a
// whole PBS replayed with the kernel's own phase functions -- rotate + decompose
// once per polynomial (n8192_load_digits2 / n8192_unpack_digits), 16 x 16 x 16
// transforms, the four spectra of a step kept aside (a park area on the GPU),
// thread-local Fourier MAC in the kernel's order (level slot, row), key layout
// n8192_key_offset, u32 accumulators.
// ---------------------------------------------------------------------------
extern "C" void emu_bsk_convert_n8192(const uint64_t *src, uint32_t n, double *dst_) {
  cplx *dst = reinterpret_cast<cplx *>(dst_);
  std::vector<cplx> in(P8K_M), out(P8K_M);
  for (uint32_t poly = 0; poly < n * 8; poly++) {
    const uint64_t *p = src + (size_t)poly * P8K_N;
    for (int j = 0; j < P8K_M; j++)
      in[j] = cmake(ll_to_double((int64_t)p[j]) * P8K_KEY_SCALE,
                    ll_to_double((int64_t)p[j + P8K_M]) * P8K_KEY_SCALE);
    fwd4096(in.data(), out.data());
    for (int t3 = 0; t3 < 256; t3++)
      for (int b = 0; b < 16; b++)
        dst[n8192_key_offset(poly >> 3, (poly >> 2) & 1, (poly >> 1) & 1, poly & 1, b, t3)] = out[16 * t3 + b];
  }
}

extern "C" void emu_pbs_n8192(const double *bsk_, const uint64_t *lut, const uint64_t *cts, uint32_t n,
                              uint32_t base_log, int centered_ms, int ties_even, uint32_t num_many_lut,
                              uint32_t lut_stride, uint32_t count, uint64_t *out_base) {
  const cplx *bsk = reinterpret_cast<const cplx *>(bsk_);
  const uint32_t log_mod = 14;
  std::vector<uint32_t> acc(2 * P8K_N);
  std::vector<uint32_t> a_hat(n);
  std::vector<cplx> in0(P8K_M), in1(P8K_M), outc(P8K_M), res(P8K_M);
  std::vector<std::vector<cplx>> spec(4, std::vector<cplx>(P8K_M));
  for (uint32_t s = 0; s < count; s++) {
    const uint64_t *ct = cts + (size_t)s * (n + 1);
    CenteredMsSums sums;
    for (uint32_t i = 0; i < n; i++) {
      a_hat[i] = modulus_switch_u64(ct[i], log_mod) & 0xFFFFu;
      sums.add(ct[i], log_mod);
    }
    const uint32_t b_hat = ms_b_hat(ct[n], centered_ms, &sums.half, &sums.dbl, 1, log_mod);
    rotate_lut(acc.data(), P8K_N, lut, 2, P8K_N, b_hat, 0, 1, Torus64To32());
    for (uint32_t i = 0; i < n; i++) {
      const uint32_t a = a_hat[i];
      if (a == 0)
        continue;
      for (uint32_t r = 0; r < 2; r++) {
        for (int t = 0; t < 256; t++) {
          cplx v[16];
          uint32_t packed[16];
          n8192_load_digits2(&acc[r * P8K_N], t, a, base_log, ties_even != 0, v, packed);
          for (int j1 = 0; j1 < 16; j1++)
            in0[256 * j1 + t] = v[j1];
          n8192_unpack_digits(packed, v);
          for (int j1 = 0; j1 < 16; j1++)
            in1[256 * j1 + t] = v[j1];
        }
        fwd4096(in0.data(), spec[r].data());
        fwd4096(in1.data(), spec[2 + r].data());
      }
      for (uint32_t c = 0; c < 2; c++) {
        for (int t3 = 0; t3 < 256; t3++)
          for (int b = 0; b < 16; b++) {
            const int pos = 16 * t3 + b;
            cplx o = cmul(spec[0][pos], bsk[n8192_key_offset(i, 0, 0, c, b, t3)]);
            for (uint32_t sp = 1; sp < 4; sp++)
              o = cfma(spec[sp][pos], bsk[n8192_key_offset(i, sp >> 1, sp & 1, c, b, t3)], o);
            outc[pos] = o;
          }
        inv4096(outc.data(), res.data());
        uint32_t *acc_c = &acc[c * P8K_N];
        for (int j = 0; j < P8K_M; j++) {
          acc_c[j] += scaled_double_to_torus32(res[j].re);
          acc_c[j + P8K_M] += scaled_double_to_torus32(res[j].im);
        }
      }
    }
    sample_extract_many_lut(out_base, s, count, num_many_lut, lut_stride, acc.data(), P8K_N,
                            1, P8K_N, 0, 1, Torus32To64());
  }
}

// digits2_u32 against digits_u32<2> on `count` words (a multiplicative walk that
// covers every residue class of the low bits, plus the edge words); returns the
// number of mismatches
extern "C" uint64_t emu_digits2_mismatches(uint32_t base_log, uint64_t count, int ties_even) {
  uint64_t bad = 0;
  const uint32_t R = 2 * base_log, drop = 32 - R;
  auto check = [&](uint32_t x) {
    int32_t a[2] = {0, 0}, b[2] = {0, 0};
    digits_u32<2>(x, base_log, 2, a, ties_even != 0);
    digits2_u32(x, base_log, b, ties_even != 0);
    bad += (a[0] != b[0]) | (a[1] != b[1]);
  };
  uint32_t x = 12345u;
  for (uint64_t i = 0; i < count; i++) {
    check(x);
    x = x * 2654435761u + 0x9E3779B9u;
  }
  // edges: around 0, +-2^(R-1) (top-level balance), digit boundaries B/2, every low pattern
  for (uint32_t low = 0; low < (1u << drop); low++)
    for (int32_t hi = -4; hi <= 4; hi++)
      for (uint32_t base : {0u, 0x80000000u, 0x7FFFFFFFu, 0x40000000u, (1u << (drop + base_log - 1)),
                            (1u << (drop + base_log)), (1u << (drop + 2 * base_log - 1)), 0xFFFFFFFFu})
        check(base + (uint32_t)(hi * (int32_t)(1u << drop)) + low);
  return bad;
}

// digits_u32 (multi-bit register kernels) exposed for the tie-rule test
extern "C" void emu_digits_u32(uint32_t x, uint32_t base_log, uint32_t l, int32_t *out) {
  int32_t d[2] = {0, 0};
  digits_u32<2>(x, base_log, l, d);
  out[0] = d[0];
  out[1] = d[1];
}
// same with the reference's round-half-up (b200_set_multibit_tie_rule(1))
extern "C" void emu_digits_u32_reference_ties(uint32_t x, uint32_t base_log, uint32_t l, int32_t *out) {
  int32_t d[2] = {0, 0};
  digits_u32<2>(x, base_log, l, d, false);
  out[0] = d[0];
  out[1] = d[1];
}

// ---------------------------------------------------------------------------
// any-(N, k, l) kernel (pbs_generic.cuh), classic and multi-bit, 64- or 32-bit
// torus: one CTA of 256 threads replayed phase by phase with the kernel's own
// phases (modulus switch, rotation, gen_decompose, radix-2 levels, gen_mac,
// gen_acc_update, sample extraction with TorusIo's widen / narrow).  Both
// variants of the kernel (shared memory and global workspace) compute the same
// words: they differ only in where the working set lives.
// ---------------------------------------------------------------------------
namespace {
constexpr uint32_t GEN_THREADS = 256, GEN_MAX_LOGM = 13; // N = 16384

// twiddle and root tables of every transform size, filled once, as the
// backend's device tables are (b200_fill_generic_tables)
struct GenTables {
  std::vector<cplx> tw, root;
};
const GenTables &gen_tables(uint32_t logM) {
  static const std::vector<GenTables> *all = [] {
    auto *v = new std::vector<GenTables>(GEN_MAX_LOGM + 1);
    for (uint32_t L = 1; L <= GEN_MAX_LOGM; L++) {
      (*v)[L].tw.resize(1u << L);
      (*v)[L].root.resize(4u << L);
      b200_fill_generic_tables(L, (*v)[L].tw.data(), (*v)[L].root.data());
    }
    return v;
  }();
  return (*all)[logM];
}

uint32_t log2_exact(uint32_t x) {
  uint32_t r = 0;
  while ((1u << r) < x)
    r++;
  return r;
}

// mirrors bsk_convert_generic_kernel over `polys` polynomials of N words
template <typename Torus>
void emu_bsk_convert_generic_impl(const Torus *src, size_t polys, uint32_t N, cplx *dst) {
  const uint32_t M = N >> 1, logM = log2_exact(M);
  const GenTables &tb = gen_tables(logM);
  const double scale = ldexp(1.0, -64 - (int)logM);
  std::vector<cplx> buf(M);
  for (size_t b = 0; b < polys; b++) {
    const Torus *p = src + b * N;
    for (uint32_t j = 0; j < M; j++)
      buf[j] = cmake(ll_to_double((int64_t)TorusIo<Torus>::widen(p[j])) * scale,
                     ll_to_double((int64_t)TorusIo<Torus>::widen(p[j + M])) * scale);
    for (uint32_t L = 1; L <= logM; L++)
      for (uint32_t tid = 0; tid < 256; tid++)
        gen_fwd_level(buf.data(), logM, L, tb.tw.data(), 1, tid, 256);
    std::memcpy(dst + b * M, buf.data(), M * sizeof(cplx));
  }
}

// mirrors pbs_generic_kernel for one sample (out_idx 0 of a batch of `count`)
template <typename Torus>
void emu_pbs_generic_impl(const cplx *bsk, const Torus *lut, const Torus *ct, uint32_t n, uint32_t k, uint32_t N,
                          uint32_t base_log, uint32_t l, uint32_t grouping, int centered_ms, int ties_even,
                          uint32_t num_many_lut, uint32_t lut_stride, uint32_t count, Torus *out_base) {
  using Io = TorusIo<Torus>;
  constexpr uint32_t NT = GEN_THREADS;
  const uint32_t M = N >> 1, logM = log2_exact(M), log_mod = logM + 2;
  const GenTables &tb = gen_tables(logM);
  const bool multibit = grouping > 1;
  std::vector<uint64_t> acc((size_t)(k + 1) * N);
  std::vector<cplx> F((size_t)l * (k + 1) * M), out((size_t)(k + 1) * M);
  std::vector<uint32_t> a_hat(n + 1);
  uint32_t degs[16] = {0};
  CenteredMsSums sums;
  if (!multibit)
    for (uint32_t i = 0; i < n; i++) {
      const uint64_t a = Io::widen(ct[i]);
      a_hat[i] = modulus_switch_u64(a, log_mod);
      if (centered_ms)
        sums.add(a, log_mod);
    }
  const uint32_t b_hat = ms_b_hat(Io::widen(ct[n]), !multibit && centered_ms, &sums.half, &sums.dbl, 1, log_mod);
  rotate_lut(acc.data(), N, lut, k + 1, N, b_hat, 0, 1, [](Torus x) { return Io::widen(x); });
  const uint32_t nggsw = multibit ? (1u << grouping) : 1u;
  const uint32_t steps = multibit ? n / grouping : n;
  const size_t ggsw_len = (size_t)l * (k + 1) * (k + 1) * M;
  for (uint32_t i = 0; i < steps; i++) {
    uint32_t a = 0;
    if (multibit) {
      for (uint32_t s = 0; s < nggsw; s++) {
        uint64_t sum = 0;
        for (uint32_t u = 0; u < grouping; u++)
          if ((s >> (grouping - 1 - u)) & 1u)
            sum += Io::widen(ct[i * grouping + u]);
        degs[s] = modulus_switch_u64(sum, log_mod);
      }
    } else {
      a = a_hat[i];
      if (a == 0)
        continue;
    }
    for (uint32_t tid = 0; tid < NT; tid++)
      gen_decompose(acc.data(), F.data(), N, k, base_log, l, a, multibit, tid, NT, ties_even != 0);
    for (uint32_t L = 1; L <= logM; L++)
      for (uint32_t tid = 0; tid < NT; tid++)
        gen_fwd_level(F.data(), logM, L, tb.tw.data(), l * (k + 1), tid, NT);
    for (uint32_t tid = 0; tid < NT; tid++)
      gen_mac(F.data(), out.data(), bsk + (size_t)i * nggsw * ggsw_len, N, k, l, nggsw, degs, tb.root.data(), tid,
              NT, HostLoader());
    for (uint32_t L = logM; L >= 1; L--)
      for (uint32_t tid = 0; tid < NT; tid++)
        gen_inv_level(out.data(), logM, L, tb.tw.data(), k + 1, tid, NT);
    for (uint32_t tid = 0; tid < NT; tid++)
      gen_acc_update(acc.data(), out.data(), N, k, multibit, tid, NT);
  }
  sample_extract_many_lut(out_base, 0, count, num_many_lut, lut_stride, acc.data(), N, k, N, 0, 1,
                          [](uint64_t x) { return Io::narrow(x); });
}
} // namespace

// torus_bits 64: u64 words; 32: u32 words (the _32 entry points)
extern "C" void emu_bsk_convert_generic(const void *src, uint64_t polys, uint32_t N, int torus_bits, double *dst) {
  cplx *d = reinterpret_cast<cplx *>(dst);
  if (torus_bits == 32)
    emu_bsk_convert_generic_impl(static_cast<const uint32_t *>(src), polys, N, d);
  else
    emu_bsk_convert_generic_impl(static_cast<const uint64_t *>(src), polys, N, d);
}

extern "C" void emu_pbs_generic(const double *bsk_, const void *lut, const void *ct, uint32_t n, uint32_t k,
                                uint32_t N, uint32_t base_log, uint32_t l, uint32_t grouping, int centered_ms,
                                int ties_even, uint32_t num_many_lut, uint32_t lut_stride, uint32_t count,
                                int torus_bits, void *out_base) {
  const cplx *bsk = reinterpret_cast<const cplx *>(bsk_);
  if (torus_bits == 32)
    emu_pbs_generic_impl(bsk, static_cast<const uint32_t *>(lut), static_cast<const uint32_t *>(ct), n, k, N,
                         base_log, l, grouping, centered_ms, ties_even, num_many_lut, lut_stride, count,
                         static_cast<uint32_t *>(out_base));
  else
    emu_pbs_generic_impl(bsk, static_cast<const uint64_t *>(lut), static_cast<const uint64_t *>(ct), n, k, N,
                         base_log, l, grouping, centered_ms, ties_even, num_many_lut, lut_stride, count,
                         static_cast<uint64_t *>(out_base));
}

// ---------------------------------------------------------------------------
// N = 512, l = 1, k <= 4 register kernel (pbs_n512.cuh): one LWE of the CTA,
// 16 (k + 1) threads, replayed with the kernel's phases (pbs_n512_phases.cuh).
// The G LWEs of a CTA and the spare thread groups of a partial last group do
// not change an LWE's words; the key mode does (the two MACs sum the rows in
// different orders).
// ---------------------------------------------------------------------------
// mirrors bsk_convert_n512_kernel for polynomials first .. first + count - 1 of
// the key: src [i][r][c][N] (l = 1), dst [i][c][r][b][q]
extern "C" void emu_bsk_convert_n512(const uint64_t *src, uint32_t k, uint64_t first, uint64_t count,
                                     double *dst_) {
  cplx *dst = reinterpret_cast<cplx *>(dst_);
  const Fft256Tables *tb = tables256();
  const uint64_t P = k + 1;
  std::vector<Regs> R(16);
  std::vector<cplx> xb(P512_M);
  for (uint64_t poly = first; poly < first + count; poly++) {
    const uint64_t c = poly % P, r = (poly / P) % P, i = poly / (P * P);
    for (int u = 0; u < 16; u++) {
      n512_key_load(src + poly * P512_N, u, R[u].v);
      radix16_fwd(R[u].v, tb->pass1);
      xq_store_p1(xb.data(), u, R[u].v);
    }
    for (int u = 0; u < 16; u++) {
      xq_load_p2(xb.data(), u, R[u].v);
      radix16_fwd(R[u].v, tb->pass2[u]);
      spec256_store(dst + ((i * P + c) * P + r) * P512_M, u, R[u].v);
    }
  }
}

// Fourier MAC of the register mode (pbs_n512_kernel<K, 2, false>), restated
// from the kernel's loop: the same sum from row 0 up, the key
// (`krow`: the P rows of this thread's column, element u) streaming through a
// ring of three 8-value chunks; the first two are requested before `barrier`
// (the CTA barrier after which every spectrum of xs_l is stored)
template <int P, typename Load, typename Barrier>
static void n512_mac_regs(cplx v[16], const cplx *xs_l, const cplx *krow, int u,
                           Load load, Barrier barrier) {
  cplx kbuf[3][8];
  auto key_chunk = [&](int ch, cplx (&dst)[8]) {
    const int r = ch >> 1, hb = (ch & 1) * 8;
#pragma unroll
    for (int b = 0; b < 8; b++)
      dst[b] = load(krow + (size_t)r * P512_M + (hb + b) * 16);
  };
  key_chunk(0, kbuf[0]);
  key_chunk(1, kbuf[1]);
  barrier();
  // ---- Fourier MAC: out[b] = sum_r spec_r[b][q] * key[i][p][r][b][q] -------
#pragma unroll
  for (int ch = 0; ch < 2 * P; ch++) {
    const int r = ch >> 1, hb = (ch & 1) * 8;
    if (ch + 2 < 2 * P)
      key_chunk(ch + 2, kbuf[(ch + 2) % 3]);
#pragma unroll
    for (int b = 0; b < 8; b++) {
      const cplx f = xs_l[(size_t)r * P512_M + (hb + b) * 16 + u];
      v[hb + b] = r == 0 ? cmul(f, kbuf[ch % 3][b]) : cfma(f, kbuf[ch % 3][b], v[hb + b]);
    }
  }
}

template <int P>
static void emu_pbs_n512_impl(const cplx *bsk, const uint64_t *lut, const uint64_t *ct, uint32_t n,
                              uint32_t base_log, int centered_ms, bool ring, uint32_t num_many_lut,
                              uint32_t lut_stride, uint32_t count, uint64_t *out_base) {
  const Fft256Tables *tb = tables256();
  const uint32_t log_mod = 10;
  std::vector<uint16_t> a_hat(n);
  CenteredMsSums sums;
  for (uint32_t i = 0; i < n; i++) {
    a_hat[i] = (uint16_t)modulus_switch_u64(ct[i], log_mod);
    if (centered_ms)
      sums.add(ct[i], log_mod);
  }
  const uint32_t b_hat = ms_b_hat(ct[n], centered_ms, &sums.half, &sums.dbl, 1, log_mod);
  std::vector<uint32_t> acc(P * P512_N);
  for (uint32_t j = 0; j < (uint32_t)(P * P512_N); j++) {
    const uint32_t r = j >> 9, jj = j & (P512_N - 1);
    acc[r * P512_N + jj] = torus64_to_32(rot_div_coeff(lut + r * P512_N, P512_N, jj, b_hat));
  }
  std::vector<Regs> R(16 * P);
  std::vector<cplx> xs(P * P512_M);
#define N512_THREADS                                                           \
  for (int tl = 0; tl < 16 * P; tl++) {                                        \
    const int p = tl >> 4, u = tl & 15;                                        \
    cplx *v = R[tl].v;                                                         \
    uint32_t *acc_p = acc.data() + p * P512_N;                                 \
    cplx *xs_p = xs.data() + p * P512_M;                                       \
    (void)v; (void)acc_p; (void)xs_p;
  N512_THREADS
    for (int j1 = 0; j1 < 16; j1++) {
      R[tl].own[j1] = acc_p[16 * j1 + u];
      R[tl].own[16 + j1] = acc_p[16 * j1 + u + P512_M];
    }
  END_THREADS
  const size_t key_step = (size_t)P * P * P512_M;
  for (uint32_t i = 0; i < n; i++) { // every step, a = 0 included, as the kernel
    const uint32_t a = a_hat[i];
    N512_THREADS
      n512_load_digits(acc_p, u, a, base_log, R[tl].own, v);
      radix16_fwd(v, tb->pass1);
      xq_store_p1(xs_p, u, v);
    END_THREADS
    N512_THREADS
      xq_load_p2(xs_p, u, v);
      radix16_fwd(v, tb->pass2[u]);
    END_THREADS
    N512_THREADS
      spec256_store(xs_p, u, v);
    END_THREADS
    N512_THREADS
      const cplx *block = bsk + (size_t)i * key_step + (size_t)p * (P * P512_M);
      if (ring)
        n512_mac_ring<P>(v, xs.data(), block, p, u, HostLoader());
      else
        n512_mac_regs<P>(v, xs.data(), block + u, u, HostLoader(), [] {});
    END_THREADS
    N512_THREADS
      radix16_inv(v, tb->pass2[u]);
      xq_store_p2(xs_p, u, v);
    END_THREADS
    N512_THREADS
      xq_load_p1(xs_p, u, v);
      radix16_inv(v, tb->pass1);
      n512_acc_update(acc_p, u, v, R[tl].own);
    END_THREADS
  }
  sample_extract_many_lut(out_base, 0, count, num_many_lut, lut_stride, acc.data(), P512_N, P - 1, P512_N, 0, 1,
                          Torus32To64());
}

// ring != 0: the TMA key-ring instances (n512<k,G,true>); 0: the register
// key-ring instances (n512<k,2,false>)
extern "C" void emu_pbs_n512(const double *bsk_, const uint64_t *lut, const uint64_t *ct, uint32_t n, uint32_t k,
                             uint32_t base_log, int centered_ms, int ring, uint32_t num_many_lut,
                             uint32_t lut_stride, uint32_t count, uint64_t *out_base) {
  const cplx *bsk = reinterpret_cast<const cplx *>(bsk_);
  switch (k) {
  case 1: return emu_pbs_n512_impl<2>(bsk, lut, ct, n, base_log, centered_ms, ring, num_many_lut, lut_stride, count, out_base);
  case 2: return emu_pbs_n512_impl<3>(bsk, lut, ct, n, base_log, centered_ms, ring, num_many_lut, lut_stride, count, out_base);
  case 3: return emu_pbs_n512_impl<4>(bsk, lut, ct, n, base_log, centered_ms, ring, num_many_lut, lut_stride, count, out_base);
  default: return emu_pbs_n512_impl<5>(bsk, lut, ct, n, base_log, centered_ms, ring, num_many_lut, lut_stride, count, out_base);
  }
}
