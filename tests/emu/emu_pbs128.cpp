// emu_pbs128.cpp -- CPU model of the 128-bit PBS kernel's arithmetic, TEST
// INFRASTRUCTURE ONLY: the B200_HD phases of tfhe-rs_b200/csrc/pbs128_phases.cuh
// compiled by g++ -- the double-double transform, its twiddles, the kernel's
// u128 decomposition -- and the same product through the plain fp64
// transform of the 64-bit kernels, to pin the transform's error on the CPU
// against the exact product of tests/emu/pbs128_exact.cpp; and a replay of the
// kernel (pbs128.cuh) and of its key conversion, phase by phase with the
// kernel's thread count, which tests/test_gpu_replay_words.py compares with the
// GPU word for word.  u128 words cross the ABI as two u64, low then high.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../tfhe-rs_b200/csrc/pbs128_phases.cuh"

extern "C" {

// the kernel's digits of each word, least significant first: digits[i][t]
void emu128_decompose(const u128 *x, uint32_t count, uint32_t base_log,
                      uint32_t l, u128 *digits) {
  for (uint32_t i = 0; i < count; i++) {
    u128 s = decomp128_init_state(x[i], base_log, l);
    for (uint32_t t = 0; t < l; t++)
      digits[(size_t)i * l + t] = (u128)decomp128_next_digit(&s, base_log);
  }
}

// ---- the transforms -----------------------------------------------------------
// double-double twiddles of size 2^logM: M - 1 entries of 4 doubles
void emu128_twiddles(uint32_t logM, double *out) {
  std::vector<ddc> tw((size_t)1 << logM);
  b200_fill_dd_twiddles(logM, tw.data());
  memcpy(out, tw.data(), ((size_t)1 << logM) * sizeof(ddc));
}

// d * g mod (X^N + 1, 2^128) through the kernel's double-double transform:
// key polynomial as at key conversion, digits as at decomposition, one MAC,
// inverse transform and rounding into a zero accumulator
void emu128_product(const u128 *d, const u128 *g, uint32_t N, u128 *out) {
  const uint32_t M = N / 2;
  uint32_t logM = 0;
  while ((1u << logM) < M)
    logM++;
  std::vector<ddc> tw(M), G(M), F(M), O(M);
  b200_fill_dd_twiddles(logM, tw.data());
  p128_load_key_poly(g, G.data(), M, 0, 1);
  for (uint32_t j = 0; j < M; j++)
    F[j] = ddc_make(i128_to_dd(d[j]), i128_to_dd(d[j + M]));
  for (uint32_t L = 1; L <= logM; L++) {
    p128_fwd_level(G.data(), logM, L, tw.data(), 0, 1);
    p128_fwd_level(F.data(), logM, L, tw.data(), 0, 1);
  }
  p128_mac(F.data(), O.data(), G.data(), M, 0, true, 0, 1);
  for (uint32_t L = logM; L >= 1; L--)
    p128_inv_level(O.data(), logM, L, tw.data(), 0, 1);
  memset(out, 0, N * sizeof(u128));
  p128_acc_add(out, O.data(), M, 0, 1);
}

// the same product through the fp64 transform of the 64-bit kernels
// (pbs_generic_phases.cuh), every value rounded to a double: the negative
// control of the double-double transform
void emu64_product(const u128 *d, const u128 *g, uint32_t N, u128 *out) {
  const uint32_t M = N / 2;
  uint32_t logM = 0;
  while ((1u << logM) < M)
    logM++;
  std::vector<cplx> tw(M), G(M), F(M);
  b200_fill_generic_tables(logM, tw.data(), nullptr);
  const auto to_d = [](u128 x) { const dd v = i128_to_dd(x); return v.hi + v.lo; };
  for (uint32_t j = 0; j < M; j++) {
    G[j] = cmake(to_d(g[j]) / M, to_d(g[j + M]) / M);
    F[j] = cmake(to_d(d[j]), to_d(d[j + M]));
  }
  for (uint32_t L = 1; L <= logM; L++) {
    gen_fwd_level(G.data(), logM, L, tw.data(), 1, 0, 1);
    gen_fwd_level(F.data(), logM, L, tw.data(), 1, 0, 1);
  }
  for (uint32_t j = 0; j < M; j++)
    F[j] = cmul(F[j], G[j]);
  for (uint32_t L = logM; L >= 1; L--)
    gen_inv_level(F.data(), logM, L, tw.data(), 1, 0, 1);
  for (uint32_t j = 0; j < M; j++) {
    out[j] = dd_to_u128(dd_make(F[j].re, 0.0));
    out[j + M] = dd_to_u128(dd_make(F[j].im, 0.0));
  }
}

// ---- the kernel ----------------------------------------------------------------
// the double-double twiddles of every size pbs128_kernel runs (N = 256 ..
// 4096), filled once before any caller reads them: the replays are called from
// many threads at once
static const ddc *dd_tables(uint32_t logM) {
  static const std::vector<std::vector<ddc>> *all = [] {
    auto *v = new std::vector<std::vector<ddc>>(12);
    for (uint32_t L = 7; L <= 11; L++) {
      (*v)[L].resize((size_t)1 << L);
      b200_fill_dd_twiddles(L, (*v)[L].data());
    }
    return v;
  }();
  return (*all)[logM].data();
}
static uint32_t log2_exact(uint32_t x) {
  uint32_t r = 0;
  while ((1u << r) < x)
    r++;
  return r;
}

// mirrors bsk_convert_128_kernel over `polys` polynomials of N u128 words
void emu128_bsk_convert(const u128 *src, uint64_t polys, uint32_t N, double *dst_) {
  ddc *dst = reinterpret_cast<ddc *>(dst_);
  const uint32_t M = N / 2, logM = log2_exact(M);
  const ddc *tw = dd_tables(logM);
  std::vector<ddc> buf(M);
  for (uint64_t b = 0; b < polys; b++) {
    for (uint32_t tid = 0; tid < 256; tid++)
      p128_load_key_poly(src + b * N, buf.data(), M, tid, 256);
    for (uint32_t L = 1; L <= logM; L++)
      for (uint32_t tid = 0; tid < 256; tid++)
        p128_fwd_level(buf.data(), logM, L, tw, tid, 256);
    memcpy(dst + b * M, buf.data(), M * sizeof(ddc));
  }
}

// mirrors pbs128_kernel for one sample: u64 LWE of n + 1 words in, u128 LWE of
// k N + 1 words out
void emu128_pbs(const double *bsk_, const u128 *lut, const uint64_t *ct, uint32_t n, uint32_t k, uint32_t N,
                uint32_t base_log, uint32_t l, int centered_ms, u128 *lwe_out) {
  const ddc *bsk = reinterpret_cast<const ddc *>(bsk_);
  const uint32_t NT = 512; // PBS128_THREADS
  const uint32_t M = N / 2, logM = log2_exact(M), log_mod = logM + 2;
  const ddc *tw = dd_tables(logM);
  const size_t ggsw_len = (size_t)l * (k + 1) * (k + 1) * M;
  std::vector<u128> acc((size_t)(k + 1) * N);
  std::vector<ddc> buf(M), out((size_t)(k + 1) * M);
  std::vector<uint32_t> a_hat(n);
  CenteredMsSums sums;
  for (uint32_t i = 0; i < n; i++) {
    a_hat[i] = modulus_switch_u64(ct[i], log_mod);
    if (centered_ms)
      sums.add(ct[i], log_mod);
  }
  const uint32_t b_hat = ms_b_hat(ct[n], centered_ms, &sums.half, &sums.dbl, 1, log_mod);
  rotate_lut(acc.data(), N, lut, k + 1, N, b_hat, 0, 1, SameWord());
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t a = a_hat[i];
    if (a == 0)
      continue;
    const ddc *ggsw = bsk + (size_t)i * ggsw_len;
    for (uint32_t t = 0; t < l; t++)
      for (uint32_t r = 0; r <= k; r++) {
        for (uint32_t tid = 0; tid < NT; tid++)
          p128_decompose(acc.data() + (size_t)r * N, buf.data(), N, a, base_log, l, t, tid, NT);
        for (uint32_t L = 1; L <= logM; L++)
          for (uint32_t tid = 0; tid < NT; tid++)
            p128_fwd_level(buf.data(), logM, L, tw, tid, NT);
        for (uint32_t tid = 0; tid < NT; tid++)
          p128_mac(buf.data(), out.data(), ggsw + ((size_t)t * (k + 1) + r) * (k + 1) * M, M, k,
                   t == 0 && r == 0, tid, NT);
      }
    for (uint32_t c = 0; c <= k; c++) {
      memcpy(buf.data(), out.data() + (size_t)c * M, M * sizeof(ddc));
      for (uint32_t L = logM; L >= 1; L--)
        for (uint32_t tid = 0; tid < NT; tid++)
          p128_inv_level(buf.data(), logM, L, tw, tid, NT);
      for (uint32_t tid = 0; tid < NT; tid++)
        p128_acc_add(acc.data() + (size_t)c * N, buf.data(), M, tid, NT);
    }
  }
  sample_extract_lwe(lwe_out, acc.data(), N, k, N, 0, 0, 1, SameWord());
}

} // extern "C"
