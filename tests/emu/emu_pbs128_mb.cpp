// emu_pbs128_mb.cpp -- CPU model of the multi-bit 128-bit PBS kernel's folded
// MAC, TEST INFRASTRUCTURE ONLY: the B200_HD phases of
// tfhe-rs_b200/csrc/pbs128_phases.cuh compiled by g++ (key conversion,
// double-double transform, p128_mb_mac over the double-double root table,
// inverse transform and assignment), to pin the fold's error against the
// exact product of tests/emu/pbs128_mb_exact.cpp; and a replay of the kernel
// (pbs128_multibit.cuh) phase by phase with the kernel's thread count, which
// tests/test_noise_squashing_multibit.py compares with the GPU word for word
// (the key conversion is the classic one, replayed by emu128_bsk_convert of
// tests/emu/emu_pbs128.cpp).  u128 words cross the ABI as two u64, low then
// high.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../tfhe-rs_b200/csrc/pbs128_phases.cuh"

extern "C" {

// d * sum_b X^{degs[b]} G_b mod (X^N + 1, 2^128), b < nggsw (degs[0] is not
// read: GGSW 0 is not rotated), G: nggsw polynomials of N words
void emu128_mb_product(const u128 *d, const u128 *G, const uint32_t *degs,
                       uint32_t nggsw, uint32_t N, u128 *out) {
  const uint32_t M = N / 2;
  uint32_t logM = 0;
  while ((1u << logM) < M)
    logM++;
  std::vector<ddc> tw(M), root(4 * (size_t)M), Gs((size_t)nggsw * M), F(M), O(M);
  b200_fill_dd_twiddles(logM, tw.data());
  b200_fill_dd_roots(logM, root.data());
  for (uint32_t b = 0; b < nggsw; b++) {
    p128_load_key_poly(G + (size_t)b * N, Gs.data() + (size_t)b * M, M, 0, 1);
    for (uint32_t L = 1; L <= logM; L++)
      p128_fwd_level(Gs.data() + (size_t)b * M, logM, L, tw.data(), 0, 1);
  }
  for (uint32_t j = 0; j < M; j++)
    F[j] = ddc_make(i128_to_dd(d[j]), i128_to_dd(d[j + M]));
  for (uint32_t L = 1; L <= logM; L++)
    p128_fwd_level(F.data(), logM, L, tw.data(), 0, 1);
  p128_mb_mac(F.data(), O.data(), Gs.data(), M, nggsw, degs, root.data(), logM,
              0, true, 0, 1);
  for (uint32_t L = logM; L >= 1; L--)
    p128_inv_level(O.data(), logM, L, tw.data(), 0, 1);
  p128_acc_assign(out, O.data(), M, 0, 1);
}

// the kernel's degrees of GGSWs 0..2^g-1 of one group of g mask words
void emu128_mb_degrees(const uint64_t *mask, uint32_t g, uint32_t log_mod,
                       uint32_t *degs) {
  for (uint32_t b = 0; b < (1u << g); b++)
    degs[b] = p128_mb_degree(mask, g, b, log_mod);
}

// mirrors pbs128_mb_kernel for one sample: u64 LWE of n + 1 words in, u128
// LWE of k N + 1 words out; bsk is the converted key
void emu128_mb_pbs(const double *bsk_, const u128 *lut, const uint64_t *ct,
                   uint32_t n, uint32_t k, uint32_t N, uint32_t g,
                   uint32_t base_log, uint32_t l, u128 *lwe_out) {
  const ddc *bsk = reinterpret_cast<const ddc *>(bsk_);
  const uint32_t NT = 512; // PBS128_THREADS
  const uint32_t M = N / 2, nggsw = 1u << g;
  uint32_t logM = 0;
  while ((1u << logM) < M)
    logM++;
  const uint32_t log_mod = logM + 2;
  std::vector<ddc> tw(M), root(4 * (size_t)M);
  b200_fill_dd_twiddles(logM, tw.data());
  b200_fill_dd_roots(logM, root.data());
  const size_t ggsw_len = (size_t)l * (k + 1) * (k + 1) * M;
  std::vector<u128> acc((size_t)(k + 1) * N);
  std::vector<ddc> buf(M), out((size_t)(k + 1) * M);
  uint32_t degs[16];
  rotate_lut(acc.data(), N, lut, k + 1, N, modulus_switch_u64(ct[n], log_mod), 0,
             1, SameWord());
  for (uint32_t i = 0; i < n / g; i++) {
    for (uint32_t b = 0; b < nggsw; b++)
      degs[b] = p128_mb_degree(ct + (size_t)i * g, g, b, log_mod);
    const ddc *group = bsk + (size_t)i * nggsw * ggsw_len;
    for (uint32_t t = 0; t < l; t++)
      for (uint32_t r = 0; r <= k; r++) {
        for (uint32_t tid = 0; tid < NT; tid++)
          p128_decompose_acc(acc.data() + (size_t)r * N, buf.data(), N, base_log, l, t, tid, NT);
        for (uint32_t L = 1; L <= logM; L++)
          for (uint32_t tid = 0; tid < NT; tid++)
            p128_fwd_level(buf.data(), logM, L, tw.data(), tid, NT);
        for (uint32_t tid = 0; tid < NT; tid++)
          p128_mb_mac(buf.data(), out.data(), group + ((size_t)t * (k + 1) + r) * (k + 1) * M, ggsw_len,
                      nggsw, degs, root.data(), logM, k, t == 0 && r == 0, tid, NT);
      }
    for (uint32_t c = 0; c <= k; c++) {
      memcpy(buf.data(), out.data() + (size_t)c * M, M * sizeof(ddc));
      for (uint32_t L = logM; L >= 1; L--)
        for (uint32_t tid = 0; tid < NT; tid++)
          p128_inv_level(buf.data(), logM, L, tw.data(), tid, NT);
      for (uint32_t tid = 0; tid < NT; tid++)
        p128_acc_assign(acc.data() + (size_t)c * N, buf.data(), M, tid, NT);
    }
  }
  sample_extract_lwe(lwe_out, acc.data(), N, k, N, 0, 0, 1, SameWord());
}

} // extern "C"
