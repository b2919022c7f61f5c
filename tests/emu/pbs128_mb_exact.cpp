// pbs128_mb_exact.cpp -- the EXACT multi-bit u128 blind rotation, TEST
// INFRASTRUCTURE ONLY.
//
// Builds on the exact classic model (pbs128_exact.cpp: schoolbook negacyclic
// products in unsigned __int128, its own decomposition, rotation and TUniform
// key generation), so nothing here comes from the kernel's sources either.
// tfhe-rs' multi-bit algorithm (core_crypto/algorithms/
// lwe_multi_bit_bootstrap_key_generation.rs combine_key_bits,
// lwe_multi_bit_programmable_bootstrapping.rs modulus_switch_multi_bit,
// selection_bit): GGSW b of group j encrypts prod_u (s_{jg+u} if bit g-1-u of
// b is set, else 1 - s_{jg+u}); each step builds the bundle
// sum_b X^{deg_b} GGSW_b exactly and multiplies the accumulator's digits by it.
#include "pbs128_exact.cpp"

namespace {

// the plain modulus switch of a u64 word to [0, 2^log_mod)
static uint32_t switch_u64(uint64_t x, uint32_t log_mod) {
  return (uint32_t)(((x >> (63 - log_mod)) + 1) >> 1) & ((1u << log_mod) - 1);
}

} // namespace

extern "C" {

// multi-bit BSK [n/g][2^g][l][k+1][k+1][N] u128; level index t holds level
// l - t, as p128_gen_bsk
void p128mb_gen_bsk(uint64_t seed, const uint64_t *lwe_sk, uint32_t n,
                    const uint64_t *glwe_sk, uint32_t k, uint32_t N,
                    uint32_t base_log, uint32_t l, uint32_t g,
                    uint32_t noise_log2, u128 *bsk) {
  const size_t row = (size_t)(k + 1) * N, ggsw_len = (size_t)l * (k + 1) * row;
  const uint32_t nggsw = 1u << g, groups = n / g;
#pragma omp parallel for schedule(dynamic, 1)
  for (uint32_t gi = 0; gi < groups * nggsw; gi++) {
    const uint32_t j = gi / nggsw, b = gi % nggsw;
    Rng rng{seed ^ (0x5A5A5A5Aull * (gi + 1))};
    u128 m = 1;
    for (uint32_t u = 0; u < g; u++) {
      const uint64_t bit = (b >> (g - 1 - u)) & 1u;
      m *= (u128)(lwe_sk[j * g + u] ^ bit ^ 1u);
    }
    for (uint32_t t = 0; t < l; t++) {
      const uint32_t level = l - t;
      const u128 factor = ((u128)0 - m) << (128 - base_log * level);
      for (uint32_t r = 0; r <= k; r++) {
        u128 *gg = bsk + (size_t)gi * ggsw_len + ((size_t)t * (k + 1) + r) * row;
        u128 *body = gg + (size_t)k * N;
        memset(body, 0, N * sizeof(u128));
        if (r < k)
          for (uint32_t i = 0; i < N; i++)
            body[i] = (u128)glwe_sk[(size_t)r * N + i] * factor;
        else
          body[0] = (u128)0 - factor;
        glwe_encrypt_assign(rng, glwe_sk, k, N, noise_log2, gg, body);
      }
    }
  }
}

// the 2^g - 1 degrees of GGSWs 1..2^g-1 of one group of g mask words
void p128mb_degrees(const uint64_t *mask, uint32_t g, uint32_t log_mod,
                    uint32_t *degs) {
  for (uint32_t b = 1; b < (1u << g); b++) {
    uint64_t sum = 0;
    for (uint32_t u = 0; u < g; u++)
      if ((b >> (g - 1 - u)) & 1u)
        sum += mask[u];
    degs[b - 1] = switch_u64(sum, log_mod);
  }
}

// exact multi-bit PBS of `count` u64 LWEs cts[s][0..n] into u128 LWEs of
// k*N + 1 words: plain modulus switch of the body, n / g steps
void p128mb_pbs_exact(const u128 *bsk, const u128 *lut, const uint64_t *cts,
                      uint32_t count, uint32_t n, uint32_t k, uint32_t N,
                      uint32_t g, uint32_t base_log, uint32_t l,
                      u128 *lwe_out) {
  const size_t row = (size_t)(k + 1) * N, ggsw_len = (size_t)l * (k + 1) * row;
  const uint32_t nggsw = 1u << g;
  uint32_t log_mod = 1;
  while ((1u << log_mod) < 2 * N)
    log_mod++;
#pragma omp parallel for schedule(dynamic, 1)
  for (uint32_t s = 0; s < count; s++) {
    const uint64_t *ct = cts + (size_t)s * (n + 1);
    std::vector<u128> acc(row), nacc(row), bundle(ggsw_len), rot(N),
        digits((size_t)(k + 1) * l * N);
    std::vector<i128> d(l);
    std::vector<uint32_t> degs(nggsw);
    const uint32_t b_hat = switch_u64(ct[n], log_mod);
    for (uint32_t r = 0; r <= k; r++)
      monomial_mul(acc.data() + (size_t)r * N, lut + (size_t)r * N, N,
                   (2 * N - b_hat) % (2 * N));
    for (uint32_t j = 0; j < n / g; j++) {
      p128mb_degrees(ct + (size_t)j * g, g, log_mod, degs.data() + 1);
      degs[0] = 0;
      const u128 *grp = bsk + (size_t)j * nggsw * ggsw_len;
      memcpy(bundle.data(), grp, ggsw_len * sizeof(u128));
      for (uint32_t b = 1; b < nggsw; b++)
        for (size_t p = 0; p < ggsw_len / N; p++) {
          monomial_mul(rot.data(), grp + (size_t)b * ggsw_len + p * N, N, degs[b]);
          for (uint32_t i = 0; i < N; i++)
            bundle[p * N + i] += rot[i];
        }
      for (uint32_t r = 0; r <= k; r++)
        for (uint32_t i = 0; i < N; i++) {
          decompose_word(acc[(size_t)r * N + i], base_log, l, d.data());
          for (uint32_t t = 0; t < l; t++)
            digits[((size_t)r * l + t) * N + i] = (u128)d[t];
        }
      std::fill(nacc.begin(), nacc.end(), (u128)0);
      for (uint32_t r = 0; r <= k; r++)
        for (uint32_t t = 0; t < l; t++) {
          const u128 *gg = bundle.data() + ((size_t)t * (k + 1) + r) * row;
          for (uint32_t c = 0; c <= k; c++)
            negacyclic_mul_add(nacc.data() + (size_t)c * N,
                               digits.data() + ((size_t)r * l + t) * N,
                               gg + (size_t)c * N, N);
        }
      acc.swap(nacc);
    }
    u128 *o = lwe_out + (size_t)s * ((size_t)k * N + 1);
    for (uint32_t r = 0; r < k; r++)
      for (uint32_t t = 0; t < N; t++)
        o[(size_t)r * N + t] = t == 0 ? acc[(size_t)r * N] : (u128)0 - acc[(size_t)r * N + N - t];
    o[(size_t)k * N] = acc[(size_t)k * N];
  }
}

} // extern "C"
