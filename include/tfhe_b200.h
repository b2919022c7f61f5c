/*
 * tfhe_b200.h -- C ABI of libtfhe_cuda_backend_b200.so
 *
 * Drop-in boundary: every symbol below has the NAME and SIGNATURE of the
 * symbol of the same name exported by tfhe-rs' `backends/tfhe-cuda-backend`
 * (static lib libtfhe_cuda_backend.a, bound from Rust by bindgen in
 * backends/tfhe-cuda-backend/src/bindings.rs).  The citation after each
 * declaration is the reference header that declares it, relative to
 * backends/ of tfhe-rs.  All `void *` ciphertext / key / index
 * arguments are DEVICE pointers unless stated; `stream` is a cudaStream_t.
 *
 * Conventions kept from the reference:
 *   - no return codes: any CUDA error or violated precondition prints to
 *     stderr and abort()s;
 *   - every call is asynchronous on `stream` and first selects `gpu_index`;
 *   - the caller owns all ciphertext / key / index buffers, the callee owns
 *     only the scratch object between scratch_* and cleanup_*;
 *   - the Fourier bootstrap key layout inside `dest` is private to the
 *     engine but fits the caller-allocated n*(k+1)^2*l*N f64 words.
 *
 * Symbols prefixed b200_ are additions (test / measurement entry points and
 * the multi-GPU key broadcast); the reference has no equivalent.
 */
#ifndef TFHE_B200_H
#define TFHE_B200_H

#include <stdbool.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* tfhe-cuda-backend/cuda/include/pbs/pbs_enums.h:4-6 */
typedef enum { MULTI_BIT = 0, CLASSICAL = 1 } PBS_TYPE;
typedef enum { DEFAULT = 0, CG = 1, TBC = 2 } PBS_VARIANT;
typedef enum { NO_REDUCTION = 0, CENTERED = 1 } PBS_MS_REDUCTION_T;

/* ---- device helpers: tfhe-cuda-common/cuda/include/device.h:59-88 ------- */
void *cuda_create_stream_ffi(uint32_t gpu_index);
void cuda_destroy_stream(void *stream, uint32_t gpu_index);
void cuda_synchronize_stream(void *stream, uint32_t gpu_index);
uint32_t cuda_is_available(void);
void *cuda_malloc(uint64_t size, uint32_t gpu_index);
void *cuda_malloc_async(uint64_t size, void *stream, uint32_t gpu_index);
bool cuda_check_valid_malloc(uint64_t size, uint32_t gpu_index);
uint64_t cuda_device_total_memory(uint32_t gpu_index);
void cuda_memcpy_async_to_gpu(void *dest, const void *src, uint64_t size,
                              void *stream, uint32_t gpu_index);
void cuda_memcpy_async_gpu_to_gpu(void *dest, void const *src, uint64_t size,
                                  void *stream, uint32_t gpu_index);
void cuda_memcpy_gpu_to_gpu(void *dest, void const *src, uint64_t size,
                            uint32_t gpu_index);
void cuda_memcpy_async_to_cpu(void *dest, const void *src, uint64_t size,
                              void *stream, uint32_t gpu_index);
void cuda_memset_async(void *dest, uint64_t val, uint64_t size, void *stream,
                       uint32_t gpu_index);
int cuda_get_number_of_gpus(void);
int cuda_get_number_of_sms(void);
void cuda_synchronize_device(uint32_t gpu_index);
void cuda_drop(void *ptr, uint32_t gpu_index);
void cuda_drop_async(void *ptr, void *stream, uint32_t gpu_index);
uint32_t cuda_get_max_shared_memory(uint32_t gpu_index);

/* ---- classic PBS: tfhe-cuda-backend/cuda/include/pbs/programmable_bootstrap.h */
/* :50-53  src = HOST pointer, standard-domain BSK [i][level][row][col][N] u64 */
void cuda_convert_lwe_programmable_bootstrap_key_64_async(
    void *stream, uint32_t gpu_index, void *dest, void const *src,
    uint32_t input_lwe_dim, uint32_t glwe_dim, uint32_t level_count,
    uint32_t polynomial_size);
/* :60-64  returns the scratch bytes; allocate_gpu_memory=false = size query */
uint64_t scratch_cuda_programmable_bootstrap_64_async(
    void *stream, uint32_t gpu_index, int8_t **buffer, uint32_t lwe_dimension,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t level_count,
    uint32_t input_lwe_ciphertext_count, bool allocate_gpu_memory,
    PBS_MS_REDUCTION_T noise_reduction_type);
/* :81-88 */
void cuda_programmable_bootstrap_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lut_vector,
    void const *lut_vector_indexes, void const *lwe_array_in,
    void const *lwe_input_indexes, void const *bootstrapping_key,
    int8_t *buffer, uint32_t lwe_dimension, uint32_t glwe_dimension,
    uint32_t polynomial_size, uint32_t base_log, uint32_t level_count,
    uint32_t num_samples, uint32_t num_many_lut, uint32_t lut_stride);
/* :97-98 */
void cleanup_cuda_programmable_bootstrap_64(void *stream, uint32_t gpu_index,
                                            int8_t **pbs_buffer);

/* u32 torus, programmable_bootstrap.h:47-50,72-79: key words, ciphertexts,
 * accumulators and the three index vectors are u32.  The reference exposes no
 * scratch function for this variant; `buffer` is a scratch object made by
 * scratch_cuda_programmable_bootstrap_64_async with the same (k, N, l).  Words
 * are widened to the top half of a u64 inside the kernel and rounded back to 32
 * bits on output (the blind rotation itself is the 64-bit path). */
void cuda_convert_lwe_programmable_bootstrap_key_32_async(
    void *stream, uint32_t gpu_index, void *dest, void const *src,
    uint32_t input_lwe_dim, uint32_t glwe_dim, uint32_t level_count,
    uint32_t polynomial_size);
void cuda_programmable_bootstrap_lwe_ciphertext_vector_32_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lut_vector,
    void const *lut_vector_indexes, void const *lwe_array_in,
    void const *lwe_input_indexes, void const *bootstrapping_key,
    int8_t *buffer, uint32_t lwe_dimension, uint32_t glwe_dimension,
    uint32_t polynomial_size, uint32_t base_log, uint32_t level_count,
    uint32_t num_samples, uint32_t num_many_lut, uint32_t lut_stride);

/* u128 torus (noise squashing), programmable_bootstrap.h:57-60,68-72,92-97,
 * 102-103.  u128 words are two u64, low then high.  src = HOST standard-domain
 * key [i][level][row][col][N] of u128; dest holds n*(k+1)^2*l*N*2 f64 words
 * (one double-double complex per frequency, layout private).  The PBS reads
 * num_samples u64 LWEs of lwe_dimension + 1 words, one u128 GLWE LUT of
 * (k+1)*N words, and writes u128 LWEs of k*N + 1 words; indexes are trivial.
 * The modulus switch is the 64-bit one, centered when the scratch object was
 * made with CENTERED.  Shapes: N a power of two in [256, 4096], k >= 1,
 * l >= 1, base_log * l <= 128; anything else aborts.  The blind rotation runs
 * in double-double arithmetic (DESIGN.md section 8f). */
void cuda_convert_lwe_programmable_bootstrap_key_128_async(
    void *stream, uint32_t gpu_index, void *dest, void const *src,
    uint32_t input_lwe_dim, uint32_t glwe_dim, uint32_t level_count,
    uint32_t polynomial_size);
uint64_t scratch_cuda_programmable_bootstrap_128_async(
    void *stream, uint32_t gpu_index, int8_t **buffer, uint32_t lwe_dimension,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t level_count,
    uint32_t input_lwe_ciphertext_count, bool allocate_gpu_memory,
    PBS_MS_REDUCTION_T noise_reduction_type);
void cuda_programmable_bootstrap_128_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lut_vector, void const *lwe_array_in,
    void const *bootstrapping_key, int8_t *buffer, uint32_t lwe_dimension,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t base_log,
    uint32_t level_count, uint32_t num_samples);
void cleanup_cuda_programmable_bootstrap_128(void *stream, uint32_t gpu_index,
                                             int8_t **pbs_buffer);

/* multi-bit u128 torus (noise squashing with grouped keys),
 * programmable_bootstrap_multibit.h:18-21, 64-80.  src = HOST standard-domain
 * key [group][2^g][level][row][col][N] of u128 (GGSW b of a group encrypts the
 * product of s_u or 1 - s_u as bit g - 1 - u of b is set or clear); dest holds
 * as many f64 words as src has u64 (layout private).  The PBS reads
 * num_samples u64 LWEs, LWE lwe_input_indexes[s] (u64) for sample s, and
 * writes u128 LWEs of k*N + 1 words to rows lwe_output_indexes[s] (u64); one
 * u128 GLWE LUT of (k+1)*N words serves every sample.  The modulus switch is
 * the plain one; the degrees are tfhe-rs' modulus_switch_multi_bit.  Shapes:
 * those of the classic 128-bit PBS, grouping factor 2, 3 or 4, lwe_dimension
 * a positive multiple of it, num_many_lut = 1; anything else aborts.  One
 * launch (csrc/pbs128_multibit.cuh, DESIGN.md section 8f); b200_last_pbs_
 * kernel reports "pbs128_mb<N>". */
void cuda_convert_lwe_multi_bit_programmable_bootstrap_key_128_async(
    void *stream, uint32_t gpu_index, void *dest, void const *src,
    uint32_t input_lwe_dim, uint32_t glwe_dim, uint32_t level_count,
    uint32_t polynomial_size, uint32_t grouping_factor);
uint64_t scratch_cuda_multi_bit_programmable_bootstrap_128_async(
    void *stream, uint32_t gpu_index, int8_t **buffer, uint32_t glwe_dimension,
    uint32_t polynomial_size, uint32_t level_count,
    uint32_t input_lwe_ciphertext_count, bool allocate_gpu_memory);
void cuda_multi_bit_programmable_bootstrap_128_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lut_vector,
    void const *lwe_array_in, void const *lwe_input_indexes,
    void const *bootstrapping_key, int8_t *mem_ptr, uint32_t lwe_dimension,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t grouping_factor,
    uint32_t base_log, uint32_t level_count, uint32_t num_samples,
    uint32_t num_many_lut, uint32_t lut_stride);
void cleanup_cuda_multi_bit_programmable_bootstrap_128(void *stream,
                                                       const uint32_t gpu_index,
                                                       int8_t **buffer);

/* ---- multi-bit PBS: .../include/pbs/programmable_bootstrap_multibit.h:9-42 */
bool has_support_to_cuda_programmable_bootstrap_cg_multi_bit(
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t level_count,
    uint32_t num_samples, uint32_t max_shared_memory);
void cuda_convert_lwe_multi_bit_programmable_bootstrap_key_64_async(
    void *stream, uint32_t gpu_index, void *dest, void const *src,
    uint32_t input_lwe_dim, uint32_t glwe_dim, uint32_t level_count,
    uint32_t polynomial_size, uint32_t grouping_factor);
uint64_t scratch_cuda_multi_bit_programmable_bootstrap_64_async(
    void *stream, uint32_t gpu_index, int8_t **pbs_buffer,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t level_count,
    uint32_t input_lwe_ciphertext_count, bool allocate_gpu_memory);
void cuda_multi_bit_programmable_bootstrap_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lut_vector,
    void const *lut_vector_indexes, void const *lwe_array_in,
    void const *lwe_input_indexes, void const *bootstrapping_key,
    int8_t *buffer, uint32_t lwe_dimension, uint32_t glwe_dimension,
    uint32_t polynomial_size, uint32_t grouping_factor, uint32_t base_log,
    uint32_t level_count, uint32_t num_samples, uint32_t num_many_lut,
    uint32_t lut_stride);
void cleanup_cuda_multi_bit_programmable_bootstrap_64(void *stream,
                                                      uint32_t gpu_index,
                                                      int8_t **pbs_buffer);

/* ---- keyswitch: .../include/keyswitch/keyswitch.h:18-44 ----------------- */
void cuda_keyswitch_lwe_ciphertext_vector_64_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lwe_array_in,
    void const *lwe_input_indexes, void const *ksk, uint32_t lwe_dimension_in,
    uint32_t lwe_dimension_out, uint32_t base_log, uint32_t level_count,
    uint32_t num_samples);
void cuda_keyswitch_gemm_64_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lwe_array_in,
    void const *lwe_input_indexes, void const *ksk, uint32_t lwe_dimension_in,
    uint32_t lwe_dimension_out, uint32_t base_log, uint32_t level_count,
    uint32_t num_samples, bool uses_trivial_indexes);
/* Packing keyswitch, keyswitch.h:30-33,49-54,68-70: num_lwes <= N LWEs of
 * input_lwe_dimension + 1 words (device) into ONE GLWE of (k + 1) * N words,
 * GLWE = sum_s X^s * PKS(LWE s) (keyswitch_lwe_ciphertext_list_and_pack_in_
 * glwe_ciphertext, lwe_packing_keyswitch.rs:296-380).  fp_ksk_array: the
 * LwePackingKeyswitchKey [i][level slot][(k + 1) * N], slot 0 = level
 * level_count as in the LWE keyswitch key.  Each LWE is keyswitched by the
 * kernels and exactness rules of cuda_keyswitch_lwe_ciphertext_vector_64_64_
 * async (b200_set_keyswitch_path, b200_last_keyswitch_kernel) into the scratch
 * buffer, then one kernel sums the rows.  The scratch returns its size in
 * bytes, num_lwes * (k + 1) * N * 8, and allocates it stream-ordered only when
 * allocate_gpu_memory (false = size query).  cleanup frees it when
 * gpu_memory_allocated and synchronises the stream. */
uint64_t scratch_cuda_packing_keyswitch_lwe_list_to_glwe_64_async(
    void *stream, uint32_t gpu_index, int8_t **fp_ks_buffer,
    uint32_t lwe_dimension, uint32_t glwe_dimension, uint32_t polynomial_size,
    uint32_t num_lwes, bool allocate_gpu_memory);
void cuda_packing_keyswitch_lwe_list_to_glwe_64_async(
    void *stream, uint32_t gpu_index, void *glwe_array_out,
    void const *lwe_array_in, void const *fp_ksk_array, int8_t *fp_ks_buffer,
    uint32_t input_lwe_dimension, uint32_t output_glwe_dimension,
    uint32_t output_polynomial_size, uint32_t base_log, uint32_t level_count,
    uint32_t num_lwes);
void cleanup_cuda_packing_keyswitch_lwe_list_to_glwe_64(
    void *stream, uint32_t gpu_index, int8_t **fp_ks_buffer,
    bool gpu_memory_allocated);
/* u128 packing keyswitch, keyswitch.h:56-74: the same contract as the _64
 * trio on u128 words (two u64, low then high): num_lwes <= N LWEs of
 * input_lwe_dimension + 1 words into ONE GLWE of (k + 1) * N words; key
 * [i][level slot][(k + 1) * N] with the _64 key's nesting and level order.
 * The digits are SignedDecomposer<u128>'s: 1 <= base_log <= 63,
 * level_count >= 1, base_log * level_count <= 128; anything else aborts.  One
 * kernel keyswitches every LWE into the scratch buffer (integer pipe,
 * csrc/keyswitch128.cuh; b200_last_keyswitch_kernel reports "ks128"), one
 * kernel sums the rows.  The scratch buffer is num_lwes * (k + 1) * N * 16
 * bytes, allocated stream-ordered when allocate_gpu_memory; cleanup frees it
 * when gpu_memory_allocated and synchronises the stream. */
void scratch_cuda_packing_keyswitch_lwe_list_to_glwe_128_async(
    void *stream, uint32_t gpu_index, int8_t **fp_ks_buffer,
    uint32_t lwe_dimension, uint32_t glwe_dimension, uint32_t polynomial_size,
    uint32_t num_lwes, bool allocate_gpu_memory);
void cuda_packing_keyswitch_lwe_list_to_glwe_128_async(
    void *stream, uint32_t gpu_index, void *glwe_array_out,
    void const *lwe_array_in, void const *fp_ksk_array, int8_t *fp_ks_buffer,
    uint32_t input_lwe_dimension, uint32_t output_glwe_dimension,
    uint32_t output_polynomial_size, uint32_t base_log, uint32_t level_count,
    uint32_t num_lwes);
void cleanup_cuda_packing_keyswitch_lwe_list_to_glwe_128(
    void *stream, uint32_t gpu_index, int8_t **fp_ks_buffer,
    bool gpu_memory_allocated);
/* KS32 variants, keyswitch.h:23-28,42-47: u64 input ciphertexts and indexes,
 * u32 keyswitch key (same [i][level slot][n_out+1] nesting), u32 output; body =
 * input body rounded to its top 32 bits (lwe_keyswitch.rs:331-455).
 * base_log * level_count <= 32. */
void cuda_keyswitch_lwe_ciphertext_vector_64_32_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lwe_array_in,
    void const *lwe_input_indexes, void const *ksk, uint32_t lwe_dimension_in,
    uint32_t lwe_dimension_out, uint32_t base_log, uint32_t level_count,
    uint32_t num_samples);
void cuda_keyswitch_gemm_64_32_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lwe_array_in,
    void const *lwe_input_indexes, void const *ksk, uint32_t lwe_dimension_in,
    uint32_t lwe_dimension_out, uint32_t base_log, uint32_t level_count,
    uint32_t num_samples, bool uses_trivial_indexes);

/* ---- stand-alone integer stages: .../include/ciphertext.h:15-32 ---------- */
/* LWE id = sample extraction of coefficient nth_array[id] % num_lwes_stored_per_glwe
 * of GLWE id / num_lwes_to_extract_per_glwe (nth_array on the device). */
void cuda_glwe_sample_extract_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *glwe_array_in, uint32_t const *nth_array, uint32_t num_nths,
    uint32_t num_lwes_to_extract_per_glwe, uint32_t num_lwes_stored_per_glwe,
    uint32_t glwe_dimension, uint32_t polynomial_size);
/* x -> (x + 2^(63 - log_modulus)) >> (64 - log_modulus), element-wise */
void cuda_modulus_switch_inplace_64_async(void *stream, uint32_t gpu_index,
                                          void *lwe_array_out, uint32_t size,
                                          uint32_t log_modulus);
void cuda_modulus_switch_64_async(void *stream, uint32_t gpu_index,
                                  void *lwe_out, const void *lwe_in,
                                  uint32_t size, uint32_t log_modulus);
/* one LWE of lwe_dimension + 1 words: mask switched as above, body after the
 * centered-mean correction (algorithms/modulus_switch.rs:35-100) */
void cuda_centered_modulus_switch_64_async(void *stream, uint32_t gpu_index,
                                           void *lwe_out, const void *lwe_in,
                                           uint32_t lwe_dimension,
                                           uint32_t log_modulus);

/* ---- additions (no reference equivalent) -------------------------------- */
/* forward negacyclic transform of `total_polynomials` real polynomials given
 * as N/2 interleaved (re,im) = (p[j], p[j+N/2]) f64 pairs; output in NATURAL
 * frequency order with the reference's convention
 * X[k] = sum_j z_j e^{i pi j/N} e^{-2 pi i jk/(N/2)} (the contract of the
 * reference's test-only cuda_forward_fft16x4x16_async,
 * include/pbs/programmable_bootstrap.h:26-29).  polynomial_size must be 2048. */
void b200_forward_negacyclic_fft_async(void *stream, uint32_t gpu_index,
                                       void const *input, void *output,
                                       uint32_t polynomial_size,
                                       uint32_t total_polynomials);
/* Seeded (compressed) bootstrap key ingest: `seeded_bodies` = HOST pointer to
 * the body polynomials of a SeededLweBootstrapKey / SeededLweMultiBitBootstrapKey
 * ([ggsw][level][glwe row][N] u64, tfhe/src/core_crypto/entities/
 * seeded_lwe_bootstrap_key.rs); the masks are regenerated ON THE GPU from the
 * compression seed's AES-128 counter-mode table (tfhe-csprng generic.rs:178-193;
 * decompression order of seeded_lwe_bootstrap_key_decompression.rs:36-60) and
 * the key is converted exactly as cuda_convert_lwe_[multi_bit_]programmable_
 * bootstrap_key_64_async would convert the decompressed key.  `aes_key` = the
 * 16 key bytes (Seed(u128) little endian, or the XOF-derived key),
 * counter = first AES index + offset of the generator, first_byte_index in
 * {0, 8}.  grouping_factor 0/1 = classic key.  `dest` sized as for the
 * non-seeded conversion. */
void b200_convert_seeded_lwe_programmable_bootstrap_key_64_async(
    void *stream, uint32_t gpu_index, void *dest, void const *seeded_bodies,
    const uint8_t *aes_key, uint64_t counter_lo, uint64_t counter_hi,
    uint32_t first_byte_index, uint32_t input_lwe_dim, uint32_t glwe_dim,
    uint32_t level_count, uint32_t polynomial_size, uint32_t grouping_factor);
/* Oblivious pseudo-random generation (OPRF), the engine's stand-in for the
 * reference's cuda_integer_grouped_oprf_64_async (tfhe-cuda-backend/cuda/
 * include/integer/integer.h:664-679), whose integer-layer FFI structs
 * (CudaStreamsFFI, CudaRadixCiphertextFFI) this library does not export.
 *
 * Expansion: writes num_blocks LWEs of lwe_dimension + 1 u64 words to
 * `lwe_out`.  Mask word j of block b is
 *   (le(stream[w * (b * lwe_dimension + j) ..]) & (2^log_modulus - 1))
 *     << (64 - log_modulus),      w = ceil(log_modulus / 8) bytes,
 * the body word is 0 (tfhe/src/shortint/oprf.rs: create_random_from_seed_
 * modulus_switched + raw_seeded_msed_to_lwe).  stream[p] is byte
 * first_byte_index + p of the AES-128 counter-mode table of `aes_key` (16 key
 * bytes) starting at AES index counter = counter_hi:counter_lo, the table of
 * b200_convert_seeded_lwe_programmable_bootstrap_key_64_async.  Any
 * first_byte_index; 1 <= log_modulus <= 16 (2N <= 2^16). */
void b200_oprf_expand_seeded_lwe_64_async(
    void *stream, uint32_t gpu_index, void *lwe_out, const uint8_t *aes_key,
    uint64_t counter_lo, uint64_t counter_hi, uint32_t first_byte_index,
    uint32_t lwe_dimension, uint32_t num_blocks, uint32_t log_modulus);
/* Grouped OPRF: expands num_blocks seeded blocks (first_byte_index 0,
 * log_modulus = log2(2 * polynomial_size)) into a stream-ordered workspace,
 * bootstraps block b with LUT lut_indexes[b] of `lut_vector` through the same
 * kernels as cuda_[multi_bit_]programmable_bootstrap_64_async (trivial
 * input/output indexes, num_many_lut = 1), then adds corrections[b] (one u64
 * per block, device) to the body of output b.  `lwe_out` holds num_blocks LWEs
 * of glwe_dimension * polynomial_size + 1 words.  grouping_factor <= 1: classic
 * key, `buffer` from scratch_cuda_programmable_bootstrap_64_async; >= 2:
 * multi-bit key, `buffer` from scratch_cuda_multi_bit_programmable_bootstrap_
 * 64_async.  A CENTERED scratch object is accepted, but this call always runs
 * NO_REDUCTION: the expanded inputs are exact switched values, and the
 * centered-mean correction would move their body off 0. */
void b200_grouped_oprf_64_async(
    void *stream, uint32_t gpu_index, void *lwe_out, const uint8_t *aes_key,
    uint64_t counter_lo, uint64_t counter_hi, void const *lut_vector,
    void const *lut_indexes, void const *corrections,
    void const *bootstrapping_key, int8_t *buffer, uint32_t lwe_dimension,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t base_log,
    uint32_t level_count, uint32_t grouping_factor, uint32_t num_blocks);
/* Compact public-key ciphertext lists (tfhe-rs LweCompactCiphertextList), the
 * input format of tfhe-rs clients.  lwe_flattened_compact_array_in holds
 * num_compact_lists lists back to back (device, u64): list k is lwe_dimension
 * mask words followed by its c_k = num_lwes_per_compact_list[k] bodies, with
 * 1 <= c_k <= lwe_dimension (the reference's flattened_compact_lwe_lists,
 * tfhe-cuda-backend/cuda/include/zk/zk_utilities.h:48-80).
 *
 * NO_CASTING expansion: lwe_array_out = T = sum(c_k) LWEs of lwe_dimension + 1
 * words, list after list.  Expanded LWE i of a list has mask X^i * mask in
 * Z_{2^64}[X]/(X^n + 1) and body i (core_crypto/algorithms/
 * lwe_compact_ciphertext_list_expansion.rs).  num_lwes_per_compact_list is a
 * HOST array of num_compact_lists counts.  lwe_dimension is a power of two in
 * [256, 16384]. */
void b200_expand_lwe_compact_ciphertext_lists_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_flattened_compact_array_in,
    const uint32_t *num_lwes_per_compact_list, uint32_t num_compact_lists,
    uint32_t lwe_dimension);
/* Stand-in for cuda_expand_without_verification_64_async (tfhe-cuda-backend/
 * cuda/include/zk/zk.h), whose CudaStreamsFFI / CudaLweKeyswitchKeyParamsFFI
 * structs this library does not export.  lwe_array_out = 2T LWEs of
 * glwe_dimension * polynomial_size + 1 words, output s = PBS(cast(expanded
 * [s >> 1]), lut_indexes[s]) (device lut_indexes, 2T u64).
 *
 * Casting (shortint KeySwitchingKey::cast_and_apply_functions, cast_rshift 0):
 * casting_to_big = false: one keyswitch with casting_ksk from the compact key
 * (compact_lwe_dimension) to the small key (lwe_dimension); true: casting_ksk
 * to the big key (glwe_dimension * polynomial_size), then computing_ksk to the
 * small key.  Both through cuda_keyswitch_lwe_ciphertext_vector_64_64_async and
 * its kernel choice.  computing_ksk is read only when casting_to_big.
 * grouping_factor <= 1: classic key, `buffer` from scratch_cuda_programmable_
 * bootstrap_64_async, whose noise-reduction type the PBS honours (the cast
 * inputs are ordinary noisy LWEs); >= 2: multi-bit key and scratch.  The
 * scratch is made for >= 2T samples with the same (k, N, l).  Launches, in
 * order: the expansion, the keyswitch(es), one index kernel, the PBS.  The
 * workspaces are stream-ordered pool allocations freed by the call. */
void b200_expand_without_verification_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_flattened_compact_array_in,
    const uint32_t *num_lwes_per_compact_list, uint32_t num_compact_lists,
    uint32_t compact_lwe_dimension, void const *casting_ksk,
    uint32_t casting_base_log, uint32_t casting_level_count, bool casting_to_big,
    void const *computing_ksk, uint32_t computing_base_log,
    uint32_t computing_level_count, void const *lut_vector,
    void const *lut_indexes, void const *bootstrapping_key, int8_t *buffer,
    uint32_t lwe_dimension, uint32_t glwe_dimension, uint32_t polynomial_size,
    uint32_t pbs_base_log, uint32_t pbs_level_count, uint32_t grouping_factor);
/* Compact public-key encryptions of zero from seeds, the randomness of
 * ciphertext re-randomization (tfhe-rs prepare_cpk_zero_for_rerand,
 * shortint/ciphertext/re_randomization.rs:280-320, i.e.
 * encrypt_lwe_compact_ciphertext_list_with_compact_public_key with plaintexts 0
 * and TUniform(noise_bound_log2) for both noises).  compact_public_key: device,
 * 2 * lwe_dimension u64, mask then body.  seeds: HOST, num_seeds x 40 bytes,
 * each the XofSeed data (8-byte domain separator, then the 32-byte seed).
 * entries: HOST, num_entries x 3 u64 {seed index, first stream byte, count c}:
 * entry e encrypts c >= 1 zeros with the generator of its seed started at that
 * byte (0 for one list per seed; accumulated offsets for several lists drawn
 * from one generator, re_randomize_compact_ciphertext_lists).  A list of c
 * zeros draws, in order, ceil(c/n) * n / 8 bytes of r bits, ceil(c/n) * n mask
 * samples and c body samples of ceil((noise_bound_log2 + 2) / 8) bytes each.
 * lwe_flattened_compact_array_out (device): the entries back to back, each in
 * the flattened bin layout of b200_expand_lwe_compact_ciphertext_lists_64_async
 * (per bin of at most n: the mask, then its bodies), ceil(c/n) * n + c words per
 * entry.  accumulate: add the zeros into the words already there instead of
 * storing them.  lwe_dimension is a power of two in [256, 16384];
 * noise_bound_log2 in [0, 62].  Launches: the seed initialisation, the
 * generation.  The XOF initialisation and key schedules run on the device;
 * the workspace is a stream-ordered pool allocation freed by the call. */
void b200_cpk_encrypt_zeros_from_seeds_64_async(
    void *stream, uint32_t gpu_index, void *lwe_flattened_compact_array_out,
    void const *compact_public_key, const uint8_t *seeds, uint32_t num_seeds,
    const uint64_t *entries, uint32_t num_entries, uint32_t lwe_dimension,
    uint32_t noise_bound_log2, bool accumulate);
/* Stand-in for cuda_rerand_64_async (tfhe-cuda-backend/cuda/src/integer/
 * rerand.cuh), whose CudaStreamsFFI / CudaLweKeyswitchKeyParamsFFI structs this
 * library does not export.  lwe_array (device, in place): T = sum(counts) LWEs
 * of lwe_dimension + 1 words; LWE t += zero t.  The zeros are the compact lists
 * lwe_flattened_compact_array_in (device, flattened bins, host counts as in
 * b200_expand_lwe_compact_ciphertext_lists_64_async) expanded at
 * compact_lwe_dimension, then, when ksk is not null, keyswitched with it
 * (ksk_base_log, ksk_level_count) from compact_lwe_dimension to lwe_dimension
 * through cuda_keyswitch_lwe_ciphertext_vector_64_64_async.  A null ksk is the
 * derived compact key (no keyswitch): lwe_dimension must equal
 * compact_lwe_dimension.  Launches: the expansion, the keyswitch (if any), one
 * add kernel; the workspace is a stream-ordered pool allocation freed by the
 * call. */
void b200_rerand_64_async(void *stream, uint32_t gpu_index, void *lwe_array,
                          void const *lwe_flattened_compact_array_in,
                          const uint32_t *num_lwes_per_compact_list,
                          uint32_t num_compact_lists,
                          uint32_t compact_lwe_dimension, void const *ksk,
                          uint32_t ksk_base_log, uint32_t ksk_level_count,
                          uint32_t lwe_dimension);
/* Ciphertext-list compression, the engine's stand-in for
 * cuda_integer_compress_radix_ciphertext_64_async (tfhe-cuda-backend/cuda/
 * include/integer/compression/compression.h), whose CudaStreamsFFI /
 * CudaPackedGlweCiphertextListFFI structs this library does not export
 * (shortint CompressionKey::compress_ciphertexts_into_list,
 * list_compression/compression.rs).  lwe_array_in: num_lwes LWEs of
 * lwe_dimension + 1 words (device), each multiplied by `scale`
 * (message_modulus) into a workspace, packing-keyswitched with packing_ksk
 * (as in cuda_packing_keyswitch_lwe_list_to_glwe_64_async) and packed
 * lwe_per_glwe per GLWE: GLWE g holds LWEs g * lwe_per_glwe + s, s < c_g.
 * Its first k * N + c_g coefficients are switched to storage_log_modulus bits
 * and bit-packed least-significant bit first (PackedIntegers::pack,
 * core_crypto/entities/packed_integers.rs).  packed_out (device): GLWE g at
 * word g * W, W = (k + 1) * N * storage_log_modulus / 64; its first
 * ceil((k * N + c_g) * storage_log_modulus / 64) words are tfhe-rs'
 * packed_coeffs, the rest are zero.  1 <= lwe_per_glwe <= N,
 * 1 <= storage_log_modulus <= 64.  Launches, in order: the scale, the
 * keyswitch (digits + int8 GEMM, or one fp64/integer kernel), the
 * accumulate/switch/pack kernel; the workspaces are stream-ordered pool
 * allocations freed by the call. */
void b200_compress_lwe_ciphertexts_64_async(
    void *stream, uint32_t gpu_index, void *packed_out, void const *lwe_array_in,
    uint32_t num_lwes, uint32_t lwe_dimension, uint64_t scale,
    void const *packing_ksk, uint32_t glwe_dimension, uint32_t polynomial_size,
    uint32_t base_log, uint32_t level_count, uint32_t lwe_per_glwe,
    uint32_t storage_log_modulus);
/* Decompression, the stand-in for cuda_integer_decompress_radix_ciphertext_
 * 64_async (DecompressionKey::unpack, list_compression/compression.rs):
 * lwe_out (device) = num_indexes LWEs of glwe_dimension * polynomial_size + 1
 * words, output r = PBS(extract(indexes[r])) with the single LUT lut_vector.
 * extract(i) is the sample extraction of coefficient i % lwe_per_glwe of
 * packed GLWE i / lwe_per_glwe of packed_in (the layout of
 * b200_compress_lwe_ciphertexts_64_async, compression_glwe_dimension and
 * compression_polynomial_size), every field read as field << (64 -
 * storage_log_modulus): an LWE of compression_glwe_dimension *
 * compression_polynomial_size, the input dimension of bootstrapping_key.
 * indexes: HOST, each < num_lwes_in_list, repeats allowed.  grouping_factor
 * <= 1: classic key and scratch_cuda_programmable_bootstrap_64_async buffer;
 * >= 2: multi-bit key and scratch; made for >= num_indexes samples with the
 * same (k, N, l).  Always NO_REDUCTION: the extracted words are exact
 * multiples of 2^(64 - storage_log_modulus) and the centered-mean correction
 * would move them.  Launches: one unpack/extract kernel, then the PBS route's
 * own (trivial indexes, num_many_lut 1); the workspace is a stream-ordered pool
 * allocation freed by the call. */
void b200_decompress_lwe_ciphertexts_64_async(
    void *stream, uint32_t gpu_index, void *lwe_out, void const *packed_in,
    uint32_t num_lwes_in_list, const uint32_t *indexes, uint32_t num_indexes,
    uint32_t compression_glwe_dimension, uint32_t compression_polynomial_size,
    uint32_t lwe_per_glwe, uint32_t storage_log_modulus, void const *lut_vector,
    void const *bootstrapping_key, int8_t *buffer, uint32_t glwe_dimension,
    uint32_t polynomial_size, uint32_t base_log, uint32_t level_count,
    uint32_t grouping_factor);
/* Stand-in for cuda_apply_noise_squashing_async (tfhe-cuda-backend/cuda/
 * include/integer/integer.h), whose FFI structs this library does not export:
 * shortint NoiseSquashingKey::squash_radix_ciphertext_noise.  lwe_array_in:
 * num_blocks u64 LWEs of input_lwe_dimension + 1 words (big key).  Pairs are
 * packed as in[2i] + message_modulus * in[2i + 1] (an odd last block alone),
 * keyswitched with ksk to lwe_dimension through cuda_keyswitch_lwe_ciphertext_
 * vector_64_64_async's kernel choice, then bootstrapped by cuda_programmable_
 * bootstrap_128_async with lut_vector (one u128 GLWE) and the 128-bit Fourier
 * key; `buffer` is a scratch_cuda_programmable_bootstrap_128_async object made
 * for >= ceil(num_blocks / 2) samples.  lwe_array_out: ceil(num_blocks / 2)
 * u128 LWEs of glwe_dimension * polynomial_size + 1 words.  Launches, in
 * order: the packing, the keyswitch, the PBS.  The workspace is a
 * stream-ordered pool allocation freed by the call; nothing synchronises. */
void b200_apply_noise_squashing_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_array_in, uint32_t num_blocks, uint32_t input_lwe_dimension,
    uint32_t message_modulus, void const *ksk, uint32_t ks_base_log,
    uint32_t ks_level_count, void const *lut_vector,
    void const *bootstrapping_key, int8_t *buffer, uint32_t lwe_dimension,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t pbs_base_log,
    uint32_t pbs_level_count);
/* b200_apply_noise_squashing_64_async with a multi-bit squashing key: the
 * same packing and keyswitch, then cuda_multi_bit_programmable_bootstrap_
 * 128_async's kernel with grouping_factor and trivial indexes; `buffer` is a
 * scratch_cuda_multi_bit_programmable_bootstrap_128_async object made for
 * >= ceil(num_blocks / 2) samples.  Launches, in order: the packing, the
 * keyswitch, the PBS. */
void b200_apply_noise_squashing_multi_bit_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_array_in, uint32_t num_blocks, uint32_t input_lwe_dimension,
    uint32_t message_modulus, void const *ksk, uint32_t ks_base_log,
    uint32_t ks_level_count, void const *lut_vector,
    void const *bootstrapping_key, int8_t *buffer, uint32_t lwe_dimension,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t grouping_factor,
    uint32_t pbs_base_log, uint32_t pbs_level_count);
/* Noise-squashing compression, the stand-in for cuda_integer_compress_radix_
 * ciphertext_128_async (NoiseSquashingCompressionKey::compress_noise_squashed_
 * ciphertexts_into_list, list_compression/noise_squashing_compression.rs).
 * lwe_array_in: num_lwes squashed u128 LWEs of lwe_dimension + 1 words
 * (device), packing-keyswitched with packing_ksk as in
 * cuda_packing_keyswitch_lwe_list_to_glwe_128_async, as they are (no scaling,
 * no modulus switch: the storage modulus is 2^128), lwe_per_glwe per GLWE:
 * GLWE g holds LWEs g * lwe_per_glwe + s, s < c_g.  packed_out (device):
 * GLWE g at u128 word g * (k + 1) * N; its first k * N + c_g words are
 * tfhe-rs' packed_coeffs, the rest are zero.  1 <= lwe_per_glwe <= N and the
 * decomposition limits of the _128 packing keyswitch; anything else aborts.
 * Launches: the keyswitch, the pack.  The workspace (num_lwes * (k + 1) * N *
 * 16 bytes) is a stream-ordered pool allocation freed by the call. */
void b200_compress_lwe_ciphertexts_128_async(
    void *stream, uint32_t gpu_index, void *packed_out, void const *lwe_array_in,
    uint32_t num_lwes, uint32_t lwe_dimension, void const *packing_ksk,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t base_log,
    uint32_t level_count, uint32_t lwe_per_glwe);
/* Noise-squashing decompression, the stand-in for cuda_integer_decompress_
 * radix_ciphertext_128_async (CompressedSquashedNoiseCiphertextList::unpack):
 * no PBS.  lwe_out (device) = num_indexes u128 LWEs of glwe_dimension *
 * polynomial_size + 1 words; output r is the sample extraction of coefficient
 * indexes[r] % lwe_per_glwe of GLWE indexes[r] / lwe_per_glwe of packed_in
 * (the layout of b200_compress_lwe_ciphertexts_128_async).  indexes: HOST,
 * each < num_lwes_in_list (else abort), repeats allowed.  One launch; the
 * index copy is a stream-ordered pool allocation freed by the call. */
void b200_decompress_lwe_ciphertexts_128_async(
    void *stream, uint32_t gpu_index, void *lwe_out, void const *packed_in,
    uint32_t num_lwes_in_list, const uint32_t *indexes, uint32_t num_indexes,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t lwe_per_glwe);
/* The linear step of a compiled bit circuit (tfhe-rs_b200/bit_circuit.py;
 * no reference counterpart: tfhe-rs flushes every XOR-sum of its AES with its
 * own PBS).  All arrays on the DEVICE.  pool: LWEs of lwe_dimension + 1 words;
 * slot s < num_shared_slots is pool row s, slot s >= num_shared_slots of
 * instance i is pool row num_shared_slots + (s - num_shared_slots) *
 * num_instances + i.  Logical row r < num_rows reads the terms
 * [row_offsets[r], row_offsets[r + 1]) of term_slots (u32) / term_coefs (i64,
 * signed) -- offsets index those arrays directly -- and its body constant
 * body_constants[r * num_instances + i] (u64, added to the body word).  Rows
 * r < num_shared_rows are computed once, for instance 0; every other row once
 * per instance.  lwe_array_out: num_shared_rows + (num_rows - num_shared_rows)
 * * num_instances LWEs, shared rows first, then row-major, instance-minor:
 * out = sum coef * pool[row] + body, wrapping mod 2^64.  One launch (one CTA
 * per output LWE); must not alias the pool. */
void b200_lwe_linear_combination_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out, void const *pool,
    uint32_t lwe_dimension, uint32_t num_shared_slots, uint32_t num_instances,
    uint32_t num_rows, uint32_t num_shared_rows, void const *row_offsets,
    void const *term_slots, void const *term_coefs, void const *body_constants);
/* A whole compiled bit circuit in one call: for every layer L <
 * num_layers (HOST arrays layer_rows[num_layers + 1], layer_shared_rows
 * [num_layers]: logical rows layer_rows[L] .. layer_rows[L + 1], the first
 * layer_shared_rows[L] of them shared), in order:
 *   1. b200_lwe_linear_combination_64_async's kernel on those rows (tables as
 *      there, body_constants indexed by the global row) into a staging buffer
 *      of big_lwe_dimension + 1 word LWEs;
 *   2. the keyswitch of cuda_keyswitch_lwe_ciphertext_vector_64_64_async,
 *      with its own kernel choice (ksk, ks_base_log, ks_level_count), to
 *      lwe_dimension;
 *   3. the PBS of cuda_programmable_bootstrap_64_async (grouping_factor <= 1:
 *      classic key and scratch, the scratch's noise-reduction type) or of
 *      cuda_multi_bit_programmable_bootstrap_64_async (>= 2: multi-bit key and
 *      scratch), num_many_lut 1, with the DEVICE per-output arrays lut_indexes
 *      (into lut_vector) and output_indexes (pool rows: the PBS writes into
 *      the pool), both consumed layer after layer (output rows of layer L
 *      start after those of the layers before it), and input_indexes = 0, 1,
 *      ... of the widest layer.
 * The scratch must be made for the (k, N, l) and at least the widest layer's
 * output rows; big_lwe_dimension must be glwe_dimension * polynomial_size.
 * Launches per non-empty layer: one linear kernel, then the keyswitch's and
 * the PBS route's own.  The staging buffers (widest layer, big and small LWEs)
 * are one stream-ordered pool allocation freed by the call; nothing
 * synchronises. */
void b200_bit_circuit_64_async(
    void *stream, uint32_t gpu_index, void *pool, uint32_t num_shared_slots,
    uint32_t num_instances, uint32_t num_layers, const uint32_t *layer_rows,
    const uint32_t *layer_shared_rows, void const *row_offsets,
    void const *term_slots, void const *term_coefs, void const *body_constants,
    void const *lut_indexes, void const *output_indexes,
    void const *input_indexes, void const *ksk, uint32_t ks_base_log,
    uint32_t ks_level_count, void const *lut_vector,
    void const *bootstrapping_key, int8_t *buffer, uint32_t big_lwe_dimension,
    uint32_t lwe_dimension, uint32_t glwe_dimension, uint32_t polynomial_size,
    uint32_t pbs_base_log, uint32_t pbs_level_count, uint32_t grouping_factor);
/* pin the keyswitch kernel: 0 automatic (default), 1 int8 tensor cores
 * (keyswitch_imma.cuh), 2 fp64 pipe, 3 integer pipe (keyswitch.cuh).  A path
 * whose exactness precondition does not hold for the given decomposition
 * falls through to the next one (1 -> 2 -> 3); base_log >= 32 always runs the
 * integer pipe's s64-digit instance.  b200_last_keyswitch_kernel names the
 * kernel that ran.  Also settable with B200_KS_PATH. */
void b200_set_keyswitch_path(int path);
/* pin the classic-PBS kernel of the (N = 2048, k = 1, l = 1) fast path for A/B
 * measurements and bit-identity tests: 0 automatic (default), 1 first kernel
 * (u64 accumulator), 3 round-1 register kernel, 5 lean rotate/decompose with
 * exchange 2 through shared memory, 4 / 6 other key-prefetch schedules, 7 TMA
 * key ring (one CTA per SM), 8 exchange 2 through warp shuffles (x2_shfl.cuh),
 * 9 shuffle exchange + one-slot TMA key ring at two CTAs per SM (v6),
 * 14 the same with the switched mask staged in shared memory (one CTA per SM),
 * 15..19 v6 with other rotate/decompose instruction sequences, 20..22 v6
 * with the CTA barriers around the MAC replaced by arrive / wait pairs (19 and 20
 * are what the automatic dispatch launches for <= / > one CTA per SM),
 * 10 v6 with the register key prefetch, 11 v6 with the own key row in
 * registers and the other row through the ring.
 * All variants compute the same function; 3..8 are bit-identical to each
 * other.  Any other value aborts.  Also settable with B200_PBS_VARIANT. */
void b200_set_pbs_variant(int variant);
/* (N = 512, l = 1, k <= 4) register kernel (csrc/pbs_n512.cuh), e.g.
 * PARAM_MESSAGE_1_CARRY_1: 0 automatic (TMA key ring, one CTA per SM, 1 / 2 / 3
 * LWEs per CTA by launch size), 3 / 2 / 4 ring with one / two / three LWEs per
 * CTA, 1 register key ring with two CTAs per SM.  Modes 0, 2, 3 and 4 give
 * bit-identical results; mode 1 computes the same function, with output words
 * that differ from theirs (another f64 evaluation order; both within the same
 * bound of the exact blind rotation, tests/test_pbs_routes.py).
 * Also B200_N512_MODE; B200_N512_GENERIC=1 keeps these shapes on the generic
 * kernel (read at library load: it also selects the key layout). */
void b200_set_n512_mode(int mode);
/* Which shapes run on their dedicated register kernels: bit 0 (N = 512, l = 1,
 * k <= 4; csrc/pbs_n512.cuh), bit 1 (N = 8192, k = 1, l = 2; csrc/pbs_n8192.cuh,
 * PARAM_MESSAGE_3_CARRY_3).  Default 3; a cleared bit keeps the shape on the
 * generic kernels (A/B measurements).  Bit 2 (value 4) selects the
 * first-generation N = 8192 kernel (per-thread key loads instead of the TMA
 * ring; same key layout, same results; B200_N8192_GEN1=1).  Bit 3 (value 8)
 * selects a debug instance of the default kernel for compute-sanitizer
 * racecheck (every thread arrives on the ring's `empty` barriers itself;
 * B200_N8192_RACECHECK=1).  The setting selects the device key
 * layout: convert a key and run its PBS under the same value.  Environment:
 * B200_N512_GENERIC=1 / B200_N8192_GENERIC=1 clear bit 0 / bit 1 at load. */
void b200_set_register_kernels(int mask);
/* DEVIATION FROM THE REFERENCE, switchable.  The multi-bit PBS kernels round
 * an exact tie of the bits dropped by the gadget decomposition to EVEN; the
 * reference (commons/math/decomposition/decomposer.rs:163-188) rounds it up.
 * Their accumulator is re-assigned from f64 every step (and is a 32-bit word
 * in the N = 2048 register kernels), so exact ties are common and always-up
 * biases every coefficient: measured output-noise variance 7.6x (g = 3) /
 * 1.10x (g = 4) of the reference formula with the reference rule against
 * 0.21x / 0.40x with the even rule.  Outputs are valid
 * ciphertexts of the same plaintext either way.  reference_exact != 0 selects
 * the reference's rule bit for bit (also B200_MULTIBIT_TIES=reference).  The
 * same switch governs the classic (N = 8192, k = 1, l = 2) register kernel
 * (csrc/pbs_n8192.cuh): its 32-bit accumulator leaves two bits below the
 * gadget's 30, a tie is hit by one value in four, and always-up measured 10x
 * the oracle's output noise on PARAM_MESSAGE_3_CARRY_3.  Every other classic PBS kernel and the keyswitch always use the
 * reference rule (their ties have probability <= 2^-9). */
void b200_set_multibit_tie_rule(int reference_exact);
/* multi-bit PBS (N = 2048, k = 1): launches of at most `max_samples` LWEs take
 * the low-latency path -- the per-sample key bundle of all n/g groups is built
 * by one GPU-wide kernel into a stream-ordered workspace, then one CTA per LWE
 * runs the n/g external products (the reference's keybundle + accumulate
 * split, programmable_bootstrap_multibit.cuh:30-430); larger launches use the
 * fused kernel that never materialises the bundle.  -1 = default (the SM
 * count), 0 = never.  Also settable with B200_MULTIBIT_LL_MAX. */
void b200_set_multibit_ll_max(int max_samples);
/* number of kernels this library has launched in the calling process */
uint64_t b200_kernel_launch_count(void);
/* name of the kernel instance the calling thread's last PBS launch ran (classic,
 * multi-bit, u32 torus and the PBS of the grouped OPRF), e.g.
 * "n2048_v6<2,true,2,1>", "n512<4,3,true>", "n8192_v2<false>",
 * "multibit_fused<3,2>", "multibit_ll<4,1,tma>", "generic_workspace",
 * "pbs128<2048>" (the 128-bit PBS, by polynomial size), "pbs128_mb<2048>"
 * (the multi-bit 128-bit PBS); "" before
 * the first one.  A static string: valid for the life of the library. */
const char *b200_last_pbs_kernel(void);
/* name of the kernel the calling thread's last keyswitch launch ran:
 * "ks_imma<1>", "ks_imma<2>" (int8 tensor cores), "ks_f64" (fp64 pipe),
 * "ks_int" (integer pipe, s32 digits), "ks_int_wide" (integer pipe, s64 digits:
 * base_log >= 32), "ks_64_32" or "ks128" (the u128 packing keyswitch); ""
 * before the first one.  A static string:
 * valid for the life of the library. */
const char *b200_last_keyswitch_kernel(void);
/* 1 if (lwe_dim, glwe_dim, N, level_count) runs on the register-FFT kernel */
int b200_pbs_uses_fast_path(uint32_t lwe_dimension, uint32_t glwe_dimension,
                            uint32_t polynomial_size, uint32_t level_count);
const char *b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* TFHE_B200_H */
