// b200_backend.cu -- the single translation unit of
// libtfhe_cuda_backend_b200.so: device helpers, per-device tables and the
// extern "C" entry points declared in include/tfhe_b200.h (same names and
// signatures as tfhe-rs' backends/tfhe-cuda-backend C ABI).
//
// There is NO CPU fallback anywhere in this file: every entry point launches
// sm_90a kernels or aborts.
#include "../../include/tfhe_b200.h"

#include <algorithm>
#include <atomic>
#include <cstring>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "keyswitch.cuh"
#include "keyswitch_imma.cuh"
#include "pbs_generic.cuh"
#include "pbs_n2048.cuh"
#include "pbs_n512.cuh"
#include "pbs_n8192.cuh"
#include "pbs_multibit_n2048.cuh"
#include "seeded_key.cuh"
#include "oprf.cuh"
#include "compact_expand.cuh"
#include "ciphertext_ops.cuh"

namespace b200 {

static std::atomic<uint64_t> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

// name of the kernel instance the calling thread's last PBS launch ran
// (b200_last_pbs_kernel): one pointer store per launch, next to count_launch
static thread_local const char *t_last_pbs_kernel = "";

void set_device(uint32_t gpu_index) {
  // every static per-GPU table in this file is indexed by gpu_index
  B200_PANIC_IF_FALSE(gpu_index < MAX_GPUS, "gpu_index %u out of range (max %d)",
                      gpu_index, MAX_GPUS);
  B200_CHECK(cudaSetDevice((int)gpu_index));
}

static std::mutex g_tables_mutex;
static DeviceTables g_tables[MAX_GPUS];

const DeviceTables &device_tables(uint32_t gpu_index, uint32_t logM) {
  B200_PANIC_IF_FALSE(gpu_index < MAX_GPUS, "gpu_index %u out of range",
                      gpu_index);
  B200_PANIC_IF_FALSE(logM <= MAX_LOGM, "unsupported transform size 2^%u",
                      logM);
  std::lock_guard<std::mutex> lock(g_tables_mutex);
  DeviceTables &t = g_tables[gpu_index];
  set_device(gpu_index);
  if (!t.fft1024) {
    Fft1024Tables *host = new Fft1024Tables;
    b200_fill_fft1024_tables(host);
    B200_CHECK(cudaMalloc(&t.fft1024, sizeof(Fft1024Tables)));
    B200_CHECK(cudaMemcpy(t.fft1024, host, sizeof(Fft1024Tables),
                          cudaMemcpyHostToDevice));
    B200_CHECK(cudaMemcpyToSymbol(c_fft1024_pass1, host->pass1,
                                  sizeof(host->pass1)));
    {
      const char *e = std::getenv("B200_P22_STAGGER");
      const uint32_t stagger = e ? (uint32_t)std::atoi(e) : 0u;
      B200_CHECK(cudaMemcpyToSymbol(c_p22_stagger, &stagger, sizeof(stagger)));
    }
    delete host;
    Fft256Tables *h256 = new Fft256Tables;
    b200_fill_fft256_tables(h256);
    B200_CHECK(cudaMalloc(&t.fft256, sizeof(Fft256Tables)));
    B200_CHECK(cudaMemcpy(t.fft256, h256, sizeof(Fft256Tables),
                          cudaMemcpyHostToDevice));
    B200_CHECK(cudaMemcpyToSymbol(c_fft256_pass1, h256->pass1,
                                  sizeof(h256->pass1)));
    delete h256;
    Fft4096Tables *h4096 = new Fft4096Tables;
    b200_fill_fft4096_tables(h4096);
    B200_CHECK(cudaMalloc(&t.fft4096, sizeof(Fft4096Tables)));
    B200_CHECK(cudaMemcpy(t.fft4096, h4096, sizeof(Fft4096Tables),
                          cudaMemcpyHostToDevice));
    B200_CHECK(cudaMemcpyToSymbol(c_fft4096_pass1, h4096->pass1,
                                  sizeof(h4096->pass1)));
    delete h4096;
  }
  if (logM && !t.gen_tw[logM]) {
    const size_t M = (size_t)1 << logM;
    std::vector<cplx> tw(M), root(4 * M);
    b200_fill_generic_tables(logM, tw.data(), root.data());
    B200_CHECK(cudaMalloc(&t.gen_tw[logM], M * sizeof(cplx)));
    B200_CHECK(cudaMalloc(&t.gen_root[logM], 4 * M * sizeof(cplx)));
    B200_CHECK(cudaMemcpy(t.gen_tw[logM], tw.data(), M * sizeof(cplx),
                          cudaMemcpyHostToDevice));
    B200_CHECK(cudaMemcpy(t.gen_root[logM], root.data(), 4 * M * sizeof(cplx),
                          cudaMemcpyHostToDevice));
    if (logM == 10) {
      std::vector<cplx> mono((size_t)4096 * 64);
      for (uint32_t deg = 0; deg < 4096; deg++)
        for (uint32_t tt = 0; tt < 64; tt++)
          mono[(size_t)deg * 64 + tt] =
              root[(deg * (1u + 4u * b200_bitrev(tt, 6))) & 4095u];
      B200_CHECK(cudaMalloc(&t.mono2048, mono.size() * sizeof(cplx)));
      B200_CHECK(cudaMemcpy(t.mono2048, mono.data(), mono.size() * sizeof(cplx),
                            cudaMemcpyHostToDevice));
    }
  }
  return t;
}

static uint32_t ilog2_exact(uint32_t x) {
  uint32_t l = 0;
  while ((1u << l) < x)
    l++;
  B200_PANIC_IF_FALSE((1u << l) == x, "%u is not a power of two", x);
  return l;
}

// The same predicate picks the Fourier-BSK layout at key conversion and the
// kernel at PBS time (cf. the reference's supports_specialized_2_2_params,
// programmable_bootstrap_classic.cuh:198-212).
static bool uses_fast_path(uint32_t n, uint32_t k, uint32_t N, uint32_t l) {
  return N == 2048 && k == 1 && l == 1 && n <= 1024;
}

// (N = 512, l = 1, k <= 4, n <= 1024): register kernel of pbs_n512.cuh, e.g.
// PARAM_MESSAGE_1_CARRY_1_KS_PBS.  Same predicate at key conversion and at PBS
// time; B200_N512_GENERIC=1 keeps these shapes on the generic kernel (A/B).
// b200_set_register_kernels(mask) switches them at run time (bit 0: N = 512,
// bit 1: N = 8192); a key must be converted and used under the same setting.
static std::atomic<int> &register_kernel_mask() {
  static std::atomic<int> v((std::getenv("B200_N512_GENERIC") ? 0 : 1) | (std::getenv("B200_N8192_GENERIC") ? 0 : 2) |
                            (std::getenv("B200_N8192_GEN1") ? 4 : 0) | (std::getenv("B200_N8192_RACECHECK") ? 8 : 0));
  return v;
}
static bool uses_n512_path(uint32_t n, uint32_t k, uint32_t N, uint32_t l) {
  return (register_kernel_mask().load() & 1) && N == 512 && l == 1 && k >= 1 && k <= 4 && n <= 1024;
}

// (N = 8192, k = 1, l = 2, n <= 2048): register kernel of pbs_n8192.cuh
// (PARAM_MESSAGE_3_CARRY_3_KS_PBS).  B200_N8192_GENERIC=1 keeps the shape on the
// global-workspace kernel (A/B; read at library load: it selects the key layout).
static bool uses_n8192_path(uint32_t n, uint32_t k, uint32_t N, uint32_t l) {
  return (register_kernel_mask().load() & 2) && N == 8192 && k == 1 && l == 2 && n <= 2048;
}

// B200_PBS_VARIANT pins a kernel for A/B measurements: 1 first-generation
// kernel (u64 accumulator), 3 the round-1 register kernel, 5 round-1 MAC
// schedule + lean rotate/decompose (the default), 4 all key values in flight
// across the share barrier + lean rotate/decompose.  Read once per process.
// kernel generations b200_set_pbs_variant / B200_PBS_VARIANT can pin (see launch_pbs)
static bool is_pbs_variant(int v) {
  return v == 0 || v == 1 || (v >= 3 && v <= 11) || (v >= 14 && v <= 22);
}
static std::atomic<int> &fast_variant_sel() {
  static std::atomic<int> v([] {
    const char *e = std::getenv("B200_PBS_VARIANT");
    const int x = e ? std::atoi(e) : 0;
    B200_PANIC_IF_FALSE(is_pbs_variant(x), "B200_PBS_VARIANT=%d names no kernel", x);
    return x;
  }());
  return v;
}
static int fast_variant() { return fast_variant_sel().load(); }
static std::atomic<int> &n512_mode_sel() {
  static std::atomic<int> v([] {
    const char *e = std::getenv("B200_N512_MODE");
    return e ? std::atoi(e) : 0;
  }());
  return v;
}

// multi-bit twin of uses_fast_path (layout + kernel predicate)
static bool uses_multibit_fast_path(uint32_t k, uint32_t N, uint32_t l,
                                    uint32_t grouping) {
  static const bool disabled = std::getenv("B200_MULTIBIT_GENERIC") != nullptr;
  return !disabled && N == 2048 && k == 1 && l >= 1 && l <= 2 &&
         grouping >= 2 && grouping <= 4;
}

static void check_polynomial_size(uint32_t N) {
  B200_PANIC_IF_FALSE(
      N >= 256 && N <= 16384 && (N & (N - 1)) == 0,
      "Cuda error (classical PBS): unsupported polynomial size. Supported N's "
      "are powers of two in the interval [256..16384]. Got %u", N);
}

// ABI twin of the reference's `pbs_buffer_base` (include/pbs/pbs_utilities.h:
// 93-96): one pure virtual `release(stream, gpu_index)` and a virtual
// destructor, nothing else.  The reference's integer layer keeps every scratch
// object as a `pbs_buffer_base *` and ends its life with
//   buffer->release(stream, gpu_index); delete buffer;
// (include/integer/integer_utilities.h:1212-1216).  Deriving the scratch object
// from an identically declared base gives it the same Itanium-ABI layout (vptr
// at offset 0; vtable = {release, complete dtor, deleting dtor}), so those two
// calls land in this library when it sits under the reference's integer .cu
// files -- tests/test_gpu_parity.py::test_scratch_object_is_vtable_compatible
// makes them the way compiled C++ does, through the vtable.
struct pbs_buffer_base_abi {
  virtual void release(cudaStream_t stream, uint32_t gpu_index) = 0;
  virtual ~pbs_buffer_base_abi() = default;
};

constexpr uint32_t SCRATCH_MAGIC = 0xB2005C7Au;
// scratch object handed back through int8_t **buffer (opaque to the Rust side)
struct PbsScratch : public pbs_buffer_base_abi {
  uint32_t magic;
  PBS_TYPE type;
  uint32_t glwe_dim, poly_size, level_count, max_samples;
  int centered_ms;
  bool gpu_memory_allocated;
  // the persistent kernels keep their intermediates on chip or in per-call
  // stream-ordered pool allocations (N = 8192 park area, keyswitch digits,
  // multi-bit bundles) that each launch frees itself: nothing to free here
  void release(cudaStream_t stream, uint32_t gpu_index) override {
    (void)stream;
    (void)gpu_index;
    B200_PANIC_IF_FALSE(magic == SCRATCH_MAGIC,
                        "Cuda error (PBS): invalid scratch buffer");
  }
  ~PbsScratch() override { magic = 0; }
};

// stream-ordered workspace pool shared by the entry points that need scratch
// memory per call (keyswitch digit matrix, multi-bit bundles): freed blocks stay
// in the pool across synchronisations (release threshold = max), so steady-state
// calls never reach the driver allocator.
static cudaMemPool_t workspace_pool(uint32_t gpu_index) {
  static std::once_flag once[MAX_GPUS];
  static cudaMemPool_t pool[MAX_GPUS];
  std::call_once(once[gpu_index], [gpu_index] {
    cudaMemPoolProps props = {};
    props.allocType = cudaMemAllocationTypePinned;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = (int)gpu_index;
    B200_CHECK(cudaMemPoolCreate(&pool[gpu_index], &props));
    uint64_t keep = UINT64_MAX;
    B200_CHECK(cudaMemPoolSetAttribute(pool[gpu_index],
                                       cudaMemPoolAttrReleaseThreshold, &keep));
  });
  return pool[gpu_index];
}

// largest launch served by the low-latency multi-bit path; default = one CTA per
// SM (above that the fused kernel's 2 CTAs / SM win).  B200_MULTIBIT_LL_MAX
// overrides (0 disables the path; tests pin either path with it).
// multi-bit decomposition tie rule: 1 = ties of the dropped bits round to even
// (default; see digits_u32), 0 = the reference's round-half-up, bit for bit
static std::atomic<int> &multibit_ties_even() {
  static std::atomic<int> v([] {
    const char *e = std::getenv("B200_MULTIBIT_TIES");
    return (e && std::string(e) == "reference") ? 0 : 1;
  }());
  return v;
}
static std::atomic<int> &multibit_ll_override() {
  static std::atomic<int> v([] {
    const char *e = std::getenv("B200_MULTIBIT_LL_MAX");
    return e ? std::atoi(e) : -1;
  }());
  return v;
}
static uint32_t sm_count(uint32_t gpu_index) {
  static std::atomic<int> sms[MAX_GPUS] = {};
  int v = sms[gpu_index].load();
  if (!v) {
    B200_CHECK(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount,
                                      (int)gpu_index));
    sms[gpu_index].store(v);
  }
  return (uint32_t)v;
}
static uint32_t multibit_ll_max_samples(uint32_t gpu_index) {
  const int env = multibit_ll_override().load();
  if (env >= 0)
    return (uint32_t)env;
  return sm_count(gpu_index);
}

static void launch_multibit_ll(cudaStream_t stream, uint32_t gpu_index,
                               uint64_t *lwe_out, const uint64_t *out_idx,
                               const uint64_t *luts, const uint64_t *lut_idx,
                               const uint64_t *lwe_in, const uint64_t *in_idx,
                               const cplx *bsk, const DeviceTables &t,
                               uint32_t n, uint32_t base_log, uint32_t l,
                               uint32_t grouping, uint32_t num_samples,
                               uint32_t num_many_lut, uint32_t lut_stride) {
  const uint32_t steps = n / grouping;
  const size_t bytes =
      (size_t)num_samples * steps * l * 4 * P22_M * sizeof(cplx);
  cplx *bundle = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(&bundle, bytes, workspace_pool(gpu_index),
                                     stream));
  static std::once_flag once[MAX_GPUS];
  std::call_once(once[gpu_index], [] {
    B200_CHECK(cudaFuncSetAttribute(
        pbs_multibit_seq_kernel<1, false>,
        cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MbSeqSmem)));
    B200_CHECK(cudaFuncSetAttribute(
        pbs_multibit_seq_kernel<2, false>,
        cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MbSeqSmem)));
    B200_CHECK(cudaFuncSetAttribute(
        pbs_multibit_seq_kernel<1, true>,
        cudaFuncAttributeMaxDynamicSharedMemorySize,
        (int)sizeof(MbSeqSmemTma)));
  });
  auto for_each_instance = [&](auto &&fn) {
    fn(mb_bundle_kernel<2, 1>, 2u, 1u);
    fn(mb_bundle_kernel<2, 2>, 2u, 2u);
    fn(mb_bundle_kernel<3, 1>, 3u, 1u);
    fn(mb_bundle_kernel<3, 2>, 3u, 2u);
    fn(mb_bundle_kernel<4, 1>, 4u, 1u);
    fn(mb_bundle_kernel<4, 2>, 4u, 2u);
  };
  for_each_instance([&](auto bun, uint32_t kg, uint32_t kl) {
    if (kg != grouping || kl != l)
      return;
    bun<<<dim3(steps, 2, 4), 256, 0, stream>>>(bundle, bsk, t.gen_root[10],
                                              t.mono2048, lwe_in, in_idx, n,
                                              num_samples);
  });
  B200_CHECK(cudaGetLastError());
  count_launch();
  // l = 1: the bundle block of a step comes through the bulk-copy (TMA) ring
  // B200_MULTIBIT_SEQ_TMA=0 selects the register-prefetch variant for A/B runs
  static const bool use_tma = [] {
    const char *e = std::getenv("B200_MULTIBIT_SEQ_TMA");
    return !e || std::atoi(e) != 0;
  }();
  // [grouping - 2][l - 1][register prefetch, TMA ring]
  static const char *const ll_names[3][2][2] = {
      {{"multibit_ll<2,1,regs>", "multibit_ll<2,1,tma>"}, {"multibit_ll<2,2,regs>", ""}},
      {{"multibit_ll<3,1,regs>", "multibit_ll<3,1,tma>"}, {"multibit_ll<3,2,regs>", ""}},
      {{"multibit_ll<4,1,regs>", "multibit_ll<4,1,tma>"}, {"multibit_ll<4,2,regs>", ""}}};
  t_last_pbs_kernel = ll_names[grouping - 2][l - 1][l == 1 && use_tma];
  if (l == 1 && use_tma) {
    pbs_multibit_seq_kernel<1, true>
        <<<num_samples, 128, sizeof(MbSeqSmemTma), stream>>>(
            lwe_out, out_idx, luts, lut_idx, lwe_in, in_idx, bundle, t.fft1024,
            n, steps, base_log, num_many_lut, lut_stride,
            multibit_ties_even().load());
  } else {
    auto seq = l == 1 ? pbs_multibit_seq_kernel<1, false>
                      : pbs_multibit_seq_kernel<2, false>;
    seq<<<num_samples, 128, sizeof(MbSeqSmem), stream>>>(
        lwe_out, out_idx, luts, lut_idx, lwe_in, in_idx, bundle, t.fft1024, n,
        steps, base_log, num_many_lut, lut_stride,
        multibit_ties_even().load());
  }
  B200_CHECK(cudaGetLastError());
  count_launch();
  B200_CHECK(cudaFreeAsync(bundle, stream));
}

// any-(N, k, l) kernel, shared memory or global workspace, 64- or 32-bit torus
template <typename Torus>
static void launch_pbs_generic(cudaStream_t stream, uint32_t gpu_index,
                               Torus *lwe_out, const Torus *out_idx,
                               const Torus *luts, const Torus *lut_idx,
                               const Torus *lwe_in, const Torus *in_idx,
                               const void *bsk, uint32_t n, uint32_t k,
                               uint32_t N, uint32_t base_log, uint32_t l,
                               uint32_t grouping, uint32_t num_samples,
                               uint32_t num_many_lut, uint32_t lut_stride,
                               int centered_ms) {
  const uint32_t logM = ilog2_exact(N) - 1;
  const DeviceTables &t = device_tables(gpu_index, logM);
  const size_t smem = generic_smem_bytes(grouping > 1 ? 16 : n, k, N, l);
  int max_smem = 0;
  B200_CHECK(cudaDeviceGetAttribute(
      &max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, (int)gpu_index));
  // The attribute value must not depend on call arguments in a way that races
  // between host threads: always raise it to the device maximum.
  static std::once_flag gen_once[MAX_GPUS];
  cudaFuncAttributes fattr;
  B200_CHECK(
      cudaFuncGetAttributes(&fattr, pbs_generic_kernel<256, false, Torus>));
  const int max_dyn = max_smem - (int)fattr.sharedSizeBytes;
  std::call_once(gen_once[gpu_index], [max_dyn] {
    B200_CHECK(cudaFuncSetAttribute(
        pbs_generic_kernel<256, false, Torus>,
        cudaFuncAttributeMaxDynamicSharedMemorySize, max_dyn));
  });
  if (smem > (size_t)max_dyn) {
    // working set larger than one SM's shared memory (N >= 8192 ...): same
    // kernel over a per-CTA slice of a stream-ordered global workspace, a
    // persistent grid striding over the samples
    int sms = 0;
    B200_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount,
                                      (int)gpu_index));
    const uint32_t grid = std::min<uint32_t>(num_samples, 2u * (uint32_t)sms);
    const size_t stride = (smem + 255) / 256 * 256;
    unsigned char *ws = nullptr;
    B200_CHECK(cudaMallocFromPoolAsync(&ws, stride * grid,
                                       workspace_pool(gpu_index), stream));
    pbs_generic_kernel<256, true, Torus><<<grid, 256, 0, stream>>>(
        lwe_out, out_idx, luts, lut_idx, lwe_in, in_idx,
        static_cast<const cplx *>(bsk), t.gen_tw[logM], t.gen_root[logM], n, k,
        N, logM, base_log, l, grouping, num_many_lut, lut_stride, centered_ms,
        multibit_ties_even().load(), num_samples, ws, stride);
    B200_CHECK(cudaGetLastError());
    count_launch();
    t_last_pbs_kernel = std::is_same<Torus, uint32_t>::value
                            ? "generic_workspace_u32"
                            : "generic_workspace";
    B200_CHECK(cudaFreeAsync(ws, stream));
    return;
  }
  pbs_generic_kernel<256, false, Torus><<<num_samples, 256, smem, stream>>>(
      lwe_out, out_idx, luts, lut_idx, lwe_in, in_idx,
      static_cast<const cplx *>(bsk), t.gen_tw[logM], t.gen_root[logM], n, k,
      N, logM, base_log, l, grouping, num_many_lut, lut_stride, centered_ms,
      multibit_ties_even().load());
  B200_CHECK(cudaGetLastError());
  count_launch();
  t_last_pbs_kernel =
      std::is_same<Torus, uint32_t>::value ? "generic_smem_u32" : "generic_smem";
}

static void launch_pbs(cudaStream_t stream, uint32_t gpu_index,
                       uint64_t *lwe_out, const uint64_t *out_idx,
                       const uint64_t *luts, const uint64_t *lut_idx,
                       const uint64_t *lwe_in, const uint64_t *in_idx,
                       const void *bsk, uint32_t n, uint32_t k, uint32_t N,
                       uint32_t base_log, uint32_t l, uint32_t grouping,
                       uint32_t num_samples, uint32_t num_many_lut,
                       uint32_t lut_stride, int centered_ms) {
  if (num_samples == 0)
    return;
  check_polynomial_size(N);
  B200_PANIC_IF_FALSE(base_log * l <= 63 && base_log >= 1 && l >= 1,
                      "Cuda error (PBS): base_log * level_count must be < 64");
  if (num_many_lut == 0)
    num_many_lut = 1;
  const uint32_t logM = ilog2_exact(N) - 1;
  if (grouping <= 1 && uses_fast_path(n, k, N, l)) {
    B200_PANIC_IF_FALSE(base_log <= 31, "Cuda error (PBS): base_log > 31");
    const DeviceTables &t = device_tables(gpu_index, 0);
    static std::once_flag attr_once[MAX_GPUS];
    std::call_once(attr_once[gpu_index], [] {
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(P22Smem)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v3_kernel<0, 0>,
          cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(P22SmemV3)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v3_kernel<0, 1>,
          cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(P22SmemV3)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v3_kernel<1, 1>,
          cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(P22SmemV3)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v3_kernel<2, 1>,
          cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(P22SmemV3)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v3_kernel<3, 1>,
          cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(P22SmemV3Tma)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v3_kernel<0, 1, 1>,
          cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(P22SmemV3)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v6_kernel<0, false>,
          cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(P22SmemV6<4, false>)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v6_kernel<0, true>,
          cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(P22SmemV6<4, true>)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v6_kernel<1, true>,
          cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(P22SmemV6<1, true>)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v6_kernel<2, true>,
          cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(P22SmemV6<2, true>)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v6_kernel<0, true, 1>,
          cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(P22SmemV6<4, true>)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v6_kernel<2, true, 1>,
          cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(P22SmemV6<2, true>)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v6_kernel<0, true, 2, 1>,
          cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(P22SmemV6<4, true>)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v6_kernel<2, true, 2, 1>,
          cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(P22SmemV6<2, true>)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v6_kernel<2, true, 2, 2>,
          cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(P22SmemV6<2, true>)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v6_kernel<0, true, 2>,
          cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(P22SmemV6<4, true>)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v6_kernel<2, true, 2>,
          cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(P22SmemV6<2, true>)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n2048_k1_l1_v6_kernel<2, true, 3>,
          cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(P22SmemV6<2, true>)));
    });
    auto launch_reg = [&](auto kernel, size_t smem, const char *name) {
      kernel<<<num_samples, 128, smem, stream>>>(
          lwe_out, out_idx, luts, lut_idx, lwe_in, in_idx,
          static_cast<const cplx *>(bsk), t.fft1024, n, base_log,
          num_many_lut, lut_stride, centered_ms);
      t_last_pbs_kernel = name;
    };
    const int variant = fast_variant();
    if (variant == 1 || base_log > 30) {
      // v1: 64-bit accumulator (A/B measurements and base_log = 31)
      launch_reg(pbs_n2048_k1_l1_kernel, sizeof(P22Smem), "n2048_v1");
    } else if (variant == 3) {
      launch_reg(pbs_n2048_k1_l1_v3_kernel<0, 0>, sizeof(P22SmemV3), "n2048_v3<0,0>"); // round 1
    } else if (variant == 5) {
      launch_reg(pbs_n2048_k1_l1_v3_kernel<0, 1>, sizeof(P22SmemV3), "n2048_v3<0,1>");
    } else if (variant == 4) {
      launch_reg(pbs_n2048_k1_l1_v3_kernel<1, 1>, sizeof(P22SmemV3), "n2048_v3<1,1>");
    } else if (variant == 6) {
      launch_reg(pbs_n2048_k1_l1_v3_kernel<2, 1>, sizeof(P22SmemV3), "n2048_v3<2,1>");
    } else if (variant == 7) {
      // TMA ring for the key block: 208 KiB of shared memory, one CTA per SM
      launch_reg(pbs_n2048_k1_l1_v3_kernel<3, 1>, sizeof(P22SmemV3Tma), "n2048_v3<3,1>");
    } else if (variant == 8) {
      // exchange 2 through warp shuffles (x2_shfl.cuh)
      launch_reg(pbs_n2048_k1_l1_v3_kernel<0, 1, 1>, sizeof(P22SmemV3), "n2048_v3<0,1,1>");
    } else if (variant == 9) {
      // v6: shuffle exchange 2 + one-slot TMA key ring, 2 CTAs / SM
      launch_reg(pbs_n2048_k1_l1_v6_kernel<0, false>, sizeof(P22SmemV6<4, false>),
                 "n2048_v6<0,false>");
    } else if (variant == 10) {
      // v6 with v3's register key prefetch (isolates the ring)
      launch_reg(pbs_n2048_k1_l1_v6_kernel<1, true>, sizeof(P22SmemV6<1, true>),
                 "n2048_v6<1,true>");
    } else if (variant == 11) {
      // v6 hybrid: own row in registers, other row through the ring
      launch_reg(pbs_n2048_k1_l1_v6_kernel<2, true>, sizeof(P22SmemV6<2, true>),
                 "n2048_v6<2,true>");
    } else if (variant == 14) {
      // v6 with the switched mask staged in shared memory: one CTA per SM
      launch_reg(pbs_n2048_k1_l1_v6_kernel<0, true>, sizeof(P22SmemV6<4, true>),
                 "n2048_v6<0,true>");
    } else if (variant == 15) {
      // v6 ring, digits converted through the fp64 ADD pipe instead of I2F
      launch_reg(pbs_n2048_k1_l1_v6_kernel<0, true, 1>, sizeof(P22SmemV6<4, true>),
                 "n2048_v6<0,true,1>");
    } else if (variant == 16) {
      launch_reg(pbs_n2048_k1_l1_v6_kernel<2, true, 1>, sizeof(P22SmemV6<2, true>),
                 "n2048_v6<2,true,1>");
    } else if (variant == 20) {
      // the shipped two-CTA instance (lane-pair layout, see below)
      launch_reg(pbs_n2048_k1_l1_v6_kernel<2, true, 2, 1>, sizeof(P22SmemV6<2, true>),
                 "n2048_v6<2,true,2,1>");
    } else if (variant == 22) {
      // v6 hybrid with both CTA barriers of a step split (own-row products before
      // the wait for the other group's spectrum)
      launch_reg(pbs_n2048_k1_l1_v6_kernel<2, true, 2, 2>, sizeof(P22SmemV6<2, true>),
                 "n2048_v6<2,true,2,2>");
    } else if (variant == 21) {
      launch_reg(pbs_n2048_k1_l1_v6_kernel<0, true, 2, 1>, sizeof(P22SmemV6<4, true>),
                 "n2048_v6<0,true,2,1>");
    } else if (variant == 19) {
      launch_reg(pbs_n2048_k1_l1_v6_kernel<0, true, 2>, sizeof(P22SmemV6<4, true>),
                 "n2048_v6<0,true,2>");
    } else if (variant == 17) {
      launch_reg(pbs_n2048_k1_l1_v6_kernel<2, true, 2>, sizeof(P22SmemV6<2, true>),
                 "n2048_v6<2,true,2>");
    } else if (variant == 18) {
      launch_reg(pbs_n2048_k1_l1_v6_kernel<2, true, 3>, sizeof(P22SmemV6<2, true>),
                 "n2048_v6<2,true,3>");
    } else if (num_samples <= sm_count(gpu_index)) {
      // shipped, at most one CTA per SM: v6 with the whole key block of a step
      // through the one-slot TMA ring (no key value is ever waited for) and
      // exchange 2 through warp shuffles
      launch_reg(pbs_n2048_k1_l1_v6_kernel<0, true, 2>, sizeof(P22SmemV6<4, true>),
                 "n2048_v6<0,true,2>");
    } else {
      // shipped, two CTAs per SM: v6 hybrid -- own key row prefetched into
      // registers, other row (the one v3 waited a full L2 round trip for)
      // through the ring; rotate + decompose with the sign as a predicate
      // (CVT = 2); lane-pair layout: each warp holds the same 16 threads of
      // both polynomials (lanes l and l ^ 16), exchange 2 through half-warp
      // shuffles, the other polynomial's spectrum taken with one shuffle in
      // the MAC (no spectrum store, no barrier between the polynomials).
      // Bit-identical to variant 17, the same instance in the 64-thread
      // group layout.
      launch_reg(pbs_n2048_k1_l1_v6_kernel<2, true, 2, 1>, sizeof(P22SmemV6<2, true>),
                 "n2048_v6<2,true,2,1>");
    }
    B200_CHECK(cudaGetLastError());
    count_launch();
    return;
  }
  if (grouping <= 1 && uses_n8192_path(n, k, N, l)) {
    B200_PANIC_IF_FALSE(base_log * l <= 30,
                        "Cuda error (PBS): base_log * level_count > 30 is not "
                        "supported for N = 8192");
    const DeviceTables &t = device_tables(gpu_index, 0);
    static std::once_flag once8k[MAX_GPUS];
    std::call_once(once8k[gpu_index], [] {
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n8192_k1_l2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(N8192Smem)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n8192_k1_l2_v2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(N8192SmemV2)));
      B200_CHECK(cudaFuncSetAttribute(
          pbs_n8192_k1_l2_v2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(N8192SmemV2)));
    });
    const uint32_t grid = std::min(num_samples, sm_count(gpu_index));
    // per-thread park area of the four spectra of a step (pbs_n8192.cuh)
    cplx *park = nullptr;
    B200_CHECK(cudaMallocFromPoolAsync(&park, (size_t)grid * P8K_PARK_PER_CTA * sizeof(cplx),
                                       workspace_pool(gpu_index), stream));
    // mask bit 2: the first-generation kernel (per-thread key loads), for A/B
    if (register_kernel_mask().load() & 4) {
      pbs_n8192_k1_l2_kernel<<<grid, 256, sizeof(N8192Smem), stream>>>(
          lwe_out, out_idx, luts, lut_idx, lwe_in, in_idx,
          static_cast<const cplx *>(bsk), t.fft4096, n, base_log, num_samples,
          num_many_lut, lut_stride, centered_ms, multibit_ties_even().load(), park);
      t_last_pbs_kernel = "n8192_v1";
    } else {
      static const uint32_t stagger = [] {
        const char *e = std::getenv("B200_N8192_STAGGER");
        return e ? (uint32_t)std::atoi(e) : 0u;
      }();
      // mask bit 3: the racecheck instance (every thread arrives on the ring's
      // `empty` barriers itself)
      const bool racecheck = register_kernel_mask().load() & 8;
      auto kernel = racecheck ? pbs_n8192_k1_l2_v2_kernel<true>
                              : pbs_n8192_k1_l2_v2_kernel<false>;
      kernel<<<grid, 256, sizeof(N8192SmemV2), stream>>>(
          lwe_out, out_idx, luts, lut_idx, lwe_in, in_idx,
          static_cast<const cplx *>(bsk), t.fft4096, n, base_log, num_samples,
          num_many_lut, lut_stride, centered_ms, multibit_ties_even().load(),
          stagger, park);
      t_last_pbs_kernel = racecheck ? "n8192_v2<true>" : "n8192_v2<false>";
    }
    B200_CHECK(cudaGetLastError());
    count_launch();
    B200_CHECK(cudaFreeAsync(park, stream));
    return;
  }
  if (grouping <= 1 && uses_n512_path(n, k, N, l)) {
    B200_PANIC_IF_FALSE(base_log <= 31, "Cuda error (PBS): base_log > 31");
    const DeviceTables &t = device_tables(gpu_index, 0);
    // B200_N512_MODE: 0 (default) TMA key ring, one CTA per SM, 1 / 2 / 3 LWEs
    // per CTA by launch size; 2 / 3: ring with two / one LWE per CTA; 4: ring with
    // three; 1: register key ring, two LWEs per CTA, two CTAs per SM
    const int mode512 = n512_mode_sel().load();
    static std::once_flag once512[MAX_GPUS];
    auto set_attr = [](auto kernel, size_t smem) {
      B200_CHECK(cudaFuncSetAttribute(
          kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    };
    std::call_once(once512[gpu_index], [&] {
      set_attr(pbs_n512_kernel<1, 2, false>, sizeof(N512Smem<1, 2, false>));
      set_attr(pbs_n512_kernel<2, 2, false>, sizeof(N512Smem<2, 2, false>));
      set_attr(pbs_n512_kernel<3, 2, false>, sizeof(N512Smem<3, 2, false>));
      set_attr(pbs_n512_kernel<4, 2, false>, sizeof(N512Smem<4, 2, false>));
      set_attr(pbs_n512_kernel<1, 2, true>, sizeof(N512Smem<1, 2, true>));
      set_attr(pbs_n512_kernel<2, 2, true>, sizeof(N512Smem<2, 2, true>));
      set_attr(pbs_n512_kernel<3, 2, true>, sizeof(N512Smem<3, 2, true>));
      set_attr(pbs_n512_kernel<4, 2, true>, sizeof(N512Smem<4, 2, true>));
      set_attr(pbs_n512_kernel<1, 1, true>, sizeof(N512Smem<1, 1, true>));
      set_attr(pbs_n512_kernel<2, 1, true>, sizeof(N512Smem<2, 1, true>));
      set_attr(pbs_n512_kernel<3, 1, true>, sizeof(N512Smem<3, 1, true>));
      set_attr(pbs_n512_kernel<4, 1, true>, sizeof(N512Smem<4, 1, true>));
      set_attr(pbs_n512_kernel<1, 3, true>, sizeof(N512Smem<1, 3, true>));
      set_attr(pbs_n512_kernel<2, 3, true>, sizeof(N512Smem<2, 3, true>));
      set_attr(pbs_n512_kernel<3, 3, true>, sizeof(N512Smem<3, 3, true>));
      set_attr(pbs_n512_kernel<4, 3, true>, sizeof(N512Smem<4, 3, true>));
    });
    auto launch512 = [&](auto kernel, size_t smem, uint32_t G, uint32_t ctas_per_sm,
                         const char *name) {
      // persistent grid (see the kernel)
      const uint32_t groups = (num_samples + G - 1) / G;
      const uint32_t grid = std::min(groups, ctas_per_sm * sm_count(gpu_index));
      kernel<<<grid, 16 * (k + 1) * G, smem, stream>>>(
          lwe_out, out_idx, luts, lut_idx, lwe_in, in_idx,
          static_cast<const cplx *>(bsk), t.fft256, n, base_log, num_samples,
          num_many_lut, lut_stride, centered_ms);
      t_last_pbs_kernel = name;
    };
    // automatic: the fewest LWEs per CTA that still covers the launch in one
    // round of the persistent grid (latency), three per CTA beyond that
    // (throughput)
    const uint32_t sms = sm_count(gpu_index);
    const int per_cta = mode512 == 3 ? 1 : mode512 == 2 ? 2 : mode512 == 0 && num_samples <= sms ? 1
                        : mode512 == 0 && num_samples <= 2 * sms ? 2 : 3;
#define B200_LAUNCH512(K)                                                       \
  if (mode512 == 1)                                                             \
    launch512(pbs_n512_kernel<K, 2, false>, sizeof(N512Smem<K, 2, false>), 2, 2, \
              "n512<" #K ",2,false>");                                          \
  else if (per_cta == 1)                                                        \
    launch512(pbs_n512_kernel<K, 1, true>, sizeof(N512Smem<K, 1, true>), 1, 1,  \
              "n512<" #K ",1,true>");                                           \
  else if (per_cta == 2)                                                        \
    launch512(pbs_n512_kernel<K, 2, true>, sizeof(N512Smem<K, 2, true>), 2, 1,  \
              "n512<" #K ",2,true>");                                           \
  else                                                                          \
    launch512(pbs_n512_kernel<K, 3, true>, sizeof(N512Smem<K, 3, true>), 3, 1,  \
              "n512<" #K ",3,true>")
    switch (k) {
    case 1: B200_LAUNCH512(1); break;
    case 2: B200_LAUNCH512(2); break;
    case 3: B200_LAUNCH512(3); break;
    default: B200_LAUNCH512(4); break;
    }
#undef B200_LAUNCH512
    B200_CHECK(cudaGetLastError());
    count_launch();
    return;
  }
  if (grouping > 1 && uses_multibit_fast_path(k, N, l, grouping)) {
    B200_PANIC_IF_FALSE(n % grouping == 0,
                        "Cuda error (multi-bit PBS): grouping factor must "
                        "divide the lwe dimension");
    B200_PANIC_IF_FALSE(base_log * l <= 31,
                        "Cuda error (multi-bit PBS): base_log * level_count "
                        "> 31 is not supported for N = 2048, k = 1");
    const DeviceTables &t = device_tables(gpu_index, 10);
    static std::once_flag mb_once[MAX_GPUS];
    auto for_each_instance = [&](auto &&fn) {
      fn(pbs_multibit_n2048_k1_kernel<2, 1>, 2u, 1u, "multibit_fused<2,1>");
      fn(pbs_multibit_n2048_k1_kernel<2, 2>, 2u, 2u, "multibit_fused<2,2>");
      fn(pbs_multibit_n2048_k1_kernel<3, 1>, 3u, 1u, "multibit_fused<3,1>");
      fn(pbs_multibit_n2048_k1_kernel<3, 2>, 3u, 2u, "multibit_fused<3,2>");
      fn(pbs_multibit_n2048_k1_kernel<4, 1>, 4u, 1u, "multibit_fused<4,1>");
      fn(pbs_multibit_n2048_k1_kernel<4, 2>, 4u, 2u, "multibit_fused<4,2>");
    };
    std::call_once(mb_once[gpu_index], [&] {
      for_each_instance([](auto kernel, uint32_t, uint32_t, const char *) {
        B200_CHECK(cudaFuncSetAttribute(
            kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
            (int)sizeof(MbSmem)));
      });
    });
    // low-latency mode for launches that cannot fill the GPU with the fused
    // kernel: bundle for all groups at once, then the sequential products
    if (num_samples <= multibit_ll_max_samples(gpu_index)) {
      launch_multibit_ll(stream, gpu_index, lwe_out, out_idx, luts, lut_idx,
                         lwe_in, in_idx, static_cast<const cplx *>(bsk), t, n,
                         base_log, l, grouping, num_samples, num_many_lut,
                         lut_stride);
      return;
    }
    for_each_instance([&](auto kernel, uint32_t kg, uint32_t kl, const char *name) {
      if (kg != grouping || kl != l)
        return;
      kernel<<<num_samples, 128, sizeof(MbSmem), stream>>>(
          lwe_out, out_idx, luts, lut_idx, lwe_in, in_idx,
          static_cast<const cplx *>(bsk), t.fft1024, t.gen_root[10],
          t.mono2048, n, base_log, num_many_lut, lut_stride,
          multibit_ties_even().load());
      t_last_pbs_kernel = name;
    });
    B200_CHECK(cudaGetLastError());
    count_launch();
    return;
  }
  if (grouping > 1) {
    B200_PANIC_IF_FALSE(grouping <= 4 && n % grouping == 0,
                        "Cuda error (multi-bit PBS): grouping factor must be "
                        "2, 3 or 4 and divide the lwe dimension");
  }
  launch_pbs_generic<uint64_t>(stream, gpu_index, lwe_out, out_idx, luts,
                               lut_idx, lwe_in, in_idx, bsk, n, k, N, base_log,
                               l, grouping, num_samples, num_many_lut,
                               lut_stride, centered_ms);
}

// standard-domain BSK (device staging buffer) -> Fourier BSK in the engine's
// layout
static void convert_bsk_staged(cudaStream_t stream, uint32_t gpu_index,
                               void *dest, const uint64_t *staging, uint32_t k,
                               uint32_t N, uint32_t l, uint32_t num_ggsw,
                               bool fast_layout, uint32_t multibit_grouping) {
  const uint32_t logM = ilog2_exact(N) - 1;
  const size_t polys = (size_t)num_ggsw * l * (k + 1) * (k + 1);
  const DeviceTables &t = device_tables(gpu_index, fast_layout ? 0 : logM);
  if (multibit_grouping) {
    bsk_convert_multibit_n2048_kernel<<<(unsigned)polys, 64, 0, stream>>>(
        static_cast<cplx *>(dest), staging, t.fft1024, l, multibit_grouping);
  } else if (fast_layout) {
    bsk_convert_n2048_k1_l1_kernel<<<(unsigned)polys, 64, 0, stream>>>(
        static_cast<cplx *>(dest), staging, t.fft1024);
  } else if (uses_n8192_path(num_ggsw, k, N, l)) {
    static std::once_flag conv8k_once[MAX_GPUS];
    std::call_once(conv8k_once[gpu_index], [] {
      B200_CHECK(cudaFuncSetAttribute(
          bsk_convert_n8192_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)(P8K_M * sizeof(cplx))));
    });
    bsk_convert_n8192_kernel<<<(unsigned)polys, 256, P8K_M * sizeof(cplx),
                               stream>>>(static_cast<cplx *>(dest), staging,
                                         t.fft4096);
  } else if (uses_n512_path(num_ggsw, k, N, l)) {
    bsk_convert_n512_kernel<<<(unsigned)((polys + 1) / 2), 32, 0, stream>>>(
        static_cast<cplx *>(dest), staging, t.fft256, k + 1, (uint32_t)polys);
  } else {
    static std::once_flag conv_once[MAX_GPUS];
    std::call_once(conv_once[gpu_index], [] {
      B200_CHECK(cudaFuncSetAttribute(
          bsk_convert_generic_kernel<uint64_t>,
          cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 / 2 * 16));
      B200_CHECK(cudaFuncSetAttribute(
          bsk_convert_generic_kernel<uint32_t>,
          cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 / 2 * 16));
    });
    bsk_convert_generic_kernel<uint64_t>
        <<<(unsigned)polys, 256, (N / 2) * sizeof(cplx), stream>>>(
            static_cast<cplx *>(dest), staging, t.gen_tw[logM], N, logM);
  }
  B200_CHECK(cudaGetLastError());
  count_launch();
}

// host standard-domain BSK -> device Fourier BSK in the engine's layout
static void convert_bsk(cudaStream_t stream, uint32_t gpu_index, void *dest,
                        const void *src_host, uint32_t n, uint32_t k,
                        uint32_t N, uint32_t l, uint32_t num_ggsw,
                        bool fast_layout, uint32_t multibit_grouping = 0) {
  (void)n;
  check_polynomial_size(N);
  const size_t polys = (size_t)num_ggsw * l * (k + 1) * (k + 1);
  const size_t bytes = polys * N * sizeof(uint64_t);
  uint64_t *staging = nullptr;
  B200_CHECK(cudaMallocAsync(&staging, bytes, stream));
  B200_CHECK(cudaMemcpyAsync(staging, src_host, bytes, cudaMemcpyHostToDevice,
                             stream));
  convert_bsk_staged(stream, gpu_index, dest, staging, k, N, l, num_ggsw,
                     fast_layout, multibit_grouping);
  B200_CHECK(cudaFreeAsync(staging, stream));
}

// AES-128 S-box / T-table, built once on the host and once per GPU
static const AesTables &aes_host_tables() {
  static AesTables host_tables;
  static std::once_flag host_once;
  std::call_once(host_once, [] { aes_fill_tables(host_tables); });
  return host_tables;
}
static const AesTables *aes_device_tables(uint32_t gpu_index) {
  static AesTables *dev_tables[MAX_GPUS] = {};
  static std::once_flag dev_once[MAX_GPUS];
  std::call_once(dev_once[gpu_index], [gpu_index] {
    B200_CHECK(cudaMalloc(&dev_tables[gpu_index], sizeof(AesTables)));
    B200_CHECK(cudaMemcpy(dev_tables[gpu_index], &aes_host_tables(),
                          sizeof(AesTables), cudaMemcpyHostToDevice));
  });
  return dev_tables[gpu_index];
}

// seeded OPRF masks -> num_blocks LWEs of n + 1 words in blind-rotation form
// (oprf.cuh); the counter is advanced past whole blocks of first_byte
static void oprf_expand(cudaStream_t stream, uint32_t gpu_index,
                        uint64_t *lwe_out, const uint8_t aes_key[16],
                        uint64_t ctr_lo, uint64_t ctr_hi, uint64_t first_byte,
                        uint32_t n, uint32_t num_blocks, uint32_t log_modulus) {
  B200_PANIC_IF_FALSE(log_modulus >= 1 && log_modulus <= 16,
                      "Cuda error (OPRF): log_modulus %u out of [1, 16]",
                      log_modulus);
  B200_PANIC_IF_FALSE(n >= 1, "Cuda error (OPRF): lwe_dimension must be >= 1");
  if (num_blocks == 0)
    return;
  const uint64_t skip = first_byte >> 4;
  const uint64_t lo = ctr_lo + skip;
  ctr_hi += lo < ctr_lo ? 1 : 0;
  ctr_lo = lo;
  first_byte &= 15;
  const AesTables *tables = aes_device_tables(gpu_index);
  AesCtrKey key;
  aes_expand_key(aes_key, aes_host_tables(), key);
  const uint64_t width = (log_modulus + 7) / 8;
  const uint64_t last_start = first_byte + width * ((uint64_t)n * num_blocks - 1);
  const uint64_t ctas = last_start / (16 * OPRF_OWNED_BLOCKS) + 1;
  B200_PANIC_IF_FALSE(ctas < (1ull << 31), "Cuda error (OPRF): batch too large");
  oprf_expand_kernel<<<(unsigned)ctas, OPRF_THREADS, 0, stream>>>(
      lwe_out, tables, key, ctr_lo, ctr_hi, (uint32_t)first_byte, n,
      num_blocks, log_modulus);
  B200_CHECK(cudaGetLastError());
  count_launch();
}

// seeded BSK (host bodies + AES-CTR mask seed) -> device Fourier BSK
static void convert_seeded_bsk(cudaStream_t stream, uint32_t gpu_index,
                               void *dest, const void *bodies_host,
                               const uint8_t aes_key[16], uint64_t ctr_lo,
                               uint64_t ctr_hi, uint32_t first_byte_index,
                               uint32_t k, uint32_t N, uint32_t l,
                               uint32_t num_ggsw, bool fast_layout,
                               uint32_t multibit_grouping) {
  check_polynomial_size(N);
  B200_PANIC_IF_FALSE(first_byte_index == 0 || first_byte_index == 8,
                      "Cuda error (seeded key): the mask stream must start on "
                      "a u64 boundary of an AES block (byte index %u)",
                      first_byte_index);
  const AesTables *tables = aes_device_tables(gpu_index);
  AesCtrKey key;
  aes_expand_key(aes_key, aes_host_tables(), key);
  const uint64_t rows = (uint64_t)num_ggsw * l * (k + 1);
  const size_t std_bytes = rows * (k + 1) * N * sizeof(uint64_t);
  const size_t body_bytes = rows * N * sizeof(uint64_t);
  uint64_t *staging = nullptr, *bodies = nullptr;
  B200_CHECK(cudaMallocAsync(&staging, std_bytes, stream));
  B200_CHECK(cudaMallocAsync(&bodies, body_bytes, stream));
  B200_CHECK(cudaMemcpyAsync(bodies, bodies_host, body_bytes,
                             cudaMemcpyHostToDevice, stream));
  seeded_bsk_expand_kernel<<<sm_count(gpu_index) * 8, 256, 0, stream>>>(
      staging, bodies, tables, key, ctr_lo, ctr_hi,
      first_byte_index / 8, rows, k, N);
  B200_CHECK(cudaGetLastError());
  count_launch();
  convert_bsk_staged(stream, gpu_index, dest, staging, k, N, l, num_ggsw,
                     fast_layout, multibit_grouping);
  B200_CHECK(cudaFreeAsync(bodies, stream));
  B200_CHECK(cudaFreeAsync(staging, stream));
}

// ---- test-only forward transform (natural order) ---------------------------
__global__ void __launch_bounds__(64)
forward_fft_natural_kernel(cplx *__restrict__ dst, const cplx *__restrict__ src,
                           const Fft1024Tables *__restrict__ tables) {
  __shared__ cplx xa[P22_M];
  __shared__ cplx xb[P22_M];
  const int t = threadIdx.x;
  const cplx *in = src + (size_t)blockIdx.x * P22_M;
  cplx v[16];
#pragma unroll
  for (int j1 = 0; j1 < 16; j1++)
    v[j1] = in[64 * j1 + t];
  radix16_fwd(v, c_fft1024_pass1);
  x1_store_p1(xa, t, v);
  __syncthreads();
  x1_load_p2(xa, t, v);
  pass2_fwd(v, &tables->pass2[t >> 2][0]);
  x2_store_p2(xb, t, v);
  __syncthreads();
  x2_load_p3(xb, t, v);
  radix16_fwd(v, tables->pass3[t]);
  cplx *out = dst + (size_t)blockIdx.x * P22_M;
  // slot pos holds Z(t^(1 + 4 bitrev(pos))) = reference frequency
  // k = (-bitrev(pos)) mod M  (reference kernel e^{-2 pi i jk/M})
#pragma unroll
  for (int b = 0; b < 16; b++) {
    const uint32_t pos = 16 * t + b;
    const uint32_t kf = __brev(pos) >> 22;
    out[(P22_M - kf) & (P22_M - 1)] = v[b];
  }
}

// sum of the host counts of a flattened compact-list array, each checked
static uint64_t compact_lists_total(const uint32_t *h_counts,
                                    uint32_t num_lists, uint32_t n) {
  B200_PANIC_IF_FALSE(n >= 256 && n <= 16384 && (n & (n - 1)) == 0,
                      "Cuda error (expand): the compact lwe_dimension must be "
                      "a power of two in [256, 16384]. Got %u", n);
  B200_PANIC_IF_FALSE(num_lists >= 1 && h_counts,
                      "Cuda error (expand): no compact list");
  uint64_t total = 0;
  for (uint32_t k = 0; k < num_lists; k++) {
    B200_PANIC_IF_FALSE(h_counts[k] >= 1 && h_counts[k] <= n,
                        "Cuda error (expand): list %u holds %u LWEs, must be "
                        "in [1, %u]", k, h_counts[k], n);
    total += h_counts[k];
  }
  return total;
}

// compact lists -> expanded LWEs of n + 1 words (compact_expand.cuh).  The
// per-list descriptors go to the pool workspace with a stream-ordered copy
// (staged from pageable memory: the host vector may go when this returns).
static void compact_expand(cudaStream_t st, uint32_t gpu_index,
                           uint64_t *lwe_out, const uint64_t *lists_in,
                           const uint32_t *h_counts, uint32_t num_lists,
                           uint32_t n) {
  compact_lists_total(h_counts, num_lists, n);
  std::vector<CompactListDesc> descs(num_lists);
  uint64_t in_offset = 0, out_first = 0, max_count = 0;
  for (uint32_t k = 0; k < num_lists; k++) {
    descs[k] = {in_offset, out_first, h_counts[k]};
    in_offset += n + h_counts[k];
    out_first += h_counts[k];
    max_count = std::max<uint64_t>(max_count, h_counts[k]);
  }
  const size_t bytes = num_lists * sizeof(CompactListDesc);
  CompactListDesc *d_descs = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(&d_descs, bytes, workspace_pool(gpu_index),
                                     st));
  B200_CHECK(cudaMemcpyAsync(d_descs, descs.data(), bytes,
                             cudaMemcpyHostToDevice, st));
  const uint64_t words = max_count * (n + 1);
  const dim3 grid((unsigned)((words + EXPAND_THREADS - 1) / EXPAND_THREADS),
                  std::min<uint32_t>(num_lists, 65535u));
  compact_expand_kernel<<<grid, EXPAND_THREADS, 0, st>>>(lwe_out, lists_in,
                                                         d_descs, num_lists, n);
  B200_CHECK(cudaGetLastError());
  count_launch();
  B200_CHECK(cudaFreeAsync(d_descs, st));
}

// PBS indexes of the unpacking: output s reads cast LWE s >> 1
__global__ void __launch_bounds__(256)
compact_unpack_index_kernel(uint64_t *__restrict__ in_idx,
                            uint64_t *__restrict__ out_idx, uint32_t count) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < count) {
    in_idx[s] = s >> 1;
    out_idx[s] = s;
  }
}

} // namespace b200

using namespace b200;

// ===========================================================================
// extern "C" -- device helpers (tfhe-cuda-common/cuda/src/device.cu)
// ===========================================================================
#pragma GCC visibility push(default)
extern "C" {

void *cuda_create_stream_ffi(uint32_t gpu_index) {
  set_device(gpu_index);
  cudaStream_t stream;
  // non-blocking, like the reference (tfhe-cuda-common/cuda/src/device.cu:155-
  // 160): ABI streams never synchronise implicitly with the legacy default
  // stream
  B200_CHECK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  return stream;
}

void cuda_destroy_stream(void *stream, uint32_t gpu_index) {
  set_device(gpu_index);
  B200_CHECK(cudaStreamDestroy(static_cast<cudaStream_t>(stream)));
}

void cuda_synchronize_stream(void *stream, uint32_t gpu_index) {
  set_device(gpu_index);
  B200_CHECK(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
}

uint32_t cuda_is_available(void) {
  int count = 0;
  return cudaGetDeviceCount(&count) == cudaSuccess && count > 0;
}

void *cuda_malloc(uint64_t size, uint32_t gpu_index) {
  set_device(gpu_index);
  void *ptr = nullptr;
  B200_CHECK(cudaMalloc(&ptr, size));
  return ptr;
}

void *cuda_malloc_async(uint64_t size, void *stream, uint32_t gpu_index) {
  set_device(gpu_index);
  void *ptr = nullptr;
  B200_CHECK(cudaMallocAsync(&ptr, size, static_cast<cudaStream_t>(stream)));
  return ptr;
}

bool cuda_check_valid_malloc(uint64_t size, uint32_t gpu_index) {
  set_device(gpu_index);
  size_t free_mem = 0, total_mem = 0;
  B200_CHECK(cudaMemGetInfo(&free_mem, &total_mem));
  return size <= free_mem;
}

uint64_t cuda_device_total_memory(uint32_t gpu_index) {
  set_device(gpu_index);
  size_t free_mem = 0, total_mem = 0;
  B200_CHECK(cudaMemGetInfo(&free_mem, &total_mem));
  return total_mem;
}

static void check_device_ptr(const void *p, const char *what) {
  cudaPointerAttributes attr;
  B200_CHECK(cudaPointerGetAttributes(&attr, p));
  if (attr.type != cudaMemoryTypeDevice && attr.type != cudaMemoryTypeManaged)
    B200_PANIC("Cuda error: invalid device pointer in %s.", what);
}

void cuda_memcpy_async_to_gpu(void *dest, const void *src, uint64_t size,
                              void *stream, uint32_t gpu_index) {
  if (size == 0)
    return;
  set_device(gpu_index);
  check_device_ptr(dest, "cuda_memcpy_async_to_gpu");
  B200_CHECK(cudaMemcpyAsync(dest, src, size, cudaMemcpyHostToDevice,
                             static_cast<cudaStream_t>(stream)));
}

void cuda_memcpy_async_gpu_to_gpu(void *dest, void const *src, uint64_t size,
                                  void *stream, uint32_t gpu_index) {
  if (size == 0)
    return;
  // peer aware, like the reference (device.cu:314-330): the two pointers may
  // live on different GPUs (multi-GPU scatter / gather of LWE lists)
  cudaPointerAttributes sa, da;
  B200_CHECK(cudaPointerGetAttributes(&sa, src));
  B200_CHECK(cudaPointerGetAttributes(&da, dest));
  B200_PANIC_IF_FALSE(sa.type == cudaMemoryTypeDevice ||
                          sa.type == cudaMemoryTypeManaged,
                      "Cuda error: invalid device pointer (src) in "
                      "cuda_memcpy_async_gpu_to_gpu.");
  B200_PANIC_IF_FALSE(da.type == cudaMemoryTypeDevice ||
                          da.type == cudaMemoryTypeManaged,
                      "Cuda error: invalid device pointer (dest) in "
                      "cuda_memcpy_async_gpu_to_gpu.");
  set_device(gpu_index);
  if (sa.device == da.device) {
    B200_CHECK(cudaMemcpyAsync(dest, src, size, cudaMemcpyDeviceToDevice,
                               static_cast<cudaStream_t>(stream)));
  } else {
    B200_CHECK(cudaMemcpyPeerAsync(dest, da.device, src, sa.device, size,
                                   static_cast<cudaStream_t>(stream)));
  }
}

void cuda_memcpy_gpu_to_gpu(void *dest, void const *src, uint64_t size,
                            uint32_t gpu_index) {
  if (size == 0)
    return;
  set_device(gpu_index);
  B200_CHECK(cudaMemcpy(dest, src, size, cudaMemcpyDeviceToDevice));
}

void cuda_memcpy_async_to_cpu(void *dest, const void *src, uint64_t size,
                              void *stream, uint32_t gpu_index) {
  if (size == 0)
    return;
  set_device(gpu_index);
  check_device_ptr(src, "cuda_memcpy_async_to_cpu");
  B200_CHECK(cudaMemcpyAsync(dest, src, size, cudaMemcpyDeviceToHost,
                             static_cast<cudaStream_t>(stream)));
}

void cuda_memset_async(void *dest, uint64_t val, uint64_t size, void *stream,
                       uint32_t gpu_index) {
  if (size == 0)
    return;
  set_device(gpu_index);
  check_device_ptr(dest, "cuda_memset_async");
  B200_CHECK(cudaMemsetAsync(dest, (int)val, size,
                             static_cast<cudaStream_t>(stream)));
}

int cuda_get_number_of_gpus(void) {
  int count = 0;
  B200_CHECK(cudaGetDeviceCount(&count));
  return count;
}

int cuda_get_number_of_sms(void) {
  int sms = 0;
  B200_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  return sms;
}

void cuda_synchronize_device(uint32_t gpu_index) {
  set_device(gpu_index);
  B200_CHECK(cudaDeviceSynchronize());
}

void cuda_drop(void *ptr, uint32_t gpu_index) {
  set_device(gpu_index);
  B200_CHECK(cudaFree(ptr));
}

void cuda_drop_async(void *ptr, void *stream, uint32_t gpu_index) {
  set_device(gpu_index);
  B200_CHECK(cudaFreeAsync(ptr, static_cast<cudaStream_t>(stream)));
}

uint32_t cuda_get_max_shared_memory(uint32_t gpu_index) {
  int v = 0;
  B200_CHECK(cudaDeviceGetAttribute(
      &v, cudaDevAttrMaxSharedMemoryPerBlockOptin, (int)gpu_index));
  return (uint32_t)v;
}

// ===========================================================================
// classic PBS
// ===========================================================================
void cuda_convert_lwe_programmable_bootstrap_key_64_async(
    void *stream, uint32_t gpu_index, void *dest, void const *src,
    uint32_t input_lwe_dim, uint32_t glwe_dim, uint32_t level_count,
    uint32_t polynomial_size) {
  set_device(gpu_index);
  convert_bsk(static_cast<cudaStream_t>(stream), gpu_index, dest, src,
              input_lwe_dim, glwe_dim, polynomial_size, level_count,
              input_lwe_dim,
              uses_fast_path(input_lwe_dim, glwe_dim, polynomial_size,
                             level_count));
}

uint64_t scratch_cuda_programmable_bootstrap_64_async(
    void *stream, uint32_t gpu_index, int8_t **buffer, uint32_t lwe_dimension,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t level_count,
    uint32_t input_lwe_ciphertext_count, bool allocate_gpu_memory,
    PBS_MS_REDUCTION_T noise_reduction_type) {
  (void)stream;
  set_device(gpu_index);
  check_polynomial_size(polynomial_size);
  PbsScratch *s = new PbsScratch;
  s->magic = SCRATCH_MAGIC;
  s->type = CLASSICAL;
  s->glwe_dim = glwe_dimension;
  s->poly_size = polynomial_size;
  s->level_count = level_count;
  s->max_samples = input_lwe_ciphertext_count;
  s->centered_ms = noise_reduction_type == CENTERED;
  s->gpu_memory_allocated = allocate_gpu_memory;
  // per-device constant tables are built here (set-up call), so that the
  // *_async bootstrap itself never runs a synchronous copy
  device_tables(gpu_index,
                uses_fast_path(lwe_dimension, glwe_dimension, polynomial_size,
                               level_count)
                    ? 0
                    : ilog2_exact(polynomial_size) - 1);
  *buffer = reinterpret_cast<int8_t *>(s);
  // The persistent kernels keep every intermediate in shared memory /
  // registers: no device workspace is needed, whatever the batch size.
  return 0;
}

void cuda_programmable_bootstrap_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lut_vector,
    void const *lut_vector_indexes, void const *lwe_array_in,
    void const *lwe_input_indexes, void const *bootstrapping_key,
    int8_t *buffer, uint32_t lwe_dimension, uint32_t glwe_dimension,
    uint32_t polynomial_size, uint32_t base_log, uint32_t level_count,
    uint32_t num_samples, uint32_t num_many_lut, uint32_t lut_stride) {
  set_device(gpu_index);
  const PbsScratch *s = reinterpret_cast<const PbsScratch *>(buffer);
  B200_PANIC_IF_FALSE(s && s->magic == SCRATCH_MAGIC && s->type == CLASSICAL,
                      "Cuda error (classical PBS): invalid scratch buffer");
  B200_PANIC_IF_FALSE(
      s->glwe_dim == glwe_dimension && s->poly_size == polynomial_size &&
          s->level_count == level_count,
      "Cuda error (classical PBS): scratch buffer was created for other "
      "parameters");
  B200_PANIC_IF_FALSE(base_log <= 64,
                      "Cuda error (classical PBS): base log should be <= 64");
  launch_pbs(static_cast<cudaStream_t>(stream), gpu_index,
             static_cast<uint64_t *>(lwe_array_out),
             static_cast<const uint64_t *>(lwe_output_indexes),
             static_cast<const uint64_t *>(lut_vector),
             static_cast<const uint64_t *>(lut_vector_indexes),
             static_cast<const uint64_t *>(lwe_array_in),
             static_cast<const uint64_t *>(lwe_input_indexes),
             bootstrapping_key, lwe_dimension, glwe_dimension, polynomial_size,
             base_log, level_count, 1, num_samples, num_many_lut, lut_stride,
             s->centered_ms);
}

void cleanup_cuda_programmable_bootstrap_64(void *stream, uint32_t gpu_index,
                                            int8_t **pbs_buffer) {
  set_device(gpu_index);
  // release-ordering rule of the reference: synchronise before freeing
  B200_CHECK(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
  PbsScratch *s = reinterpret_cast<PbsScratch *>(*pbs_buffer);
  if (s) {
    // same two steps as the reference (programmable_bootstrap_classic.cu:939-
    // 945): release, then delete through the base
    pbs_buffer_base_abi *base = s;
    base->release(static_cast<cudaStream_t>(stream), gpu_index);
    delete base;
  }
  *pbs_buffer = nullptr;
}

// ---- u32 torus (programmable_bootstrap.h:47-50,72-79) -----------------------
// The reference has no scratch function for the 32-bit PBS (its buffer type is
// only reachable from C++): the `buffer` argument here is a scratch object of
// scratch_cuda_programmable_bootstrap_64_async with the same (k, N, l).  Key,
// ciphertexts, accumulators and the three index vectors are all u32.
void cuda_convert_lwe_programmable_bootstrap_key_32_async(
    void *stream, uint32_t gpu_index, void *dest, void const *src,
    uint32_t input_lwe_dim, uint32_t glwe_dim, uint32_t level_count,
    uint32_t polynomial_size) {
  set_device(gpu_index);
  check_polynomial_size(polynomial_size);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint32_t logM = ilog2_exact(polynomial_size) - 1;
  const size_t polys =
      (size_t)input_lwe_dim * level_count * (glwe_dim + 1) * (glwe_dim + 1);
  const size_t bytes = polys * polynomial_size * sizeof(uint32_t);
  const DeviceTables &t = device_tables(gpu_index, logM);
  uint32_t *staging = nullptr;
  B200_CHECK(cudaMallocAsync(&staging, bytes, st));
  B200_CHECK(cudaMemcpyAsync(staging, src, bytes, cudaMemcpyHostToDevice, st));
  static std::once_flag once[MAX_GPUS];
  std::call_once(once[gpu_index], [] {
    B200_CHECK(cudaFuncSetAttribute(
        bsk_convert_generic_kernel<uint32_t>,
        cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 / 2 * 16));
  });
  bsk_convert_generic_kernel<uint32_t>
      <<<(unsigned)polys, 256, (polynomial_size / 2) * sizeof(cplx), st>>>(
          static_cast<cplx *>(dest), staging, t.gen_tw[logM], polynomial_size,
          logM);
  B200_CHECK(cudaGetLastError());
  count_launch();
  B200_CHECK(cudaFreeAsync(staging, st));
}

void cuda_programmable_bootstrap_lwe_ciphertext_vector_32_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lut_vector,
    void const *lut_vector_indexes, void const *lwe_array_in,
    void const *lwe_input_indexes, void const *bootstrapping_key,
    int8_t *buffer, uint32_t lwe_dimension, uint32_t glwe_dimension,
    uint32_t polynomial_size, uint32_t base_log, uint32_t level_count,
    uint32_t num_samples, uint32_t num_many_lut, uint32_t lut_stride) {
  set_device(gpu_index);
  const PbsScratch *s = reinterpret_cast<const PbsScratch *>(buffer);
  B200_PANIC_IF_FALSE(s && s->magic == SCRATCH_MAGIC && s->type == CLASSICAL,
                      "Cuda error (classical PBS): invalid scratch buffer");
  B200_PANIC_IF_FALSE(base_log <= 32,
                      "Cuda error (classical PBS): base log should be <= 32");
  if (num_samples == 0)
    return;
  check_polynomial_size(polynomial_size);
  launch_pbs_generic<uint32_t>(
      static_cast<cudaStream_t>(stream), gpu_index,
      static_cast<uint32_t *>(lwe_array_out),
      static_cast<const uint32_t *>(lwe_output_indexes),
      static_cast<const uint32_t *>(lut_vector),
      static_cast<const uint32_t *>(lut_vector_indexes),
      static_cast<const uint32_t *>(lwe_array_in),
      static_cast<const uint32_t *>(lwe_input_indexes), bootstrapping_key,
      lwe_dimension, glwe_dimension, polynomial_size, base_log, level_count, 1,
      num_samples, num_many_lut ? num_many_lut : 1, lut_stride, s->centered_ms);
}

// ===========================================================================
// multi-bit PBS
// ===========================================================================
bool has_support_to_cuda_programmable_bootstrap_cg_multi_bit(
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t level_count,
    uint32_t num_samples, uint32_t max_shared_memory) {
  // The engine has a single multi-bit variant (persistent, bundle fused into
  // the Fourier MAC); the cooperative-groups variant does not exist here.
  (void)glwe_dimension;
  (void)polynomial_size;
  (void)level_count;
  (void)num_samples;
  (void)max_shared_memory;
  return false;
}

void cuda_convert_lwe_multi_bit_programmable_bootstrap_key_64_async(
    void *stream, uint32_t gpu_index, void *dest, void const *src,
    uint32_t input_lwe_dim, uint32_t glwe_dim, uint32_t level_count,
    uint32_t polynomial_size, uint32_t grouping_factor) {
  set_device(gpu_index);
  B200_PANIC_IF_FALSE(grouping_factor >= 1 && grouping_factor <= 4 &&
                          input_lwe_dim % grouping_factor == 0,
                      "Cuda error (multi-bit PBS): unsupported grouping factor");
  const uint32_t num_ggsw = (input_lwe_dim / grouping_factor)
                            << grouping_factor;
  const bool mb_fast = grouping_factor >= 2 &&
                       uses_multibit_fast_path(glwe_dim, polynomial_size,
                                               level_count, grouping_factor);
  convert_bsk(static_cast<cudaStream_t>(stream), gpu_index, dest, src,
              input_lwe_dim, glwe_dim, polynomial_size, level_count, num_ggsw,
              mb_fast, mb_fast ? grouping_factor : 0);
}

void b200_convert_seeded_lwe_programmable_bootstrap_key_64_async(
    void *stream, uint32_t gpu_index, void *dest, void const *seeded_bodies,
    const uint8_t *aes_key, uint64_t counter_lo, uint64_t counter_hi,
    uint32_t first_byte_index, uint32_t input_lwe_dim, uint32_t glwe_dim,
    uint32_t level_count, uint32_t polynomial_size, uint32_t grouping_factor) {
  set_device(gpu_index);
  B200_PANIC_IF_FALSE(grouping_factor <= 4 &&
                          (grouping_factor <= 1 ||
                           input_lwe_dim % grouping_factor == 0),
                      "Cuda error (seeded key): unsupported grouping factor");
  if (grouping_factor <= 1) {
    convert_seeded_bsk(static_cast<cudaStream_t>(stream), gpu_index, dest,
                       seeded_bodies, aes_key, counter_lo, counter_hi,
                       first_byte_index, glwe_dim, polynomial_size, level_count,
                       input_lwe_dim,
                       uses_fast_path(input_lwe_dim, glwe_dim, polynomial_size,
                                      level_count),
                       0);
    return;
  }
  const uint32_t num_ggsw = (input_lwe_dim / grouping_factor)
                            << grouping_factor;
  const bool mb_fast = uses_multibit_fast_path(glwe_dim, polynomial_size,
                                               level_count, grouping_factor);
  convert_seeded_bsk(static_cast<cudaStream_t>(stream), gpu_index, dest,
                     seeded_bodies, aes_key, counter_lo, counter_hi,
                     first_byte_index, glwe_dim, polynomial_size, level_count,
                     num_ggsw, mb_fast, mb_fast ? grouping_factor : 0);
}

uint64_t scratch_cuda_multi_bit_programmable_bootstrap_64_async(
    void *stream, uint32_t gpu_index, int8_t **pbs_buffer,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t level_count,
    uint32_t input_lwe_ciphertext_count, bool allocate_gpu_memory) {
  (void)stream;
  set_device(gpu_index);
  check_polynomial_size(polynomial_size);
  PbsScratch *s = new PbsScratch;
  s->magic = SCRATCH_MAGIC;
  s->type = MULTI_BIT;
  s->glwe_dim = glwe_dimension;
  s->poly_size = polynomial_size;
  s->level_count = level_count;
  s->max_samples = input_lwe_ciphertext_count;
  s->centered_ms = 0;
  s->gpu_memory_allocated = allocate_gpu_memory;
  device_tables(gpu_index, ilog2_exact(polynomial_size) - 1);
  *pbs_buffer = reinterpret_cast<int8_t *>(s);
  return 0;
}

void cuda_multi_bit_programmable_bootstrap_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lut_vector,
    void const *lut_vector_indexes, void const *lwe_array_in,
    void const *lwe_input_indexes, void const *bootstrapping_key,
    int8_t *buffer, uint32_t lwe_dimension, uint32_t glwe_dimension,
    uint32_t polynomial_size, uint32_t grouping_factor, uint32_t base_log,
    uint32_t level_count, uint32_t num_samples, uint32_t num_many_lut,
    uint32_t lut_stride) {
  set_device(gpu_index);
  const PbsScratch *s = reinterpret_cast<const PbsScratch *>(buffer);
  B200_PANIC_IF_FALSE(s && s->magic == SCRATCH_MAGIC && s->type == MULTI_BIT,
                      "Cuda error (multi-bit PBS): invalid scratch buffer");
  B200_PANIC_IF_FALSE(base_log <= 64,
                      "Cuda error (multi-bit PBS): base log should be <= 64");
  B200_PANIC_IF_FALSE(grouping_factor >= 2,
                      "Cuda error (multi-bit PBS): grouping factor must be >= 2");
  launch_pbs(static_cast<cudaStream_t>(stream), gpu_index,
             static_cast<uint64_t *>(lwe_array_out),
             static_cast<const uint64_t *>(lwe_output_indexes),
             static_cast<const uint64_t *>(lut_vector),
             static_cast<const uint64_t *>(lut_vector_indexes),
             static_cast<const uint64_t *>(lwe_array_in),
             static_cast<const uint64_t *>(lwe_input_indexes),
             bootstrapping_key, lwe_dimension, glwe_dimension, polynomial_size,
             base_log, level_count, grouping_factor, num_samples, num_many_lut,
             lut_stride, 0);
}

void cleanup_cuda_multi_bit_programmable_bootstrap_64(void *stream,
                                                      uint32_t gpu_index,
                                                      int8_t **pbs_buffer) {
  cleanup_cuda_programmable_bootstrap_64(stream, gpu_index, pbs_buffer);
}

// ===========================================================================
// keyswitch
// ===========================================================================
#pragma GCC visibility push(hidden)
// 0 = automatic, 1 = int8 tensor cores, 2 = fp64 pipe, 3 = integer pipe
static std::atomic<int> &keyswitch_path() {
  static std::atomic<int> sel([] {
    const char *e = std::getenv("B200_KS_PATH");
    const std::string v = e ? e : "";
    if (std::getenv("B200_KS_INTEGER") || v == "int")
      return 3;
    return v == "imma" ? 1 : v == "f64" ? 2 : 0;
  }());
  return sel;
}
#pragma GCC visibility pop
void b200_set_keyswitch_path(int path) { keyswitch_path().store(path); }
void b200_set_pbs_variant(int variant) {
  B200_PANIC_IF_FALSE(is_pbs_variant(variant), "b200_set_pbs_variant(%d): no such kernel", variant);
  fast_variant_sel().store(variant);
}
void b200_set_n512_mode(int mode) { n512_mode_sel().store(mode); }
void b200_set_register_kernels(int mask) { register_kernel_mask().store(mask); }
void b200_set_multibit_tie_rule(int reference_exact) {
  multibit_ties_even().store(reference_exact ? 0 : 1);
}
void b200_set_multibit_ll_max(int max_samples) {
  multibit_ll_override().store(max_samples);
}
void cuda_keyswitch_lwe_ciphertext_vector_64_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lwe_array_in,
    void const *lwe_input_indexes, void const *ksk, uint32_t lwe_dimension_in,
    uint32_t lwe_dimension_out, uint32_t base_log, uint32_t level_count,
    uint32_t num_samples) {
  set_device(gpu_index);
  if (num_samples == 0)
    return;
  B200_PANIC_IF_FALSE(level_count >= 1 && level_count <= 32 && base_log >= 1 &&
                          base_log * level_count <= 63,
                      "Cuda error (keyswitch): unsupported decomposition "
                      "(base_log %u, level_count %u)", base_log, level_count);
  // b200_set_keyswitch_path / B200_KS_PATH pin one kernel (tests, A/B timing)
  const int ks_sel = keyswitch_path().load();
  const std::string ks_path =
      ks_sel == 1 ? "imma" : ks_sel == 2 ? "f64" : ks_sel == 3 ? "int" : "";
  const bool force_int = ks_sel == 3;
  const uint64_t terms = (uint64_t)lwe_dimension_in * level_count;
  // int8 tensor-core variant: digits must fit s8 and the s32 accumulators
  // must hold terms * 255 * B/2 (see keyswitch_imma.cuh)
  const bool imma_exact =
      base_log <= 7 && terms * 255ull * (1ull << (base_log - 1)) < (1ull << 31);
  if (!force_int && imma_exact && (ks_path.empty() || ks_path == "imma")) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    static std::once_flag ki_once[MAX_GPUS];
    std::call_once(ki_once[gpu_index], [] {
      B200_CHECK(cudaFuncSetAttribute(
          keyswitch_imma_kernel<1>,
          cudaFuncAttributeMaxDynamicSharedMemorySize, KiCfg<1>::SMEM));
      B200_CHECK(cudaFuncSetAttribute(
          keyswitch_imma_kernel<2>,
          cudaFuncAttributeMaxDynamicSharedMemorySize, KiCfg<2>::SMEM));
    });
    static const bool wide = std::getenv("B200_KS_IMMA_NB2") != nullptr;
    const uint32_t rows_pad = (num_samples + KI_BM - 1) / KI_BM * KI_BM;
    const uint32_t k_pad = (uint32_t)((terms + KI_BK - 1) / KI_BK * KI_BK);
    int8_t *digits = nullptr;
    // the digit matrix is a stream-ordered allocation per call from the
    // engine's private pool (see workspace_pool)
    B200_CHECK(cudaMallocFromPoolAsync(&digits, (size_t)rows_pad * k_pad,
                                       workspace_pool(gpu_index), st));
    B200_CHECK(cudaMemsetAsync(digits, 0, (size_t)rows_pad * k_pad, st));
    ks_digits_kernel<<<dim3(num_samples, (lwe_dimension_in + 255) / 256), 256,
                       0, st>>>(
        digits, static_cast<const uint64_t *>(lwe_array_in),
        static_cast<const uint64_t *>(lwe_input_indexes), lwe_dimension_in,
        base_log, level_count, k_pad);
    B200_CHECK(cudaGetLastError());
    count_launch();
    const uint32_t n_bytes = (lwe_dimension_out + 1) * 8;
    auto launch = [&](auto kernel, int bn, int smem) {
      kernel<<<dim3(rows_pad / KI_BM, (n_bytes + bn - 1) / bn), KI_THREADS,
               smem, st>>>(
          static_cast<uint64_t *>(lwe_array_out),
          static_cast<const uint64_t *>(lwe_output_indexes),
          static_cast<const uint64_t *>(lwe_array_in),
          static_cast<const uint64_t *>(lwe_input_indexes),
          static_cast<const uint8_t *>(ksk), digits, lwe_dimension_in,
          lwe_dimension_out, level_count, k_pad, num_samples);
    };
    if (wide)
      launch(keyswitch_imma_kernel<2>, KiCfg<2>::BN, KiCfg<2>::SMEM);
    else
      launch(keyswitch_imma_kernel<1>, KiCfg<1>::BN, KiCfg<1>::SMEM);
    B200_CHECK(cudaGetLastError());
    count_launch();
    B200_CHECK(cudaFreeAsync(digits, st));
    return;
  }
  dim3 grid((num_samples + KS_TS - 1) / KS_TS,
            (lwe_dimension_out + 1 + KS_TO - 1) / KS_TO);
  // exactness condition of the fp64-pipe variant (see keyswitch.cuh)
  uint32_t terms_log2 = 0;
  while ((1ull << terms_log2) < terms)
    terms_log2++;
  if (!force_int && ks_path != "imma" && (base_log - 1) + 32 + terms_log2 <= 52) {
    static std::once_flag ks_once[MAX_GPUS];
    std::call_once(ks_once[gpu_index], [] {
      B200_CHECK(cudaFuncSetAttribute(
          keyswitch_f64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
          (int)sizeof(KsfSmem)));
    });
    keyswitch_f64_kernel<<<grid, 256, sizeof(KsfSmem),
                           static_cast<cudaStream_t>(stream)>>>(
        static_cast<uint64_t *>(lwe_array_out),
        static_cast<const uint64_t *>(lwe_output_indexes),
        static_cast<const uint64_t *>(lwe_array_in),
        static_cast<const uint64_t *>(lwe_input_indexes),
        static_cast<const uint64_t *>(ksk), lwe_dimension_in,
        lwe_dimension_out, base_log, level_count, num_samples);
    B200_CHECK(cudaGetLastError());
    count_launch();
    return;
  }
  keyswitch_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<uint64_t *>(lwe_array_out),
      static_cast<const uint64_t *>(lwe_output_indexes),
      static_cast<const uint64_t *>(lwe_array_in),
      static_cast<const uint64_t *>(lwe_input_indexes),
      static_cast<const uint64_t *>(ksk), lwe_dimension_in, lwe_dimension_out,
      base_log, level_count, num_samples);
  B200_CHECK(cudaGetLastError());
  count_launch();
}

void cuda_keyswitch_gemm_64_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lwe_array_in,
    void const *lwe_input_indexes, void const *ksk, uint32_t lwe_dimension_in,
    uint32_t lwe_dimension_out, uint32_t base_log, uint32_t level_count,
    uint32_t num_samples, bool uses_trivial_indexes) {
  // uses_trivial_indexes = true is the caller's promise that both index
  // arrays are 0..num_samples-1; like the reference (crypto/keyswitch.cuh:456,
  // 508: the `false` template instances never read them) the arrays are then
  // not dereferenced at all.
  cuda_keyswitch_lwe_ciphertext_vector_64_64_async(
      stream, gpu_index, lwe_array_out,
      uses_trivial_indexes ? nullptr : lwe_output_indexes, lwe_array_in,
      uses_trivial_indexes ? nullptr : lwe_input_indexes, ksk,
      lwe_dimension_in, lwe_dimension_out, base_log, level_count, num_samples);
}

void cuda_keyswitch_lwe_ciphertext_vector_64_32_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lwe_array_in,
    void const *lwe_input_indexes, void const *ksk, uint32_t lwe_dimension_in,
    uint32_t lwe_dimension_out, uint32_t base_log, uint32_t level_count,
    uint32_t num_samples) {
  set_device(gpu_index);
  if (num_samples == 0)
    return;
  B200_PANIC_IF_FALSE(level_count >= 1 && level_count <= 32 && base_log >= 1 &&
                          base_log * level_count <= 32,
                      "Cuda error (keyswitch 64->32): base_log * level_count "
                      "must not exceed the 32-bit output scalar (base_log %u, "
                      "level_count %u)", base_log, level_count);
  dim3 grid((num_samples + KS_TS - 1) / KS_TS,
            (lwe_dimension_out + 1 + KS_TO - 1) / KS_TO);
  keyswitch_64_32_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<uint32_t *>(lwe_array_out),
      static_cast<const uint64_t *>(lwe_output_indexes),
      static_cast<const uint64_t *>(lwe_array_in),
      static_cast<const uint64_t *>(lwe_input_indexes),
      static_cast<const uint32_t *>(ksk), lwe_dimension_in, lwe_dimension_out,
      base_log, level_count, num_samples);
  B200_CHECK(cudaGetLastError());
  count_launch();
}

void cuda_keyswitch_gemm_64_32_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lwe_array_in,
    void const *lwe_input_indexes, void const *ksk, uint32_t lwe_dimension_in,
    uint32_t lwe_dimension_out, uint32_t base_log, uint32_t level_count,
    uint32_t num_samples, bool uses_trivial_indexes) {
  cuda_keyswitch_lwe_ciphertext_vector_64_32_async(
      stream, gpu_index, lwe_array_out,
      uses_trivial_indexes ? nullptr : lwe_output_indexes, lwe_array_in,
      uses_trivial_indexes ? nullptr : lwe_input_indexes, ksk,
      lwe_dimension_in, lwe_dimension_out, base_log, level_count, num_samples);
}

// ===========================================================================
// stand-alone integer stages (ciphertext.h:15-32)
// ===========================================================================
void cuda_glwe_sample_extract_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *glwe_array_in, uint32_t const *nth_array, uint32_t num_nths,
    uint32_t num_lwes_to_extract_per_glwe, uint32_t num_lwes_stored_per_glwe,
    uint32_t glwe_dimension, uint32_t polynomial_size) {
  set_device(gpu_index);
  if (num_nths == 0)
    return;
  check_polynomial_size(polynomial_size);
  B200_PANIC_IF_FALSE(num_lwes_to_extract_per_glwe >= 1 &&
                          num_lwes_stored_per_glwe >= 1 &&
                          num_lwes_stored_per_glwe <= polynomial_size,
                      "Cuda error (sample extract): invalid extraction counts");
  glwe_sample_extract_kernel<<<num_nths, 256, 0,
                               static_cast<cudaStream_t>(stream)>>>(
      static_cast<uint64_t *>(lwe_array_out),
      static_cast<const uint64_t *>(glwe_array_in), nth_array,
      num_lwes_to_extract_per_glwe, num_lwes_stored_per_glwe, glwe_dimension,
      polynomial_size);
  B200_CHECK(cudaGetLastError());
  count_launch();
}

void cuda_modulus_switch_64_async(void *stream, uint32_t gpu_index,
                                  void *lwe_out, const void *lwe_in,
                                  uint32_t size, uint32_t log_modulus) {
  set_device(gpu_index);
  if (size == 0)
    return;
  B200_PANIC_IF_FALSE(log_modulus >= 1 && log_modulus <= 63,
                      "Cuda error (modulus switch): log_modulus %u out of range",
                      log_modulus);
  modulus_switch_kernel<<<(size + 255) / 256, 256, 0,
                          static_cast<cudaStream_t>(stream)>>>(
      static_cast<uint64_t *>(lwe_out), static_cast<const uint64_t *>(lwe_in),
      size, log_modulus);
  B200_CHECK(cudaGetLastError());
  count_launch();
}

void cuda_modulus_switch_inplace_64_async(void *stream, uint32_t gpu_index,
                                          void *lwe_array_out, uint32_t size,
                                          uint32_t log_modulus) {
  cuda_modulus_switch_64_async(stream, gpu_index, lwe_array_out, lwe_array_out,
                               size, log_modulus);
}

void cuda_centered_modulus_switch_64_async(void *stream, uint32_t gpu_index,
                                           void *lwe_out, const void *lwe_in,
                                           uint32_t lwe_dimension,
                                           uint32_t log_modulus) {
  set_device(gpu_index);
  B200_PANIC_IF_FALSE(log_modulus >= 1 && log_modulus <= 63,
                      "Cuda error (modulus switch): log_modulus %u out of range",
                      log_modulus);
  centered_modulus_switch_kernel<<<1, 256, 0,
                                   static_cast<cudaStream_t>(stream)>>>(
      static_cast<uint64_t *>(lwe_out), static_cast<const uint64_t *>(lwe_in),
      lwe_dimension, log_modulus);
  B200_CHECK(cudaGetLastError());
  count_launch();
}

// ===========================================================================
// additions
// ===========================================================================
void b200_forward_negacyclic_fft_async(void *stream, uint32_t gpu_index,
                                       void const *input, void *output,
                                       uint32_t polynomial_size,
                                       uint32_t total_polynomials) {
  set_device(gpu_index);
  B200_PANIC_IF_FALSE(polynomial_size == 2048,
                      "b200_forward_negacyclic_fft_async: N must be 2048");
  const DeviceTables &t = device_tables(gpu_index, 0);
  forward_fft_natural_kernel<<<total_polynomials, 64, 0,
                               static_cast<cudaStream_t>(stream)>>>(
      static_cast<cplx *>(output), static_cast<const cplx *>(input),
      t.fft1024);
  B200_CHECK(cudaGetLastError());
  count_launch();
}

void b200_oprf_expand_seeded_lwe_64_async(
    void *stream, uint32_t gpu_index, void *lwe_out, const uint8_t *aes_key,
    uint64_t counter_lo, uint64_t counter_hi, uint32_t first_byte_index,
    uint32_t lwe_dimension, uint32_t num_blocks, uint32_t log_modulus) {
  set_device(gpu_index);
  oprf_expand(static_cast<cudaStream_t>(stream), gpu_index,
              static_cast<uint64_t *>(lwe_out), aes_key, counter_lo, counter_hi,
              first_byte_index, lwe_dimension, num_blocks, log_modulus);
}

void b200_grouped_oprf_64_async(
    void *stream, uint32_t gpu_index, void *lwe_out, const uint8_t *aes_key,
    uint64_t counter_lo, uint64_t counter_hi, void const *lut_vector,
    void const *lut_indexes, void const *corrections,
    void const *bootstrapping_key, int8_t *buffer, uint32_t lwe_dimension,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t base_log,
    uint32_t level_count, uint32_t grouping_factor, uint32_t num_blocks) {
  set_device(gpu_index);
  check_polynomial_size(polynomial_size);
  const bool multi_bit = grouping_factor > 1;
  const PbsScratch *s = reinterpret_cast<const PbsScratch *>(buffer);
  B200_PANIC_IF_FALSE(s && s->magic == SCRATCH_MAGIC &&
                          s->type == (multi_bit ? MULTI_BIT : CLASSICAL),
                      "Cuda error (OPRF): invalid scratch buffer");
  B200_PANIC_IF_FALSE(
      s->glwe_dim == glwe_dimension && s->poly_size == polynomial_size &&
          s->level_count == level_count,
      "Cuda error (OPRF): scratch buffer was created for other parameters");
  if (num_blocks == 0)
    return;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint64_t in_words = (uint64_t)num_blocks * (lwe_dimension + 1);
  uint64_t *ws = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(
      &ws, (in_words + num_blocks) * sizeof(uint64_t),
      workspace_pool(gpu_index), st));
  uint64_t *idx = ws + in_words;
  oprf_iota_kernel<<<(num_blocks + 255) / 256, 256, 0, st>>>(idx, num_blocks);
  B200_CHECK(cudaGetLastError());
  count_launch();
  oprf_expand(st, gpu_index, ws, aes_key, counter_lo, counter_hi, 0,
              lwe_dimension, num_blocks, ilog2_exact(polynomial_size) + 1);
  // centered_ms = 0 whatever the scratch object says: the switched values
  // are exact and must not be corrected again
  launch_pbs(st, gpu_index, static_cast<uint64_t *>(lwe_out), idx,
             static_cast<const uint64_t *>(lut_vector),
             static_cast<const uint64_t *>(lut_indexes), ws, idx,
             bootstrapping_key, lwe_dimension, glwe_dimension, polynomial_size,
             base_log, level_count, multi_bit ? grouping_factor : 1, num_blocks,
             1, 0, 0);
  const uint64_t big_n = (uint64_t)glwe_dimension * polynomial_size;
  oprf_add_corrections_kernel<<<(num_blocks + 255) / 256, 256, 0, st>>>(
      static_cast<uint64_t *>(lwe_out),
      static_cast<const uint64_t *>(corrections), big_n, num_blocks);
  B200_CHECK(cudaGetLastError());
  count_launch();
  B200_CHECK(cudaFreeAsync(ws, st));
}

void b200_expand_lwe_compact_ciphertext_lists_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_flattened_compact_array_in,
    const uint32_t *num_lwes_per_compact_list, uint32_t num_compact_lists,
    uint32_t lwe_dimension) {
  set_device(gpu_index);
  compact_expand(static_cast<cudaStream_t>(stream), gpu_index,
                 static_cast<uint64_t *>(lwe_array_out),
                 static_cast<const uint64_t *>(lwe_flattened_compact_array_in),
                 num_lwes_per_compact_list, num_compact_lists, lwe_dimension);
}

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
    uint32_t pbs_base_log, uint32_t pbs_level_count, uint32_t grouping_factor) {
  set_device(gpu_index);
  check_polynomial_size(polynomial_size);
  const bool multi_bit = grouping_factor > 1;
  const PbsScratch *s = reinterpret_cast<const PbsScratch *>(buffer);
  B200_PANIC_IF_FALSE(s && s->magic == SCRATCH_MAGIC &&
                          s->type == (multi_bit ? MULTI_BIT : CLASSICAL),
                      "Cuda error (expand): invalid scratch buffer");
  B200_PANIC_IF_FALSE(
      s->glwe_dim == glwe_dimension && s->poly_size == polynomial_size &&
          s->level_count == pbs_level_count,
      "Cuda error (expand): scratch buffer was created for other parameters");
  B200_PANIC_IF_FALSE(casting_ksk && (!casting_to_big || computing_ksk),
                      "Cuda error (expand): missing keyswitching key");
  const uint64_t T = compact_lists_total(num_lwes_per_compact_list,
                                         num_compact_lists,
                                         compact_lwe_dimension);
  B200_PANIC_IF_FALSE(2 * T <= s->max_samples,
                      "Cuda error (expand): scratch buffer made for %u "
                      "samples, the call unpacks %llu", s->max_samples,
                      (unsigned long long)(2 * T));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint64_t big_n = (uint64_t)glwe_dimension * polynomial_size;
  const uint64_t exp_words = T * (compact_lwe_dimension + 1);
  const uint64_t big_words = casting_to_big ? T * (big_n + 1) : 0;
  const uint64_t small_words = T * (lwe_dimension + 1);
  uint64_t *ws = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(
      &ws, (exp_words + big_words + small_words + 4 * T) * sizeof(uint64_t),
      workspace_pool(gpu_index), st));
  uint64_t *expanded = ws, *big = ws + exp_words;
  uint64_t *small = big + big_words;
  uint64_t *in_idx = small + small_words, *out_idx = in_idx + 2 * T;
  compact_expand(st, gpu_index, expanded,
                 static_cast<const uint64_t *>(lwe_flattened_compact_array_in),
                 num_lwes_per_compact_list, num_compact_lists,
                 compact_lwe_dimension);
  // null index arrays: trivial indexes (cuda_keyswitch_gemm_64_64_async)
  if (casting_to_big) {
    cuda_keyswitch_lwe_ciphertext_vector_64_64_async(
        stream, gpu_index, big, nullptr, expanded, nullptr, casting_ksk,
        compact_lwe_dimension, (uint32_t)big_n, casting_base_log,
        casting_level_count, (uint32_t)T);
    cuda_keyswitch_lwe_ciphertext_vector_64_64_async(
        stream, gpu_index, small, nullptr, big, nullptr, computing_ksk,
        (uint32_t)big_n, lwe_dimension, computing_base_log,
        computing_level_count, (uint32_t)T);
  } else {
    cuda_keyswitch_lwe_ciphertext_vector_64_64_async(
        stream, gpu_index, small, nullptr, expanded, nullptr, casting_ksk,
        compact_lwe_dimension, lwe_dimension, casting_base_log,
        casting_level_count, (uint32_t)T);
  }
  const uint32_t samples = (uint32_t)(2 * T);
  compact_unpack_index_kernel<<<(samples + 255) / 256, 256, 0, st>>>(
      in_idx, out_idx, samples);
  B200_CHECK(cudaGetLastError());
  count_launch();
  launch_pbs(st, gpu_index, static_cast<uint64_t *>(lwe_array_out), out_idx,
             static_cast<const uint64_t *>(lut_vector),
             static_cast<const uint64_t *>(lut_indexes), small, in_idx,
             bootstrapping_key, lwe_dimension, glwe_dimension, polynomial_size,
             pbs_base_log, pbs_level_count, multi_bit ? grouping_factor : 1,
             samples, 1, 0, s->centered_ms);
  B200_CHECK(cudaFreeAsync(ws, st));
}

uint64_t b200_kernel_launch_count(void) {
  return g_launches.load(std::memory_order_relaxed);
}

const char *b200_last_pbs_kernel(void) { return t_last_pbs_kernel; }

int b200_pbs_uses_fast_path(uint32_t lwe_dimension, uint32_t glwe_dimension,
                            uint32_t polynomial_size, uint32_t level_count) {
  return uses_fast_path(lwe_dimension, glwe_dimension, polynomial_size,
                        level_count);
}

const char *b200_version(void) { return "tfhe-rs_b200 0.1 (sm_90a)"; }

} // extern "C"
#pragma GCC visibility pop
