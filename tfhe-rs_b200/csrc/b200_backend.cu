// b200_backend.cu -- the single translation unit of
// libtfhe_cuda_backend_b200.so: device helpers, per-device tables and the
// extern "C" entry points declared in include/tfhe_b200.h (same names and
// signatures as tfhe-rs' backends/tfhe-cuda-backend C ABI), and those of
// include/tfhe_b200_zk.h (backends/zk-cuda-backend's C ABI).
//
// There is NO CPU fallback anywhere in this file: every compute entry point
// launches sm_90a kernels or aborts.  The zk ABI's point and field helpers
// are host functions by definition (the reference's are too); its MSMs run on
// the GPU apart from the final combination of window sums (DESIGN §8k).
#include "../../include/tfhe_b200.h"

#include <algorithm>
#include <atomic>
#include <cstring>
#include <mutex>
#include <optional>
#include <set>
#include <string>
#include <type_traits>
#include <utility>
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
#include "rerand.cuh"
#include "compression.cuh"
#include "ciphertext_ops.cuh"
#include "pbs128.cuh"
#include "pbs128_multibit.cuh"
#include "keyswitch128.cuh"
#include "bit_circuit.cuh"
#include "msm.cuh"
#include <chrono>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace b200 {

static std::atomic<uint64_t> g_launches{0};

// kernel<<<grid, block, smem, stream>>> on device `gpu`, and where the launch is
// made from (for the message of a failed launch).  An instance launched with
// dynamic shared memory has its limit raised to `smem_max`, once per (instance,
// device): the most that instance is ever launched with.  It defaults to `smem`
// (instances of a fixed size); callers whose size varies pass their bound, so
// the value never depends on which host thread launched first.
struct LaunchCfg {
  dim3 grid, block;
  size_t smem;
  cudaStream_t stream;
  uint32_t gpu;
  size_t smem_max;
  const char *file;
  int line;
  LaunchCfg(dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
            uint32_t gpu, size_t smem_max = 0,
            const char *file = __builtin_FILE(), int line = __builtin_LINE())
      : grid(grid), block(block), smem(smem), stream(stream), gpu(gpu),
        smem_max(smem_max ? smem_max : smem), file(file), line(line) {}
};

static void check_launch(cudaError_t code, const LaunchCfg &c) {
  if (code != cudaSuccess) {
    std::fprintf(stderr, "Cuda error: %s %s %d\n", cudaGetErrorString(code),
                 c.file, c.line);
    std::abort();
  }
}

static void raise_smem_limit(const void *kernel, const LaunchCfg &c) {
  static std::mutex mutex;
  static std::set<std::pair<const void *, uint32_t>> raised;
  std::lock_guard<std::mutex> lock(mutex);
  if (raised.emplace(kernel, c.gpu).second)
    check_launch(cudaFuncSetAttribute(kernel,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)c.smem_max),
                 c);
}

// every kernel launch of the library: enqueue, check, count
// (b200_kernel_launch_count)
template <typename... Params, typename... Args>
static void launch(void (*kernel)(Params...), const LaunchCfg &c,
                   Args &&...args) {
  if (c.smem)
    raise_smem_limit(reinterpret_cast<const void *>(kernel), c);
  kernel<<<c.grid, c.block, c.smem, c.stream>>>(std::forward<Args>(args)...);
  check_launch(cudaGetLastError(), c);
  g_launches.fetch_add(1, std::memory_order_relaxed);
}

// name of the kernel instance the calling thread's last PBS launch ran
// (b200_last_pbs_kernel): one pointer store per launch
static thread_local const char *t_last_pbs_kernel = "";
// the same for the keyswitch (b200_last_keyswitch_kernel)
static thread_local const char *t_last_ks_kernel = "";

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

// The shape of a PBS: input LWE dimension n, GLWE dimension k, polynomial size
// N, decomposition (base_log, l) and the multi-bit grouping factor, 1 for the
// classic PBS.  Key conversion knows no base_log and leaves it 0.
struct PbsParams {
  uint32_t n, k, N, base_log, l, grouping;
  PBS_TYPE type() const { return grouping > 1 ? MULTI_BIT : CLASSICAL; }
  // GGSWs of the key: one per input coefficient, or 2^g per group of g
  uint32_t num_ggsw() const { return grouping > 1 ? (n / grouping) << grouping : n; }
};

// register-kernel routes switched at run time: bit 0 the N = 512 kernel, bit 1
// the N = 8192 kernel (b200_set_register_kernels; B200_N512_GENERIC=1 /
// B200_N8192_GENERIC=1 clear them, read once per process).  Bits 2 and 3 pick
// debug instances of the N = 8192 kernel (B200_N8192_GEN1,
// B200_N8192_RACECHECK).
static std::atomic<int> &register_kernel_mask() {
  static std::atomic<int> v((std::getenv("B200_N512_GENERIC") ? 0 : 1) | (std::getenv("B200_N8192_GENERIC") ? 0 : 2) |
                            (std::getenv("B200_N8192_GEN1") ? 4 : 0) | (std::getenv("B200_N8192_RACECHECK") ? 8 : 0));
  return v;
}

// The kernel family a 64-bit PBS shape runs on.  The route also fixes the
// Fourier-BSK layout, so key conversion and the PBS both ask pbs_route: a key
// converted under one answer and bootstrapped under another decrypts to
// garbage.  A key must therefore be converted and used under the same
// b200_set_register_kernels setting.
enum class PbsRoute { N2048, N8192, N512, MultiBitN2048, Generic };

static PbsRoute pbs_route(const PbsParams &p) {
  if (p.grouping > 1) {
    // N = 2048, k = 1, l <= 2: the kernels of pbs_multibit_n2048.cuh.
    // B200_MULTIBIT_GENERIC keeps every multi-bit shape on the generic kernel.
    static const bool generic_only = std::getenv("B200_MULTIBIT_GENERIC") != nullptr;
    return !generic_only && p.N == 2048 && p.k == 1 && p.l >= 1 && p.l <= 2 && p.grouping <= 4
               ? PbsRoute::MultiBitN2048
               : PbsRoute::Generic;
  }
  // cf. the reference's supports_specialized_2_2_params
  // (programmable_bootstrap_classic.cuh:198-212)
  if (p.N == 2048 && p.k == 1 && p.l == 1 && p.n <= 1024)
    return PbsRoute::N2048;
  const int mask = register_kernel_mask().load();
  // pbs_n8192.cuh, PARAM_MESSAGE_3_CARRY_3_KS_PBS
  if ((mask & 2) && p.N == 8192 && p.k == 1 && p.l == 2 && p.n <= 2048)
    return PbsRoute::N8192;
  // pbs_n512.cuh, e.g. PARAM_MESSAGE_1_CARRY_1_KS_PBS
  if ((mask & 1) && p.N == 512 && p.l == 1 && p.k >= 1 && p.k <= 4 && p.n <= 1024)
    return PbsRoute::N512;
  return PbsRoute::Generic;
}

// B200_PBS_VARIANT pins a kernel for A/B measurements: 1 first-generation
// kernel (u64 accumulator), 3 the round-1 register kernel, 5 round-1 MAC
// schedule + lean rotate/decompose (the default), 4 all key values in flight
// across the share barrier + lean rotate/decompose.  Read once per process.
// The N = 2048 kernel instances by the variant b200_set_pbs_variant /
// B200_PBS_VARIANT pins (0: the automatic choice of launch_pbs).
struct N2048Instance {
  int variant;
  decltype(&pbs_n2048_k1_l1_kernel) kernel;
  size_t smem;
  const char *name;
};
static const N2048Instance N2048_INSTANCES[] = {
    // v1: 64-bit accumulator (A/B measurements and base_log = 31)
    {1, pbs_n2048_k1_l1_kernel, sizeof(P22Smem), "n2048_v1"},
    {3, pbs_n2048_k1_l1_v3_kernel<0, 0>, sizeof(P22SmemV3), "n2048_v3<0,0>"}, // round 1
    {4, pbs_n2048_k1_l1_v3_kernel<1, 1>, sizeof(P22SmemV3), "n2048_v3<1,1>"},
    {5, pbs_n2048_k1_l1_v3_kernel<0, 1>, sizeof(P22SmemV3), "n2048_v3<0,1>"},
    {6, pbs_n2048_k1_l1_v3_kernel<2, 1>, sizeof(P22SmemV3), "n2048_v3<2,1>"},
    // TMA ring for the key block: 208 KiB of shared memory, one CTA per SM
    {7, pbs_n2048_k1_l1_v3_kernel<3, 1>, sizeof(P22SmemV3Tma), "n2048_v3<3,1>"},
    // exchange 2 through warp shuffles (x2_shfl.cuh)
    {8, pbs_n2048_k1_l1_v3_kernel<0, 1, 1>, sizeof(P22SmemV3), "n2048_v3<0,1,1>"},
    // v6: shuffle exchange 2 + one-slot TMA key ring, 2 CTAs / SM
    {9, pbs_n2048_k1_l1_v6_kernel<0, false>, sizeof(P22SmemV6<4, false>), "n2048_v6<0,false>"},
    // v6 with v3's register key prefetch (isolates the ring)
    {10, pbs_n2048_k1_l1_v6_kernel<1, true>, sizeof(P22SmemV6<1, true>), "n2048_v6<1,true>"},
    // v6 hybrid: own row in registers, other row through the ring
    {11, pbs_n2048_k1_l1_v6_kernel<2, true>, sizeof(P22SmemV6<2, true>), "n2048_v6<2,true>"},
    // v6 with the switched mask staged in shared memory: one CTA per SM
    {14, pbs_n2048_k1_l1_v6_kernel<0, true>, sizeof(P22SmemV6<4, true>), "n2048_v6<0,true>"},
    // v6 ring, digits converted through the fp64 ADD pipe instead of I2F
    {15, pbs_n2048_k1_l1_v6_kernel<0, true, 1>, sizeof(P22SmemV6<4, true>), "n2048_v6<0,true,1>"},
    {16, pbs_n2048_k1_l1_v6_kernel<2, true, 1>, sizeof(P22SmemV6<2, true>), "n2048_v6<2,true,1>"},
    {17, pbs_n2048_k1_l1_v6_kernel<2, true, 2>, sizeof(P22SmemV6<2, true>), "n2048_v6<2,true,2>"},
    {18, pbs_n2048_k1_l1_v6_kernel<2, true, 3>, sizeof(P22SmemV6<2, true>), "n2048_v6<2,true,3>"},
    // the shipped one-CTA instance (see launch_pbs)
    {19, pbs_n2048_k1_l1_v6_kernel<0, true, 2>, sizeof(P22SmemV6<4, true>), "n2048_v6<0,true,2>"},
    // the shipped two-CTA instance (lane-pair layout, exchange 2 through the
    // warp's own rows of the exchange-1 buffer; see launch_pbs)
    {20, pbs_n2048_k1_l1_v6_kernel<2, true, 2, 1>, sizeof(P22SmemV6<2, true>), "n2048_v6<2,true,2,1>"},
    {21, pbs_n2048_k1_l1_v6_kernel<0, true, 2, 1>, sizeof(P22SmemV6<4, true>), "n2048_v6<0,true,2,1>"},
    // v6 hybrid with both CTA barriers of a step split (own-row products before
    // the wait for the other group's spectrum)
    {22, pbs_n2048_k1_l1_v6_kernel<2, true, 2, 2>, sizeof(P22SmemV6<2, true>), "n2048_v6<2,true,2,2>"},
    // the shipped two-CTA instance with exchange 2 through half-warp shuffles
    // (x2_shfl.cuh), its A/B partner
    {23, pbs_n2048_k1_l1_v6_kernel<2, true, 2, 1, 0>, sizeof(P22SmemV6<2, true>), "n2048_v6<2,true,2,1,0>"},
};
static const N2048Instance *n2048_instance(int variant) {
  for (const N2048Instance &r : N2048_INSTANCES)
    if (r.variant == variant)
      return &r;
  return nullptr;
}
static bool is_pbs_variant(int v) { return v == 0 || n2048_instance(v); }
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
  bool torus128 = false; // made by scratch_cuda_programmable_bootstrap_128_async
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

// a new scratch object of `type` for (k, N, l), handed back through `buffer`.
// The persistent kernels keep every intermediate on chip or in per-call
// stream-ordered pool allocations: it holds no device workspace, whatever the
// batch size, and the size returned is 0.
static uint64_t new_pbs_scratch(int8_t **buffer, PBS_TYPE type, uint32_t k,
                                uint32_t N, uint32_t l, uint32_t max_samples,
                                bool allocate_gpu_memory, int centered_ms,
                                bool torus128 = false) {
  PbsScratch *s = new PbsScratch;
  s->magic = SCRATCH_MAGIC;
  s->type = type;
  s->glwe_dim = k;
  s->poly_size = N;
  s->level_count = l;
  s->max_samples = max_samples;
  s->centered_ms = centered_ms;
  s->gpu_memory_allocated = allocate_gpu_memory;
  s->torus128 = torus128;
  *buffer = reinterpret_cast<int8_t *>(s);
  return 0;
}

// the scratch object behind `buffer`, checked to be a live one of `type` and of
// the 128-bit PBS exactly when `torus128`; made for the (k, N, l) of `shape`
// when one is given, and for at least `samples` samples.  `what` names the
// caller in the messages.
static const PbsScratch &pbs_scratch(const int8_t *buffer, PBS_TYPE type,
                                     const char *what,
                                     std::optional<PbsParams> shape = {},
                                     uint64_t samples = 0,
                                     bool torus128 = false) {
  const PbsScratch *s = reinterpret_cast<const PbsScratch *>(buffer);
  B200_PANIC_IF_FALSE(s && s->magic == SCRATCH_MAGIC && s->type == type,
                      "Cuda error (%s): invalid scratch buffer", what);
  B200_PANIC_IF_FALSE(s->torus128 == torus128,
                      "Cuda error (%s): the scratch buffer was made for the "
                      "%s PBS", what, s->torus128 ? "128-bit" : "64-bit");
  B200_PANIC_IF_FALSE(
      !shape || (s->glwe_dim == shape->k && s->poly_size == shape->N &&
                 s->level_count == shape->l),
      "Cuda error (%s): scratch buffer was created for other parameters", what);
  B200_PANIC_IF_FALSE(samples <= s->max_samples,
                      "Cuda error (%s): scratch buffer made for %u samples, "
                      "the call runs %llu", what, s->max_samples,
                      (unsigned long long)samples);
  return *s;
}

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
                               const PbsParams &p, uint32_t num_samples,
                               uint32_t num_many_lut, uint32_t lut_stride) {
  const uint32_t n = p.n, l = p.l, grouping = p.grouping;
  const uint32_t steps = n / grouping;
  const size_t bytes =
      (size_t)num_samples * steps * l * 4 * P22_M * sizeof(cplx);
  cplx *bundle = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(&bundle, bytes, workspace_pool(gpu_index),
                                     stream));
  // [grouping - 2][l - 1]
  static const decltype(&mb_bundle_kernel<2, 1>) bundle_kernels[3][2] = {
      {mb_bundle_kernel<2, 1>, mb_bundle_kernel<2, 2>},
      {mb_bundle_kernel<3, 1>, mb_bundle_kernel<3, 2>},
      {mb_bundle_kernel<4, 1>, mb_bundle_kernel<4, 2>}};
  launch(bundle_kernels[grouping - 2][l - 1],
         {dim3(steps, 2, 4), 256, 0, stream, gpu_index}, bundle, bsk,
         t.gen_root[10], t.mono2048, lwe_in, in_idx, n, num_samples);
  // l = 1: the bundle block of a step comes through the bulk-copy (TMA) ring
  // B200_MULTIBIT_SEQ_TMA=0 selects the register-prefetch variant for A/B runs
  static const bool use_tma = [] {
    const char *e = std::getenv("B200_MULTIBIT_SEQ_TMA");
    return !e || std::atoi(e) != 0;
  }();
  // [l = 1, l = 2 with register prefetch; l = 1 with the TMA ring], named per
  // grouping - 2
  static const struct {
    decltype(&pbs_multibit_seq_kernel<1, false>) kernel;
    size_t smem;
    const char *names[3];
  } seq_kernels[3] = {
      {pbs_multibit_seq_kernel<1, false>, sizeof(MbSeqSmem),
       {"multibit_ll<2,1,regs>", "multibit_ll<3,1,regs>", "multibit_ll<4,1,regs>"}},
      {pbs_multibit_seq_kernel<2, false>, sizeof(MbSeqSmem),
       {"multibit_ll<2,2,regs>", "multibit_ll<3,2,regs>", "multibit_ll<4,2,regs>"}},
      {pbs_multibit_seq_kernel<1, true>, sizeof(MbSeqSmemTma),
       {"multibit_ll<2,1,tma>", "multibit_ll<3,1,tma>", "multibit_ll<4,1,tma>"}}};
  const auto &seq = seq_kernels[l == 1 && use_tma ? 2 : l - 1];
  launch(seq.kernel, {num_samples, 128, seq.smem, stream, gpu_index}, lwe_out,
         out_idx, luts, lut_idx, lwe_in, in_idx, bundle, t.fft1024, n, steps,
         p.base_log, num_many_lut, lut_stride, multibit_ties_even().load());
  t_last_pbs_kernel = seq.names[grouping - 2];
  B200_CHECK(cudaFreeAsync(bundle, stream));
}

// any-(N, k, l) kernel, shared memory or global workspace, 64- or 32-bit torus
template <typename Torus>
static void launch_pbs_generic(cudaStream_t stream, uint32_t gpu_index,
                               Torus *lwe_out, const Torus *out_idx,
                               const Torus *luts, const Torus *lut_idx,
                               const Torus *lwe_in, const Torus *in_idx,
                               const void *bsk, const PbsParams &p,
                               uint32_t num_samples, uint32_t num_many_lut,
                               uint32_t lut_stride, int centered_ms) {
  const uint32_t n = p.n, k = p.k, N = p.N, l = p.l, grouping = p.grouping;
  if (grouping > 1) {
    B200_PANIC_IF_FALSE(grouping <= 4 && n % grouping == 0,
                        "Cuda error (multi-bit PBS): grouping factor must be "
                        "2, 3 or 4 and divide the lwe dimension");
  }
  const uint32_t logM = ilog2_exact(N) - 1;
  const DeviceTables &t = device_tables(gpu_index, logM);
  const size_t smem = generic_smem_bytes(grouping > 1 ? 16 : n, k, N, l);
  // The limit is the device maximum, whatever the call: a value taken from
  // call arguments would race between host threads.
  static int max_dyn[MAX_GPUS];
  static std::once_flag max_dyn_once[MAX_GPUS];
  std::call_once(max_dyn_once[gpu_index], [gpu_index] {
    int max_smem = 0;
    B200_CHECK(cudaDeviceGetAttribute(
        &max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, (int)gpu_index));
    cudaFuncAttributes fattr;
    B200_CHECK(
        cudaFuncGetAttributes(&fattr, pbs_generic_kernel<256, false, Torus>));
    max_dyn[gpu_index] = max_smem - (int)fattr.sharedSizeBytes;
  });
  if (smem > (size_t)max_dyn[gpu_index]) {
    // working set larger than one SM's shared memory (N >= 8192 ...): same
    // kernel over a per-CTA slice of a stream-ordered global workspace, a
    // persistent grid striding over the samples
    const uint32_t grid = std::min(num_samples, 2u * sm_count(gpu_index));
    const size_t stride = (smem + 255) / 256 * 256;
    unsigned char *ws = nullptr;
    B200_CHECK(cudaMallocFromPoolAsync(&ws, stride * grid,
                                       workspace_pool(gpu_index), stream));
    launch(pbs_generic_kernel<256, true, Torus>,
           {grid, 256, 0, stream, gpu_index}, lwe_out, out_idx, luts, lut_idx,
           lwe_in, in_idx, static_cast<const cplx *>(bsk), t.gen_tw[logM],
           t.gen_root[logM], n, k, N, logM, p.base_log, l, grouping,
           num_many_lut, lut_stride, centered_ms, multibit_ties_even().load(),
           num_samples, ws, stride);
    t_last_pbs_kernel = std::is_same<Torus, uint32_t>::value
                            ? "generic_workspace_u32"
                            : "generic_workspace";
    B200_CHECK(cudaFreeAsync(ws, stream));
    return;
  }
  launch(pbs_generic_kernel<256, false, Torus>,
         {num_samples, 256, smem, stream, gpu_index, (size_t)max_dyn[gpu_index]},
         lwe_out, out_idx, luts, lut_idx, lwe_in, in_idx,
         static_cast<const cplx *>(bsk), t.gen_tw[logM], t.gen_root[logM], n,
         k, N, logM, p.base_log, l, grouping, num_many_lut, lut_stride,
         centered_ms, multibit_ties_even().load(), 0, nullptr,
         0); // no workspace
  t_last_pbs_kernel =
      std::is_same<Torus, uint32_t>::value ? "generic_smem_u32" : "generic_smem";
}

// PbsRoute::N2048: N = 2048, k = 1, l = 1 (pbs_n2048.cuh)
static void launch_n2048(cudaStream_t stream, uint32_t gpu_index,
                         uint64_t *lwe_out, const uint64_t *out_idx,
                         const uint64_t *luts, const uint64_t *lut_idx,
                         const uint64_t *lwe_in, const uint64_t *in_idx,
                         const void *bsk, const PbsParams &p,
                         uint32_t num_samples, uint32_t num_many_lut,
                         uint32_t lut_stride, int centered_ms) {
  B200_PANIC_IF_FALSE(p.base_log <= 31, "Cuda error (PBS): base_log > 31");
  const DeviceTables &t = device_tables(gpu_index, 0);
  int variant = fast_variant();
  if (p.base_log > 30) {
    variant = 1; // v1's 64-bit accumulator holds base_log = 31
  } else if (variant == 0 && num_samples <= sm_count(gpu_index)) {
    // shipped, at most one CTA per SM: v6 with the whole key block of a step
    // through the one-slot TMA ring (no key value is ever waited for) and
    // exchange 2 through warp shuffles
    variant = 19; // n2048_v6<0,true,2>
  } else if (variant == 0) {
    // shipped, two CTAs per SM: v6 hybrid -- own key row prefetched into
    // registers, other row (the one v3 waited a full L2 round trip for)
    // through the ring; rotate + decompose with the sign as a predicate
    // (CVT = 2); lane-pair layout: each warp holds the same 16 threads of
    // both polynomials (lanes l and l ^ 16), exchange 2 through the warp's
    // own rows of the exchange-1 buffer (no shuffles, no selects), the other
    // polynomial's spectrum taken with one shuffle in the MAC (no spectrum
    // store, no barrier between the polynomials).  Bit-identical to variant
    // 17, the same instance in the 64-thread group layout, and to variant 23,
    // the same instance with exchange 2 through half-warp shuffles.
    variant = 20; // n2048_v6<2,true,2,1>
  }
  const N2048Instance &r = *n2048_instance(variant);
  launch(r.kernel, {num_samples, 128, r.smem, stream, gpu_index}, lwe_out,
         out_idx, luts, lut_idx, lwe_in, in_idx,
         static_cast<const cplx *>(bsk), t.fft1024, p.n, p.base_log,
         num_many_lut, lut_stride, centered_ms);
  t_last_pbs_kernel = r.name;
}

// PbsRoute::N8192: N = 8192, k = 1, l = 2 (pbs_n8192.cuh)
static void launch_n8192(cudaStream_t stream, uint32_t gpu_index,
                         uint64_t *lwe_out, const uint64_t *out_idx,
                         const uint64_t *luts, const uint64_t *lut_idx,
                         const uint64_t *lwe_in, const uint64_t *in_idx,
                         const void *bsk, const PbsParams &p,
                         uint32_t num_samples, uint32_t num_many_lut,
                         uint32_t lut_stride, int centered_ms) {
  B200_PANIC_IF_FALSE(p.base_log * p.l <= 30,
                      "Cuda error (PBS): base_log * level_count > 30 is not "
                      "supported for N = 8192");
  const DeviceTables &t = device_tables(gpu_index, 0);
  const uint32_t grid = std::min(num_samples, sm_count(gpu_index));
  // per-thread park area of the four spectra of a step (pbs_n8192.cuh)
  cplx *park = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(&park, (size_t)grid * P8K_PARK_PER_CTA * sizeof(cplx),
                                     workspace_pool(gpu_index), stream));
  // mask bit 2: the first-generation kernel (per-thread key loads), for A/B
  if (register_kernel_mask().load() & 4) {
    launch(pbs_n8192_k1_l2_kernel,
           {grid, 256, sizeof(N8192Smem), stream, gpu_index}, lwe_out,
           out_idx, luts, lut_idx, lwe_in, in_idx,
           static_cast<const cplx *>(bsk), t.fft4096, p.n, p.base_log,
           num_samples, num_many_lut, lut_stride, centered_ms,
           multibit_ties_even().load(), park);
    t_last_pbs_kernel = "n8192_v1";
  } else {
    static const uint32_t stagger = [] {
      const char *e = std::getenv("B200_N8192_STAGGER");
      return e ? (uint32_t)std::atoi(e) : 0u;
    }();
    // mask bit 3: the racecheck instance (every thread arrives on the ring's
    // `empty` barriers itself)
    const bool racecheck = register_kernel_mask().load() & 8;
    launch(racecheck ? pbs_n8192_k1_l2_v2_kernel<true>
                     : pbs_n8192_k1_l2_v2_kernel<false>,
           {grid, 256, sizeof(N8192SmemV2), stream, gpu_index}, lwe_out,
           out_idx, luts, lut_idx, lwe_in, in_idx,
           static_cast<const cplx *>(bsk), t.fft4096, p.n, p.base_log,
           num_samples, num_many_lut, lut_stride, centered_ms,
           multibit_ties_even().load(), stagger, park);
    t_last_pbs_kernel = racecheck ? "n8192_v2<true>" : "n8192_v2<false>";
  }
  B200_CHECK(cudaFreeAsync(park, stream));
}

// PbsRoute::N512: N = 512, l = 1, k <= 4 (pbs_n512.cuh)
static void launch_n512(cudaStream_t stream, uint32_t gpu_index,
                        uint64_t *lwe_out, const uint64_t *out_idx,
                        const uint64_t *luts, const uint64_t *lut_idx,
                        const uint64_t *lwe_in, const uint64_t *in_idx,
                        const void *bsk, const PbsParams &p,
                        uint32_t num_samples, uint32_t num_many_lut,
                        uint32_t lut_stride, int centered_ms) {
  B200_PANIC_IF_FALSE(p.base_log <= 31, "Cuda error (PBS): base_log > 31");
  const uint32_t k = p.k;
  const DeviceTables &t = device_tables(gpu_index, 0);
  // B200_N512_MODE: 0 (default) TMA key ring, one CTA per SM, 1 / 2 / 3 LWEs
  // per CTA by launch size; 2 / 3: ring with two / one LWE per CTA; 4: ring with
  // three; 1: register key ring, two LWEs per CTA, two CTAs per SM
  const int mode512 = n512_mode_sel().load();
  // automatic: the fewest LWEs per CTA that still covers the launch in one
  // round of the persistent grid (latency), three per CTA beyond that
  // (throughput)
  const uint32_t sms = sm_count(gpu_index);
  const int per_cta = mode512 == 3 ? 1 : mode512 == 2 ? 2 : mode512 == 0 && num_samples <= sms ? 1
                      : mode512 == 0 && num_samples <= 2 * sms ? 2 : 3;
  // [k - 1][0: register key ring, two LWEs per CTA, two CTAs per SM;
  //         G = 1, 2, 3: TMA key ring, G LWEs per CTA, one CTA per SM]
  static const struct {
    decltype(&pbs_n512_kernel<1, 1, true>) kernel;
    size_t smem;
    const char *name;
  } n512_instances[4][4] = {
      {{pbs_n512_kernel<1, 2, false>, sizeof(N512Smem<1, 2, false>), "n512<1,2,false>"},
       {pbs_n512_kernel<1, 1, true>, sizeof(N512Smem<1, 1, true>), "n512<1,1,true>"},
       {pbs_n512_kernel<1, 2, true>, sizeof(N512Smem<1, 2, true>), "n512<1,2,true>"},
       {pbs_n512_kernel<1, 3, true>, sizeof(N512Smem<1, 3, true>), "n512<1,3,true>"}},
      {{pbs_n512_kernel<2, 2, false>, sizeof(N512Smem<2, 2, false>), "n512<2,2,false>"},
       {pbs_n512_kernel<2, 1, true>, sizeof(N512Smem<2, 1, true>), "n512<2,1,true>"},
       {pbs_n512_kernel<2, 2, true>, sizeof(N512Smem<2, 2, true>), "n512<2,2,true>"},
       {pbs_n512_kernel<2, 3, true>, sizeof(N512Smem<2, 3, true>), "n512<2,3,true>"}},
      {{pbs_n512_kernel<3, 2, false>, sizeof(N512Smem<3, 2, false>), "n512<3,2,false>"},
       {pbs_n512_kernel<3, 1, true>, sizeof(N512Smem<3, 1, true>), "n512<3,1,true>"},
       {pbs_n512_kernel<3, 2, true>, sizeof(N512Smem<3, 2, true>), "n512<3,2,true>"},
       {pbs_n512_kernel<3, 3, true>, sizeof(N512Smem<3, 3, true>), "n512<3,3,true>"}},
      {{pbs_n512_kernel<4, 2, false>, sizeof(N512Smem<4, 2, false>), "n512<4,2,false>"},
       {pbs_n512_kernel<4, 1, true>, sizeof(N512Smem<4, 1, true>), "n512<4,1,true>"},
       {pbs_n512_kernel<4, 2, true>, sizeof(N512Smem<4, 2, true>), "n512<4,2,true>"},
       {pbs_n512_kernel<4, 3, true>, sizeof(N512Smem<4, 3, true>), "n512<4,3,true>"}}};
  const int col = mode512 == 1 ? 0 : per_cta;
  const auto &r = n512_instances[k - 1][col];
  const uint32_t G = col ? col : 2, ctas_per_sm = col ? 1 : 2;
  // persistent grid (see the kernel)
  const uint32_t grid = std::min((num_samples + G - 1) / G, ctas_per_sm * sms);
  launch(r.kernel, {grid, 16 * (k + 1) * G, r.smem, stream, gpu_index},
         lwe_out, out_idx, luts, lut_idx, lwe_in, in_idx,
         static_cast<const cplx *>(bsk), t.fft256, p.n, p.base_log, num_samples,
         num_many_lut, lut_stride, centered_ms);
  t_last_pbs_kernel = r.name;
}

// PbsRoute::MultiBitN2048: N = 2048, k = 1, l <= 2, grouping 2 to 4
// (pbs_multibit_n2048.cuh)
static void launch_multibit_n2048(cudaStream_t stream, uint32_t gpu_index,
                                  uint64_t *lwe_out, const uint64_t *out_idx,
                                  const uint64_t *luts, const uint64_t *lut_idx,
                                  const uint64_t *lwe_in, const uint64_t *in_idx,
                                  const void *bsk, const PbsParams &p,
                                  uint32_t num_samples, uint32_t num_many_lut,
                                  uint32_t lut_stride) {
  B200_PANIC_IF_FALSE(p.n % p.grouping == 0,
                      "Cuda error (multi-bit PBS): grouping factor must "
                      "divide the lwe dimension");
  B200_PANIC_IF_FALSE(p.base_log * p.l <= 31,
                      "Cuda error (multi-bit PBS): base_log * level_count "
                      "> 31 is not supported for N = 2048, k = 1");
  const DeviceTables &t = device_tables(gpu_index, 10);
  // low-latency mode for launches that cannot fill the GPU with the fused
  // kernel: bundle for all groups at once, then the sequential products
  if (num_samples <= multibit_ll_max_samples(gpu_index)) {
    launch_multibit_ll(stream, gpu_index, lwe_out, out_idx, luts, lut_idx,
                       lwe_in, in_idx, static_cast<const cplx *>(bsk), t, p,
                       num_samples, num_many_lut, lut_stride);
    return;
  }
  // [grouping - 2][l - 1]
  static const struct {
    decltype(&pbs_multibit_n2048_k1_kernel<2, 1>) kernel;
    const char *name;
  } fused_instances[3][2] = {
      {{pbs_multibit_n2048_k1_kernel<2, 1>, "multibit_fused<2,1>"},
       {pbs_multibit_n2048_k1_kernel<2, 2>, "multibit_fused<2,2>"}},
      {{pbs_multibit_n2048_k1_kernel<3, 1>, "multibit_fused<3,1>"},
       {pbs_multibit_n2048_k1_kernel<3, 2>, "multibit_fused<3,2>"}},
      {{pbs_multibit_n2048_k1_kernel<4, 1>, "multibit_fused<4,1>"},
       {pbs_multibit_n2048_k1_kernel<4, 2>, "multibit_fused<4,2>"}}};
  const auto &r = fused_instances[p.grouping - 2][p.l - 1];
  launch(r.kernel, {num_samples, 128, sizeof(MbSmem), stream, gpu_index},
         lwe_out, out_idx, luts, lut_idx, lwe_in, in_idx,
         static_cast<const cplx *>(bsk), t.fft1024, t.gen_root[10],
         t.mono2048, p.n, p.base_log, num_many_lut, lut_stride,
         multibit_ties_even().load());
  t_last_pbs_kernel = r.name;
}

// the 64-bit PBS of every entry point: checks shared by every route, then the
// route's own checks and launch
static void launch_pbs(cudaStream_t stream, uint32_t gpu_index,
                       uint64_t *lwe_out, const uint64_t *out_idx,
                       const uint64_t *luts, const uint64_t *lut_idx,
                       const uint64_t *lwe_in, const uint64_t *in_idx,
                       const void *bsk, const PbsParams &p,
                       uint32_t num_samples, uint32_t num_many_lut,
                       uint32_t lut_stride, int centered_ms) {
  if (num_samples == 0)
    return;
  check_polynomial_size(p.N);
  B200_PANIC_IF_FALSE(p.base_log * p.l <= 63 && p.base_log >= 1 && p.l >= 1,
                      "Cuda error (PBS): base_log * level_count must be < 64");
  if (num_many_lut == 0)
    num_many_lut = 1;
  switch (pbs_route(p)) {
  case PbsRoute::N2048:
    return launch_n2048(stream, gpu_index, lwe_out, out_idx, luts, lut_idx,
                        lwe_in, in_idx, bsk, p, num_samples, num_many_lut,
                        lut_stride, centered_ms);
  case PbsRoute::N8192:
    return launch_n8192(stream, gpu_index, lwe_out, out_idx, luts, lut_idx,
                        lwe_in, in_idx, bsk, p, num_samples, num_many_lut,
                        lut_stride, centered_ms);
  case PbsRoute::N512:
    return launch_n512(stream, gpu_index, lwe_out, out_idx, luts, lut_idx,
                       lwe_in, in_idx, bsk, p, num_samples, num_many_lut,
                       lut_stride, centered_ms);
  case PbsRoute::MultiBitN2048:
    return launch_multibit_n2048(stream, gpu_index, lwe_out, out_idx, luts,
                                 lut_idx, lwe_in, in_idx, bsk, p, num_samples,
                                 num_many_lut, lut_stride);
  case PbsRoute::Generic:
    return launch_pbs_generic<uint64_t>(stream, gpu_index, lwe_out, out_idx,
                                        luts, lut_idx, lwe_in, in_idx, bsk, p,
                                        num_samples, num_many_lut, lut_stride,
                                        centered_ms);
  }
}

// standard-domain BSK (device staging buffer) -> Fourier BSK in the layout of
// `route`, the route the key's PBS takes.  The 32-bit torus has the generic
// layout only: its entry points pass PbsRoute::Generic.
template <typename Torus>
static void convert_bsk_staged(cudaStream_t stream, uint32_t gpu_index,
                               void *dest, const Torus *staging,
                               const PbsParams &p, PbsRoute route) {
  const uint32_t k = p.k, N = p.N, l = p.l;
  const uint32_t logM = ilog2_exact(N) - 1;
  const size_t polys = (size_t)p.num_ggsw() * l * (k + 1) * (k + 1);
  const bool register_fft =
      route == PbsRoute::N2048 || route == PbsRoute::MultiBitN2048;
  const DeviceTables &t = device_tables(gpu_index, register_fft ? 0 : logM);
  cplx *out = static_cast<cplx *>(dest);
  // limit: the shared memory of the largest N, 16384
  const auto generic = [&] {
    launch(bsk_convert_generic_kernel<Torus>,
           {(unsigned)polys, 256, (N / 2) * sizeof(cplx), stream, gpu_index,
            (16384 / 2) * sizeof(cplx)},
           out, staging, t.gen_tw[logM], N, logM);
  };
  if constexpr (std::is_same<Torus, uint32_t>::value) {
    generic();
  } else {
    switch (route) {
    case PbsRoute::N2048:
      return launch(bsk_convert_n2048_k1_l1_kernel,
                    {(unsigned)polys, 64, 0, stream, gpu_index}, out, staging,
                    t.fft1024);
    case PbsRoute::N8192:
      return launch(bsk_convert_n8192_kernel,
                    {(unsigned)polys, 256, P8K_M * sizeof(cplx), stream,
                     gpu_index},
                    out, staging, t.fft4096);
    case PbsRoute::N512:
      return launch(bsk_convert_n512_kernel,
                    {(unsigned)((polys + 1) / 2), 32, 0, stream, gpu_index},
                    out, staging, t.fft256, k + 1, (uint32_t)polys);
    case PbsRoute::MultiBitN2048:
      return launch(bsk_convert_multibit_n2048_kernel,
                    {(unsigned)polys, 64, 0, stream, gpu_index}, out, staging,
                    t.fft1024, l, p.grouping);
    case PbsRoute::Generic:
      return generic();
    }
  }
}

// host standard-domain BSK -> device Fourier BSK in the layout of `route`
template <typename Torus>
static void convert_bsk(cudaStream_t stream, uint32_t gpu_index, void *dest,
                        const void *src_host, const PbsParams &p,
                        PbsRoute route) {
  check_polynomial_size(p.N);
  const size_t polys = (size_t)p.num_ggsw() * p.l * (p.k + 1) * (p.k + 1);
  const size_t bytes = polys * p.N * sizeof(Torus);
  Torus *staging = nullptr;
  B200_CHECK(cudaMallocAsync(&staging, bytes, stream));
  B200_CHECK(cudaMemcpyAsync(staging, src_host, bytes, cudaMemcpyHostToDevice,
                             stream));
  convert_bsk_staged<Torus>(stream, gpu_index, dest, staging, p, route);
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
  launch(oprf_expand_kernel,
         {(unsigned)ctas, OPRF_THREADS, 0, stream, gpu_index}, lwe_out, tables,
         key, ctr_lo, ctr_hi, (uint32_t)first_byte, n, num_blocks,
         log_modulus);
}

// seeded BSK (host bodies + AES-CTR mask seed) -> device Fourier BSK
static void convert_seeded_bsk(cudaStream_t stream, uint32_t gpu_index,
                               void *dest, const void *bodies_host,
                               const uint8_t aes_key[16], uint64_t ctr_lo,
                               uint64_t ctr_hi, uint32_t first_byte_index,
                               const PbsParams &p, PbsRoute route) {
  const uint32_t k = p.k, N = p.N;
  check_polynomial_size(N);
  B200_PANIC_IF_FALSE(first_byte_index == 0 || first_byte_index == 8,
                      "Cuda error (seeded key): the mask stream must start on "
                      "a u64 boundary of an AES block (byte index %u)",
                      first_byte_index);
  const AesTables *tables = aes_device_tables(gpu_index);
  AesCtrKey key;
  aes_expand_key(aes_key, aes_host_tables(), key);
  const uint64_t rows = (uint64_t)p.num_ggsw() * p.l * (k + 1);
  const size_t std_bytes = rows * (k + 1) * N * sizeof(uint64_t);
  const size_t body_bytes = rows * N * sizeof(uint64_t);
  uint64_t *staging = nullptr, *bodies = nullptr;
  B200_CHECK(cudaMallocAsync(&staging, std_bytes, stream));
  B200_CHECK(cudaMallocAsync(&bodies, body_bytes, stream));
  B200_CHECK(cudaMemcpyAsync(bodies, bodies_host, body_bytes,
                             cudaMemcpyHostToDevice, stream));
  launch(seeded_bsk_expand_kernel,
         {sm_count(gpu_index) * 8, 256, 0, stream, gpu_index}, staging, bodies,
         tables, key, ctr_lo, ctr_hi, first_byte_index / 8, rows, k, N);
  convert_bsk_staged(stream, gpu_index, dest, staging, p, route);
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
  launch(compact_expand_kernel, {grid, EXPAND_THREADS, 0, st, gpu_index},
         lwe_out, lists_in, d_descs, num_lists, n);
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

// compact encryptions of zero from seeds (rerand.cuh).  The bin descriptors
// and the seeds go to the pool workspace with one stream-ordered copy (staged
// from pageable memory: the host buffers may go when this returns).
static void cpk_encrypt_zeros(cudaStream_t st, uint32_t gpu_index,
                              uint64_t *out, const uint64_t *cpk,
                              const uint8_t *h_seeds, uint32_t num_seeds,
                              const uint64_t *h_entries, uint32_t num_entries,
                              uint32_t n, uint32_t bound_log2,
                              bool accumulate) {
  B200_PANIC_IF_FALSE(n >= 256 && n <= 16384 && (n & (n - 1)) == 0,
                      "Cuda error (rerand): the compact lwe_dimension must be "
                      "a power of two in [256, 16384]. Got %u", n);
  B200_PANIC_IF_FALSE(bound_log2 <= 62,
                      "Cuda error (rerand): noise_bound_log2 %u out of [0, 62]",
                      bound_log2);
  B200_PANIC_IF_FALSE(num_seeds >= 1 && h_seeds && num_entries >= 1 &&
                          h_entries && cpk && out,
                      "Cuda error (rerand): no seed, entry or buffer");
  const uint64_t w = (bound_log2 + 2 + 7) / 8;
  std::vector<RerandBinDesc> descs;
  uint64_t out_offset = 0, max_count = 0;
  for (uint32_t e = 0; e < num_entries; e++) {
    const uint64_t seed = h_entries[3 * e], first = h_entries[3 * e + 1];
    const uint64_t c = h_entries[3 * e + 2];
    B200_PANIC_IF_FALSE(seed < num_seeds,
                        "Cuda error (rerand): entry %u uses seed %llu of %u", e,
                        (unsigned long long)seed, num_seeds);
    B200_PANIC_IF_FALSE(c >= 1 && c < (1ull << 32),
                        "Cuda error (rerand): entry %u encrypts %llu zeros", e,
                        (unsigned long long)c);
    const uint64_t bins = (c + n - 1) / n;
    const uint64_t mask_noise = first + bins * n / 8;
    const uint64_t body_noise = mask_noise + bins * n * w;
    for (uint64_t b = 0; b < bins; b++) {
      const uint32_t cnt = (uint32_t)std::min<uint64_t>(n, c - b * n);
      descs.push_back({out_offset + 2 * b * n, first + b * n / 8,
                       mask_noise + b * n * w, body_noise + b * n * w,
                       (uint32_t)seed, cnt});
      max_count = std::max<uint64_t>(max_count, cnt);
    }
    out_offset += bins * n + c;
  }
  const uint32_t num_bins = (uint32_t)descs.size();
  const size_t state_bytes = (size_t)num_seeds * sizeof(RerandSeedState);
  const size_t desc_bytes = descs.size() * sizeof(RerandBinDesc);
  const size_t seed_bytes = (size_t)num_seeds * XOF_SEED_BYTES;
  std::vector<uint8_t> staging(desc_bytes + seed_bytes);
  std::memcpy(staging.data(), descs.data(), desc_bytes);
  std::memcpy(staging.data() + desc_bytes, h_seeds, seed_bytes);
  uint8_t *ws = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(&ws, state_bytes + staging.size(),
                                     workspace_pool(gpu_index), st));
  RerandSeedState *d_states = reinterpret_cast<RerandSeedState *>(ws);
  RerandBinDesc *d_descs = reinterpret_cast<RerandBinDesc *>(ws + state_bytes);
  const uint8_t *d_seeds = ws + state_bytes + desc_bytes;
  B200_CHECK(cudaMemcpyAsync(ws + state_bytes, staging.data(), staging.size(),
                             cudaMemcpyHostToDevice, st));
  const AesTables *tables = aes_device_tables(gpu_index);
  launch(rerand_seed_init_kernel,
         {(num_seeds + 255) / 256, 256, 0, st, gpu_index}, d_states, d_seeds,
         tables, num_seeds);
  const uint64_t tiles = n / RERAND_THREADS +
                         (max_count + RERAND_THREADS - 1) / RERAND_THREADS;
  const dim3 grid((unsigned)tiles, std::min<uint32_t>(num_bins, 65535u));
  launch(rerand_zeros_kernel,
         {grid, RERAND_THREADS, rerand_smem_bytes(n), st, gpu_index,
          rerand_smem_bytes(16384)},
         out, cpk, d_states, d_descs, tables, num_bins, n, bound_log2,
         accumulate);
  B200_CHECK(cudaFreeAsync(ws, st));
}

// ---- 128-bit PBS (pbs128.cuh) ---------------------------------------------------
// double-double twiddles of the size-2^logM transform, created once per device
static const ddc *dd_twiddles(uint32_t gpu_index, uint32_t logM) {
  static std::mutex mutex;
  static ddc *tables[MAX_GPUS][MAX_LOGM + 1] = {};
  std::lock_guard<std::mutex> lock(mutex);
  ddc *&t = tables[gpu_index][logM];
  if (!t) {
    std::vector<ddc> host((size_t)1 << logM);
    b200_fill_dd_twiddles(logM, host.data());
    set_device(gpu_index);
    B200_CHECK(cudaMalloc(&t, host.size() * sizeof(ddc)));
    B200_CHECK(cudaMemcpy(t, host.data(), host.size() * sizeof(ddc),
                          cudaMemcpyHostToDevice));
  }
  return t;
}

// one instance per polynomial size, [log2(N) - 8]
static const struct Pbs128Instance {
  decltype(&pbs128_kernel<10>) kernel;
  decltype(&bsk_convert_128_kernel<10>) convert;
  const char *name;
} PBS128_INSTANCES[] = {
    {pbs128_kernel<7>, bsk_convert_128_kernel<7>, "pbs128<256>"},
    {pbs128_kernel<8>, bsk_convert_128_kernel<8>, "pbs128<512>"},
    {pbs128_kernel<9>, bsk_convert_128_kernel<9>, "pbs128<1024>"},
    {pbs128_kernel<10>, bsk_convert_128_kernel<10>, "pbs128<2048>"},
    {pbs128_kernel<11>, bsk_convert_128_kernel<11>, "pbs128<4096>"},
};

// the instance for (k, N, l, base_log); aborts on an unsupported shape
static const Pbs128Instance &pbs128_instance(uint32_t k, uint32_t N,
                                             uint32_t l, uint32_t base_log) {
  B200_PANIC_IF_FALSE(
      N >= 256 && N <= 4096 && (N & (N - 1)) == 0,
      "Cuda error (128-bit PBS): unsupported polynomial size. Supported N's "
      "are powers of two in the interval [256..4096]. Got %u", N);
  B200_PANIC_IF_FALSE(k >= 1, "Cuda error (128-bit PBS): glwe_dimension must "
                      "be >= 1");
  B200_PANIC_IF_FALSE(l >= 1 && base_log >= 1 && base_log * l <= 128,
                      "Cuda error (128-bit PBS): unsupported decomposition "
                      "(base_log %u, level_count %u)", base_log, l);
  return PBS128_INSTANCES[ilog2_exact(N) - 8];
}

// largest dynamic shared memory an instance may be launched with on a device
// (the switched mask grows with n): the device opt-in maximum minus the
// instance's static shared memory
static size_t pbs128_smem_max(const Pbs128Instance &r, uint32_t gpu_index) {
  constexpr size_t COUNT = sizeof(PBS128_INSTANCES) / sizeof(PBS128_INSTANCES[0]);
  static std::once_flag once[MAX_GPUS][COUNT];
  static size_t value[MAX_GPUS][COUNT];
  const size_t i = (size_t)(&r - PBS128_INSTANCES);
  std::call_once(once[gpu_index][i], [&] {
    int max_smem = 0;
    B200_CHECK(cudaDeviceGetAttribute(
        &max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, (int)gpu_index));
    cudaFuncAttributes fattr;
    B200_CHECK(cudaFuncGetAttributes(&fattr, r.kernel));
    value[gpu_index][i] = (size_t)max_smem - fattr.sharedSizeBytes;
  });
  return value[gpu_index][i];
}

static void launch_pbs128(cudaStream_t st, uint32_t gpu_index, u128 *lwe_out,
                          const u128 *lut, const uint64_t *lwe_in,
                          const ddc *bsk, uint32_t n, uint32_t k, uint32_t N,
                          uint32_t base_log, uint32_t l, uint32_t num_samples,
                          int centered_ms) {
  const Pbs128Instance &r = pbs128_instance(k, N, l, base_log);
  if (num_samples == 0)
    return;
  const uint32_t logM = ilog2_exact(N) - 1;
  const size_t smem = pbs128_smem_bytes(n, N);
  const size_t smem_max = pbs128_smem_max(r, gpu_index);
  B200_PANIC_IF_FALSE(smem <= smem_max, "Cuda error (128-bit PBS): lwe "
                      "dimension %u is too large", n);
  // one CTA per SM: its workspace slice (accumulator + output spectra, 192 KiB
  // at the squash shape) stays L2 resident
  const uint32_t grid = std::min(num_samples, sm_count(gpu_index));
  const size_t stride = pbs128_ws_bytes(k, N);
  unsigned char *ws = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(&ws, stride * grid,
                                     workspace_pool(gpu_index), st));
  launch(r.kernel, {grid, PBS128_THREADS, smem, st, gpu_index, smem_max},
         lwe_out, lut, lwe_in, bsk, dd_twiddles(gpu_index, logM), n, k,
         base_log, l, num_samples, centered_ms, ws, stride);
  t_last_pbs_kernel = r.name;
  B200_CHECK(cudaFreeAsync(ws, st));
}

// ---- multi-bit 128-bit PBS (pbs128_multibit.cuh) ---------------------------------
// double-double 2N-th roots of unity of the size-2^logM transform (4M entries),
// created once per device
static const ddc *dd_roots(uint32_t gpu_index, uint32_t logM) {
  static std::mutex mutex;
  static ddc *tables[MAX_GPUS][MAX_LOGM + 1] = {};
  std::lock_guard<std::mutex> lock(mutex);
  ddc *&t = tables[gpu_index][logM];
  if (!t) {
    std::vector<ddc> host((size_t)4 << logM);
    b200_fill_dd_roots(logM, host.data());
    set_device(gpu_index);
    B200_CHECK(cudaMalloc(&t, host.size() * sizeof(ddc)));
    B200_CHECK(cudaMemcpy(t, host.data(), host.size() * sizeof(ddc),
                          cudaMemcpyHostToDevice));
  }
  return t;
}

// the instance for (k, N, l, base_log) and a grouping factor g over n mask
// words; aborts on an unsupported shape
static const Pbs128MbInstance &pbs128_mb_instance(uint32_t k, uint32_t N,
                                                  uint32_t l, uint32_t base_log,
                                                  uint32_t grouping) {
  pbs128_instance(k, N, l, base_log); // same (k, N, l) limits as the classic PBS
  B200_PANIC_IF_FALSE(grouping >= 2 && grouping <= 4,
                      "Cuda error (multi-bit 128-bit PBS): unsupported "
                      "grouping factor %u, supported are 2, 3 and 4", grouping);
  return PBS128_MB_INSTANCES[ilog2_exact(N) - 8];
}
static void check_mb_lwe_dimension(uint32_t n, uint32_t grouping) {
  B200_PANIC_IF_FALSE(n >= grouping && n % grouping == 0,
                      "Cuda error (multi-bit 128-bit PBS): lwe dimension %u is "
                      "not a positive multiple of the grouping factor %u", n,
                      grouping);
}

static void launch_pbs128_mb(cudaStream_t st, uint32_t gpu_index,
                             u128 *lwe_out, const uint64_t *out_idx,
                             const u128 *lut, const uint64_t *lwe_in,
                             const uint64_t *in_idx, const ddc *bsk,
                             uint32_t n, uint32_t k, uint32_t N,
                             uint32_t grouping, uint32_t base_log, uint32_t l,
                             uint32_t num_samples) {
  const Pbs128MbInstance &r = pbs128_mb_instance(k, N, l, base_log, grouping);
  check_mb_lwe_dimension(n, grouping);
  if (num_samples == 0)
    return;
  const uint32_t logM = ilog2_exact(N) - 1;
  const uint32_t grid = std::min(num_samples, sm_count(gpu_index));
  const size_t stride = pbs128_ws_bytes(k, N);
  unsigned char *ws = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(&ws, stride * grid,
                                     workspace_pool(gpu_index), st));
  launch(r.kernel, {grid, PBS128_THREADS, pbs128_mb_smem_bytes(N), st, gpu_index},
         lwe_out, out_idx, lut, lwe_in, in_idx, bsk, dd_twiddles(gpu_index, logM),
         dd_roots(gpu_index, logM), n, k, grouping, base_log, l, num_samples, ws,
         stride);
  t_last_pbs_kernel = r.name;
  B200_CHECK(cudaFreeAsync(ws, st));
}

// ===========================================================================
// BLS12-446 multi-scalar multiplication (msm.cuh)
// ===========================================================================
static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// window size, task and segment sizes, and the scratch layout of one MSM
struct MsmPlan {
  int c;
  uint32_t W, B, nb, task, S, L, count, max_tasks, max_tasks_per_bucket;
  int end_bit;
  size_t sort_temp, scan_temp;
  // byte offsets: keys/values in and out, bucket [start, end), tasks per
  // bucket and their scan, task -> bucket, task partial sums, segment totals
  // and running sums, window sums, CUB temporary storage; then the total
  size_t keys_in, vals_in, keys_out, vals_out, bounds, ntasks, toff, task_bucket, partial, seg_total, seg_run,
      win, temp, bytes;
};

// c minimises W (n + 3 B): the mixed additions of the accumulation plus the
// two additions per bucket of the reduction (with the bucket's share of the
// tree).  G2 caps c lower: its buckets are twice as large.
template <class A> static MsmPlan msm_plan(uint32_t n) {
  using F = MsmField<A>;
  using X = zk::Xyzz<F>;
  MsmPlan p{};
  const int cmax = std::is_same<F, Fp>::value ? 16 : 14;
  double best = 0;
  for (int c = 4; c <= cmax; c++) {
    const double cost = zk::num_windows(c) * ((double)n + 3.0 * (double)(1u << (c - 1)));
    if (c == 4 || cost < best)
      best = cost, p.c = c;
  }
  p.W = (uint32_t)zk::num_windows(p.c);
  p.B = 1u << (p.c - 1);
  p.nb = p.W * p.B;
  p.task = 8;
  p.S = std::min<uint32_t>(p.B, MSM_MAX_SEGMENTS);
  p.L = p.B / p.S;
  B200_PANIC_IF_FALSE((uint64_t)n * p.W < (1ull << 31), "MSM error: n = %u is too large", n);
  p.count = n * p.W;
  p.max_tasks = p.count / p.task + std::min(p.nb, p.count) + 1;
  p.max_tasks_per_bucket = (n + p.task - 1) / p.task;
  p.end_bit = 32 - __builtin_clz(p.nb);
  B200_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, p.sort_temp, (uint32_t *)nullptr, (uint32_t *)nullptr,
                                             (uint32_t *)nullptr, (uint32_t *)nullptr, (int)p.count, 0,
                                             p.end_bit));
  B200_CHECK(cub::DeviceScan::ExclusiveSum(nullptr, p.scan_temp, (uint32_t *)nullptr, (uint32_t *)nullptr,
                                           (int)(p.nb + 1)));
  size_t at = 0;
  auto take = [&at](size_t bytes) {
    const size_t off = at;
    at += align256(bytes);
    return off;
  };
  p.keys_in = take(p.count * 4ull);
  p.vals_in = take(p.count * 4ull);
  p.keys_out = take(p.count * 4ull);
  p.vals_out = take(p.count * 4ull);
  p.bounds = take(2ull * p.nb * 4);
  p.ntasks = take((p.nb + 1ull) * 4);
  p.toff = take((p.nb + 1ull) * 4);
  p.task_bucket = take(p.max_tasks * 4ull);
  p.partial = take(p.max_tasks * sizeof(X));
  p.seg_total = take((size_t)p.W * p.S * sizeof(X));
  p.seg_run = take((size_t)p.W * p.S * sizeof(X));
  p.win = take((size_t)p.W * sizeof(X));
  p.temp = take(std::max(p.sort_temp, p.scan_temp));
  p.bytes = at;
  return p;
}

static thread_local char t_last_msm_config[256] = "";
static thread_local double t_last_msm_combine_us = 0;

// sum k_i P_i of n device points (Montgomery form) and scalars into
// *h_result (host); scratch holds msm_plan<A>(n).bytes.  Synchronizes `st`.
template <class A, class Proj>
static void msm_run(cudaStream_t st, uint32_t gpu, Proj *h_result, const A *d_points, const Scalar *d_scalars,
                    uint32_t n, void *scratch) {
  using F = MsmField<A>;
  using X = zk::Xyzz<F>;
  const MsmPlan p = msm_plan<A>(n);
  unsigned char *base = static_cast<unsigned char *>(scratch);
  uint32_t *keys_in = (uint32_t *)(base + p.keys_in), *vals_in = (uint32_t *)(base + p.vals_in);
  uint32_t *keys_out = (uint32_t *)(base + p.keys_out), *vals_out = (uint32_t *)(base + p.vals_out);
  uint32_t *start = (uint32_t *)(base + p.bounds), *end = start + p.nb;
  uint32_t *ntasks = (uint32_t *)(base + p.ntasks), *toff = (uint32_t *)(base + p.toff);
  uint32_t *task_bucket = (uint32_t *)(base + p.task_bucket);
  X *partial = (X *)(base + p.partial), *seg_total = (X *)(base + p.seg_total);
  X *seg_run = (X *)(base + p.seg_run), *win = (X *)(base + p.win);
  void *temp = base + p.temp;
  constexpr uint32_t T = 128;
  auto blocks = [](uint64_t threads) { return (uint32_t)((threads + T - 1) / T); };

  launch(msm_digits_kernel, {blocks(n), T, 0, st, gpu}, d_scalars, n, p.c, keys_in, vals_in);
  size_t temp_bytes = p.sort_temp;
  B200_CHECK(cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys_in, keys_out, vals_in, vals_out, (int)p.count,
                                             0, p.end_bit, st));
  B200_CHECK(cudaMemsetAsync(start, 0, 2ull * p.nb * sizeof(uint32_t), st));
  launch(msm_bucket_bounds_kernel, {blocks(p.count), T, 0, st, gpu}, keys_out, p.count, p.nb, start, end);
  launch(msm_task_count_kernel, {blocks(p.nb + 1ull), T, 0, st, gpu}, start, end, p.nb, p.task, ntasks);
  temp_bytes = p.scan_temp;
  B200_CHECK(cub::DeviceScan::ExclusiveSum(temp, temp_bytes, ntasks, toff, (int)(p.nb + 1), st));
  launch(msm_accumulate_kernel<A>, {blocks(p.max_tasks), T, 0, st, gpu}, d_points, vals_out, start, end, toff,
         p.nb, p.task, p.max_tasks, partial, task_bucket);
  for (uint32_t step = 1; step < p.max_tasks_per_bucket; step *= 2)
    launch(msm_bucket_tree_kernel<F>, {blocks(p.max_tasks), T, 0, st, gpu}, partial, task_bucket, toff, p.nb,
           p.max_tasks, step);
  launch(msm_bucket_reduce_kernel<F>, {blocks((uint64_t)p.W * p.S), T, 0, st, gpu}, partial, toff, p.W, p.B, p.L,
         seg_total, seg_run);
  launch(msm_window_sum_kernel<F>, {p.W, p.S, 0, st, gpu}, seg_total, seg_run, p.S, p.L, win);
  X h_win[zk::SCALAR_BITS / 4 + 1];
  B200_CHECK(cudaMemcpyAsync(h_win, win, p.W * sizeof(X), cudaMemcpyDeviceToHost, st));
  B200_CHECK(cudaStreamSynchronize(st));

  // 5b. Horner over the windows on the host: sum_w 2^(c w) S_w
  const auto t0 = std::chrono::steady_clock::now();
  X acc;
  zk::xyzz_set_identity(acc);
  for (int w = (int)p.W - 1; w >= 0; w--) {
    if (!zk::xyzz_is_identity(acc))
      for (int i = 0; i < p.c; i++)
        zk::xyzz_dbl(acc, acc);
    zk::xyzz_add(acc, h_win[w]);
  }
  zk::xyzz_to_projective(*h_result, acc);
  t_last_msm_combine_us =
      std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
  std::snprintf(t_last_msm_config, sizeof(t_last_msm_config),
                "c=%d windows=%u task=%u segments=%u kernels=msm_digits_kernel,cub::DeviceRadixSort,"
                "msm_bucket_bounds_kernel,msm_task_count_kernel,cub::DeviceScan,msm_accumulate_kernel,"
                "msm_bucket_tree_kernel,msm_bucket_reduce_kernel,msm_window_sum_kernel",
                p.c, p.W, p.task, p.S);
}

static void msm_check_gpu(uint32_t gpu_index) {
  int count = 0;
  B200_CHECK(cudaGetDeviceCount(&count));
  B200_PANIC_IF_FALSE(gpu_index < (uint32_t)count, "MSM error: invalid gpu_index=%u (gpu_count=%d)", gpu_index,
                      count);
  set_device(gpu_index);
}

template <class A, class Proj>
static void msm_unmanaged(cudaStream_t stream, uint32_t gpu_index, Proj *h_result, const A *d_points,
                          const Scalar *d_scalars, uint32_t n, void *d_scratch) {
  B200_PANIC_IF_FALSE(n > 0, "MSM error: n must be positive, got %u", n);
  B200_PANIC_IF_FALSE(stream && h_result && d_points && d_scalars && d_scratch, "MSM error: null argument");
  msm_check_gpu(gpu_index);
  msm_run(stream, gpu_index, h_result, d_points, d_scalars, n, d_scratch);
}

// host arrays: points, scalars and scratch from the stream-ordered pool
template <class A, class Proj>
static void msm_managed(cudaStream_t stream, uint32_t gpu_index, Proj *result, const A *points,
                        const Scalar *scalars, uint32_t n, bool points_in_montgomery, uint64_t *size_tracker) {
  B200_PANIC_IF_FALSE(n > 0, "MSM error: n must be positive, got %u", n);
  B200_PANIC_IF_FALSE(stream && result && points && scalars && size_tracker, "MSM error: null argument");
  msm_check_gpu(gpu_index);
  const size_t pb = (size_t)n * sizeof(A), sb = (size_t)n * sizeof(Scalar);
  const size_t scratch_bytes = msm_plan<A>(n).bytes;
  unsigned char *ws = nullptr;
  const size_t bytes = align256(pb) + align256(sb) + scratch_bytes;
  B200_CHECK(cudaMallocFromPoolAsync(&ws, bytes, workspace_pool(gpu_index), stream));
  *size_tracker += bytes;
  A *d_points = (A *)ws;
  Scalar *d_scalars = (Scalar *)(ws + align256(pb));
  B200_CHECK(cudaMemcpyAsync(d_points, points, pb, cudaMemcpyHostToDevice, stream));
  B200_CHECK(cudaMemcpyAsync(d_scalars, scalars, sb, cudaMemcpyHostToDevice, stream));
  if (!points_in_montgomery)
    launch(msm_to_montgomery_kernel<A>, {(n + 127) / 128, 128, 0, stream, gpu_index}, d_points, n);
  msm_run(stream, gpu_index, result, d_points, d_scalars, n, ws + align256(pb) + align256(sb));
  B200_CHECK(cudaFreeAsync(ws, stream));
  B200_CHECK(cudaStreamSynchronize(stream));
}

// (X / Z, Y / Z, 1) in normal form; with Z = 0, X and Y leave Montgomery form
// and Z stays 0
template <class Proj> static void projective_normalized(Proj *result, const Proj *point) {
  B200_PANIC_IF_FALSE(result && point && result != point, "projective_from_montgomery: bad pointers");
  *result = *point;
  if (zk::fp_is_zero(point->Z)) {
    zk::fp_from_montgomery(result->X, point->X);
    zk::fp_from_montgomery(result->Y, point->Y);
    return;
  }
  decltype(point->Z) zi;
  zk::fp_inv(zi, point->Z);
  zk::fp_mul(result->X, point->X, zi);
  zk::fp_mul(result->Y, point->Y, zi);
  zk::fp_from_montgomery(result->X, result->X);
  zk::fp_from_montgomery(result->Y, result->Y);
  zk::fp_zero(result->Z);
  reinterpret_cast<Fp *>(&result->Z)->limb[0] = 1;  // 1, or 1 + 0 u
}

template <class A> static bool on_curve_normal(const A *point) {
  B200_PANIC_IF_FALSE(point != nullptr, "is_on_curve: point is null");
  if (point->infinity)
    return true;
  decltype(point->x) x, y;
  zk::fp_to_montgomery(x, point->x);
  zk::fp_to_montgomery(y, point->y);
  return zk::on_curve_mont(x, y);
}

template <class A> static size_t msm_scratch_size(uint32_t n, uint32_t gpu_index) {
  msm_check_gpu(gpu_index);
  return msm_plan<A>(std::max<uint32_t>(n, 1)).bytes;
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
  const PbsParams p{input_lwe_dim, glwe_dim, polynomial_size, 0, level_count, 1};
  convert_bsk<uint64_t>(static_cast<cudaStream_t>(stream), gpu_index, dest, src,
                        p, pbs_route(p));
}

uint64_t scratch_cuda_programmable_bootstrap_64_async(
    void *stream, uint32_t gpu_index, int8_t **buffer, uint32_t lwe_dimension,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t level_count,
    uint32_t input_lwe_ciphertext_count, bool allocate_gpu_memory,
    PBS_MS_REDUCTION_T noise_reduction_type) {
  (void)stream;
  set_device(gpu_index);
  check_polynomial_size(polynomial_size);
  // per-device constant tables are built here (set-up call), so that the
  // *_async bootstrap itself never runs a synchronous copy: the register
  // tables on the N = 2048 route, the generic ones for every other shape,
  // whatever its route (the 32-bit PBS runs the generic kernel on this
  // scratch object)
  const PbsParams p{lwe_dimension, glwe_dimension, polynomial_size, 0, level_count, 1};
  device_tables(gpu_index, pbs_route(p) == PbsRoute::N2048
                               ? 0
                               : ilog2_exact(polynomial_size) - 1);
  return new_pbs_scratch(buffer, CLASSICAL, glwe_dimension, polynomial_size,
                         level_count, input_lwe_ciphertext_count,
                         allocate_gpu_memory, noise_reduction_type == CENTERED);
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
  const PbsParams p{lwe_dimension, glwe_dimension, polynomial_size, base_log, level_count, 1};
  const PbsScratch &s = pbs_scratch(buffer, CLASSICAL, "classical PBS", p);
  B200_PANIC_IF_FALSE(base_log <= 64,
                      "Cuda error (classical PBS): base log should be <= 64");
  launch_pbs(static_cast<cudaStream_t>(stream), gpu_index,
             static_cast<uint64_t *>(lwe_array_out),
             static_cast<const uint64_t *>(lwe_output_indexes),
             static_cast<const uint64_t *>(lut_vector),
             static_cast<const uint64_t *>(lut_vector_indexes),
             static_cast<const uint64_t *>(lwe_array_in),
             static_cast<const uint64_t *>(lwe_input_indexes),
             bootstrapping_key, p, num_samples, num_many_lut, lut_stride,
             s.centered_ms);
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
// ciphertexts, accumulators and the three index vectors are all u32.  The
// 32-bit torus has one route whatever the shape: the generic key layout and
// kernel.
void cuda_convert_lwe_programmable_bootstrap_key_32_async(
    void *stream, uint32_t gpu_index, void *dest, void const *src,
    uint32_t input_lwe_dim, uint32_t glwe_dim, uint32_t level_count,
    uint32_t polynomial_size) {
  set_device(gpu_index);
  convert_bsk<uint32_t>(static_cast<cudaStream_t>(stream), gpu_index, dest, src,
                        PbsParams{input_lwe_dim, glwe_dim, polynomial_size, 0,
                                  level_count, 1},
                        PbsRoute::Generic);
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
  const PbsScratch &s = pbs_scratch(buffer, CLASSICAL, "classical PBS");
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
      PbsParams{lwe_dimension, glwe_dimension, polynomial_size, base_log,
                level_count, 1},
      num_samples, num_many_lut ? num_many_lut : 1, lut_stride, s.centered_ms);
}

// ---- u128 torus (programmable_bootstrap.h:57-60,68-72,92-97,102-103) ---------
void cuda_convert_lwe_programmable_bootstrap_key_128_async(
    void *stream, uint32_t gpu_index, void *dest, void const *src,
    uint32_t input_lwe_dim, uint32_t glwe_dim, uint32_t level_count,
    uint32_t polynomial_size) {
  set_device(gpu_index);
  const uint32_t k = glwe_dim, N = polynomial_size, l = level_count;
  const Pbs128Instance &r = pbs128_instance(k, N, l, 1);
  const size_t polys = (size_t)input_lwe_dim * l * (k + 1) * (k + 1);
  if (polys == 0)
    return;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // staged like convert_bsk: one device copy of the standard-domain key
  u128 *staging = nullptr;
  B200_CHECK(cudaMallocAsync(&staging, polys * N * sizeof(u128), st));
  B200_CHECK(cudaMemcpyAsync(staging, src, polys * N * sizeof(u128),
                             cudaMemcpyHostToDevice, st));
  launch(r.convert, {(unsigned)polys, 256, (N / 2) * sizeof(ddc), st, gpu_index},
         static_cast<ddc *>(dest), staging,
         dd_twiddles(gpu_index, ilog2_exact(N) - 1));
  B200_CHECK(cudaFreeAsync(staging, st));
}

uint64_t scratch_cuda_programmable_bootstrap_128_async(
    void *stream, uint32_t gpu_index, int8_t **buffer, uint32_t lwe_dimension,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t level_count,
    uint32_t input_lwe_ciphertext_count, bool allocate_gpu_memory,
    PBS_MS_REDUCTION_T noise_reduction_type) {
  (void)stream;
  (void)lwe_dimension;
  set_device(gpu_index);
  pbs128_instance(glwe_dimension, polynomial_size, level_count, 1);
  // the twiddle table is built here (set-up call), so that the bootstrap
  // itself never runs a synchronous copy
  dd_twiddles(gpu_index, ilog2_exact(polynomial_size) - 1);
  return new_pbs_scratch(buffer, CLASSICAL, glwe_dimension, polynomial_size,
                         level_count, input_lwe_ciphertext_count,
                         allocate_gpu_memory, noise_reduction_type == CENTERED,
                         true);
}

void cuda_programmable_bootstrap_128_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lut_vector, void const *lwe_array_in,
    void const *bootstrapping_key, int8_t *buffer, uint32_t lwe_dimension,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t base_log,
    uint32_t level_count, uint32_t num_samples) {
  set_device(gpu_index);
  const PbsScratch &s =
      pbs_scratch(buffer, CLASSICAL, "128-bit PBS",
                  PbsParams{lwe_dimension, glwe_dimension, polynomial_size,
                            base_log, level_count, 1},
                  num_samples, true);
  launch_pbs128(static_cast<cudaStream_t>(stream), gpu_index,
                static_cast<u128 *>(lwe_array_out),
                static_cast<const u128 *>(lut_vector),
                static_cast<const uint64_t *>(lwe_array_in),
                static_cast<const ddc *>(bootstrapping_key), lwe_dimension,
                glwe_dimension, polynomial_size, base_log, level_count,
                num_samples, s.centered_ms);
}

void cleanup_cuda_programmable_bootstrap_128(void *stream, uint32_t gpu_index,
                                             int8_t **pbs_buffer) {
  cleanup_cuda_programmable_bootstrap_64(stream, gpu_index, pbs_buffer);
}

// ---- multi-bit u128 torus (programmable_bootstrap_multibit.h:18-21,64-80) ----
void cuda_convert_lwe_multi_bit_programmable_bootstrap_key_128_async(
    void *stream, uint32_t gpu_index, void *dest, void const *src,
    uint32_t input_lwe_dim, uint32_t glwe_dim, uint32_t level_count,
    uint32_t polynomial_size, uint32_t grouping_factor) {
  set_device(gpu_index);
  const uint32_t k = glwe_dim, N = polynomial_size, l = level_count;
  pbs128_mb_instance(k, N, l, 1, grouping_factor);
  check_mb_lwe_dimension(input_lwe_dim, grouping_factor);
  // [group][2^g][l][k+1][k+1] polynomials: the classic conversion over more
  const PbsParams p{input_lwe_dim, k, N, 1, l, grouping_factor};
  const size_t polys = (size_t)p.num_ggsw() * l * (k + 1) * (k + 1);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  u128 *staging = nullptr;
  B200_CHECK(cudaMallocAsync(&staging, polys * N * sizeof(u128), st));
  B200_CHECK(cudaMemcpyAsync(staging, src, polys * N * sizeof(u128),
                             cudaMemcpyHostToDevice, st));
  launch(pbs128_instance(k, N, l, 1).convert,
         {(unsigned)polys, 256, (N / 2) * sizeof(ddc), st, gpu_index},
         static_cast<ddc *>(dest), staging,
         dd_twiddles(gpu_index, ilog2_exact(N) - 1));
  B200_CHECK(cudaFreeAsync(staging, st));
}

uint64_t scratch_cuda_multi_bit_programmable_bootstrap_128_async(
    void *stream, uint32_t gpu_index, int8_t **buffer, uint32_t glwe_dimension,
    uint32_t polynomial_size, uint32_t level_count,
    uint32_t input_lwe_ciphertext_count, bool allocate_gpu_memory) {
  (void)stream;
  set_device(gpu_index);
  pbs128_instance(glwe_dimension, polynomial_size, level_count, 1);
  // both tables are built here (set-up call), so that the bootstrap itself
  // never runs a synchronous copy
  dd_twiddles(gpu_index, ilog2_exact(polynomial_size) - 1);
  dd_roots(gpu_index, ilog2_exact(polynomial_size) - 1);
  return new_pbs_scratch(buffer, MULTI_BIT, glwe_dimension, polynomial_size,
                         level_count, input_lwe_ciphertext_count,
                         allocate_gpu_memory, 0, true);
}

void cuda_multi_bit_programmable_bootstrap_128_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lut_vector,
    void const *lwe_array_in, void const *lwe_input_indexes,
    void const *bootstrapping_key, int8_t *mem_ptr, uint32_t lwe_dimension,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t grouping_factor,
    uint32_t base_log, uint32_t level_count, uint32_t num_samples,
    uint32_t num_many_lut, uint32_t lut_stride) {
  (void)lut_stride;
  set_device(gpu_index);
  B200_PANIC_IF_FALSE(num_many_lut == 1, "Cuda error (multi-bit 128-bit PBS): "
                      "num_many_lut must be 1, got %u", num_many_lut);
  pbs_scratch(mem_ptr, MULTI_BIT, "multi-bit 128-bit PBS",
              PbsParams{lwe_dimension, glwe_dimension, polynomial_size,
                        base_log, level_count, grouping_factor},
              num_samples, true);
  launch_pbs128_mb(static_cast<cudaStream_t>(stream), gpu_index,
                   static_cast<u128 *>(lwe_array_out),
                   static_cast<const uint64_t *>(lwe_output_indexes),
                   static_cast<const u128 *>(lut_vector),
                   static_cast<const uint64_t *>(lwe_array_in),
                   static_cast<const uint64_t *>(lwe_input_indexes),
                   static_cast<const ddc *>(bootstrapping_key), lwe_dimension,
                   glwe_dimension, polynomial_size, grouping_factor, base_log,
                   level_count, num_samples);
}

void cleanup_cuda_multi_bit_programmable_bootstrap_128(void *stream,
                                                       const uint32_t gpu_index,
                                                       int8_t **buffer) {
  cleanup_cuda_programmable_bootstrap_64(stream, gpu_index, buffer);
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
  if (grouping_factor == 1) {
    // No PBS reads such a key (the multi-bit PBS rejects grouping 1).  Its
    // 2n GGSWs keep the layout of a classic key of 2n GGSWs, the N = 2048
    // register layout excepted.
    const PbsParams p{2 * input_lwe_dim, glwe_dim, polynomial_size, 0, level_count, 1};
    const PbsRoute route = pbs_route(p);
    convert_bsk<uint64_t>(static_cast<cudaStream_t>(stream), gpu_index, dest,
                          src, p,
                          route == PbsRoute::N2048 ? PbsRoute::Generic : route);
    return;
  }
  const PbsParams p{input_lwe_dim, glwe_dim, polynomial_size, 0, level_count,
                    grouping_factor};
  convert_bsk<uint64_t>(static_cast<cudaStream_t>(stream), gpu_index, dest, src,
                        p, pbs_route(p));
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
  const PbsParams p{input_lwe_dim, glwe_dim, polynomial_size, 0, level_count,
                    std::max(grouping_factor, 1u)};
  convert_seeded_bsk(static_cast<cudaStream_t>(stream), gpu_index, dest,
                     seeded_bodies, aes_key, counter_lo, counter_hi,
                     first_byte_index, p, pbs_route(p));
}

uint64_t scratch_cuda_multi_bit_programmable_bootstrap_64_async(
    void *stream, uint32_t gpu_index, int8_t **pbs_buffer,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t level_count,
    uint32_t input_lwe_ciphertext_count, bool allocate_gpu_memory) {
  (void)stream;
  set_device(gpu_index);
  check_polynomial_size(polynomial_size);
  device_tables(gpu_index, ilog2_exact(polynomial_size) - 1);
  return new_pbs_scratch(pbs_buffer, MULTI_BIT, glwe_dimension,
                         polynomial_size, level_count,
                         input_lwe_ciphertext_count, allocate_gpu_memory, 0);
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
  pbs_scratch(buffer, MULTI_BIT, "multi-bit PBS");
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
             bootstrapping_key,
             PbsParams{lwe_dimension, glwe_dimension, polynomial_size, base_log,
                       level_count, grouping_factor},
             num_samples, num_many_lut, lut_stride, 0);
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
} // extern "C"

// The 64 -> 64 keyswitch dispatch, shared by the LWE keyswitch (out_len =
// n_out + 1, body_pos = n_out) and the packing keyswitch (out_len = (k + 1) *
// N, body_pos = k * N): rows of out_len words, see keyswitch.cuh.
static void keyswitch_64(void *stream, uint32_t gpu_index, void *lwe_array_out,
                         void const *lwe_output_indexes,
                         void const *lwe_array_in,
                         void const *lwe_input_indexes, void const *ksk,
                         uint32_t lwe_dimension_in, uint32_t out_len,
                         uint32_t body_pos, uint32_t base_log,
                         uint32_t level_count, uint32_t num_samples) {
  set_device(gpu_index);
  if (num_samples == 0)
    return;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
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
    static const bool wide = std::getenv("B200_KS_IMMA_NB2") != nullptr;
    const uint32_t rows_pad = (num_samples + KI_BM - 1) / KI_BM * KI_BM;
    const uint32_t k_pad = (uint32_t)((terms + KI_BK - 1) / KI_BK * KI_BK);
    int8_t *digits = nullptr;
    // the digit matrix is a stream-ordered allocation per call from the
    // engine's private pool (see workspace_pool)
    B200_CHECK(cudaMallocFromPoolAsync(&digits, (size_t)rows_pad * k_pad,
                                       workspace_pool(gpu_index), st));
    B200_CHECK(cudaMemsetAsync(digits, 0, (size_t)rows_pad * k_pad, st));
    launch(ks_digits_kernel,
           {dim3(num_samples, (lwe_dimension_in + 255) / 256), 256, 0, st,
            gpu_index},
           digits, static_cast<const uint64_t *>(lwe_array_in),
           static_cast<const uint64_t *>(lwe_input_indexes), lwe_dimension_in,
           base_log, level_count, k_pad);
    static const struct {
      decltype(&keyswitch_imma_kernel<1>) kernel;
      uint32_t bn;
      size_t smem;
      const char *name;
    } imma_instances[2] = {
        {keyswitch_imma_kernel<1>, KiCfg<1>::BN, KiCfg<1>::SMEM, "ks_imma<1>"},
        {keyswitch_imma_kernel<2>, KiCfg<2>::BN, KiCfg<2>::SMEM, "ks_imma<2>"}};
    const auto &r = imma_instances[wide];
    const uint32_t n_bytes = out_len * 8;
    launch(r.kernel,
           {dim3(rows_pad / KI_BM, (n_bytes + r.bn - 1) / r.bn), KI_THREADS,
            r.smem, st, gpu_index},
           static_cast<uint64_t *>(lwe_array_out),
           static_cast<const uint64_t *>(lwe_output_indexes),
           static_cast<const uint64_t *>(lwe_array_in),
           static_cast<const uint64_t *>(lwe_input_indexes),
           static_cast<const uint8_t *>(ksk), digits, lwe_dimension_in, out_len,
           body_pos, level_count, k_pad, num_samples);
    t_last_ks_kernel = r.name;
    B200_CHECK(cudaFreeAsync(digits, st));
    return;
  }
  dim3 grid((num_samples + KS_TS - 1) / KS_TS, (out_len + KS_TO - 1) / KS_TO);
  // exactness condition of the fp64-pipe variant (see keyswitch.cuh)
  uint32_t terms_log2 = 0;
  while ((1ull << terms_log2) < terms)
    terms_log2++;
  // a pinned path whose precondition fails falls through in the order
  // imma -> f64 -> integer, like the automatic choice
  if (!force_int && (base_log - 1) + 32 + terms_log2 <= 52) {
    launch(keyswitch_f64_kernel, {grid, 256, sizeof(KsfSmem), st, gpu_index},
           static_cast<uint64_t *>(lwe_array_out),
           static_cast<const uint64_t *>(lwe_output_indexes),
           static_cast<const uint64_t *>(lwe_array_in),
           static_cast<const uint64_t *>(lwe_input_indexes),
           static_cast<const uint64_t *>(ksk), lwe_dimension_in, out_len,
           body_pos, base_log, level_count, num_samples);
    t_last_ks_kernel = "ks_f64";
    return;
  }
  // the s32-digit MAC holds digits up to base_log 31; wider digits (|d| up to
  // 2^(base_log - 1), l = 1) take the s64 instance
  const bool wide_digits = base_log >= 32;
  launch(wide_digits ? keyswitch_kernel<int64_t> : keyswitch_kernel<int32_t>,
         {grid, 256, 0, st, gpu_index}, static_cast<uint64_t *>(lwe_array_out),
         static_cast<const uint64_t *>(lwe_output_indexes),
         static_cast<const uint64_t *>(lwe_array_in),
         static_cast<const uint64_t *>(lwe_input_indexes),
         static_cast<const uint64_t *>(ksk), lwe_dimension_in, out_len,
         body_pos, base_log, level_count, num_samples);
  t_last_ks_kernel = wide_digits ? "ks_int_wide" : "ks_int";
}

extern "C" {

void cuda_keyswitch_lwe_ciphertext_vector_64_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_output_indexes, void const *lwe_array_in,
    void const *lwe_input_indexes, void const *ksk, uint32_t lwe_dimension_in,
    uint32_t lwe_dimension_out, uint32_t base_log, uint32_t level_count,
    uint32_t num_samples) {
  keyswitch_64(stream, gpu_index, lwe_array_out, lwe_output_indexes,
               lwe_array_in, lwe_input_indexes, ksk, lwe_dimension_in,
               lwe_dimension_out + 1, lwe_dimension_out, base_log, level_count,
               num_samples);
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
  launch(keyswitch_64_32_kernel,
         {grid, 256, 0, static_cast<cudaStream_t>(stream), gpu_index},
         static_cast<uint32_t *>(lwe_array_out),
         static_cast<const uint64_t *>(lwe_output_indexes),
         static_cast<const uint64_t *>(lwe_array_in),
         static_cast<const uint64_t *>(lwe_input_indexes),
         static_cast<const uint32_t *>(ksk), lwe_dimension_in,
         lwe_dimension_out, base_log, level_count, num_samples);
  t_last_ks_kernel = "ks_64_32";
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
  launch(glwe_sample_extract_kernel,
         {num_nths, 256, 0, static_cast<cudaStream_t>(stream), gpu_index},
         static_cast<uint64_t *>(lwe_array_out),
         static_cast<const uint64_t *>(glwe_array_in), nth_array,
         num_lwes_to_extract_per_glwe, num_lwes_stored_per_glwe,
         glwe_dimension, polynomial_size);
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
  launch(modulus_switch_kernel,
         {(size + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream),
          gpu_index},
         static_cast<uint64_t *>(lwe_out),
         static_cast<const uint64_t *>(lwe_in), size, log_modulus);
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
  launch(centered_modulus_switch_kernel,
         {1, 256, 0, static_cast<cudaStream_t>(stream), gpu_index},
         static_cast<uint64_t *>(lwe_out),
         static_cast<const uint64_t *>(lwe_in), lwe_dimension, log_modulus);
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
  launch(forward_fft_natural_kernel,
         {total_polynomials, 64, 0, static_cast<cudaStream_t>(stream),
          gpu_index},
         static_cast<cplx *>(output), static_cast<const cplx *>(input),
         t.fft1024);
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
  const PbsParams p{lwe_dimension, glwe_dimension, polynomial_size, base_log,
                    level_count, std::max(grouping_factor, 1u)};
  pbs_scratch(buffer, p.type(), "OPRF", p);
  if (num_blocks == 0)
    return;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint64_t in_words = (uint64_t)num_blocks * (lwe_dimension + 1);
  uint64_t *ws = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(
      &ws, (in_words + num_blocks) * sizeof(uint64_t),
      workspace_pool(gpu_index), st));
  uint64_t *idx = ws + in_words;
  launch(oprf_iota_kernel, {(num_blocks + 255) / 256, 256, 0, st, gpu_index},
         idx, num_blocks);
  oprf_expand(st, gpu_index, ws, aes_key, counter_lo, counter_hi, 0,
              lwe_dimension, num_blocks, ilog2_exact(polynomial_size) + 1);
  // centered_ms = 0 whatever the scratch object says: the switched values
  // are exact and must not be corrected again
  launch_pbs(st, gpu_index, static_cast<uint64_t *>(lwe_out), idx,
             static_cast<const uint64_t *>(lut_vector),
             static_cast<const uint64_t *>(lut_indexes), ws, idx,
             bootstrapping_key, p, num_blocks, 1, 0, 0);
  const uint64_t big_n = (uint64_t)glwe_dimension * polynomial_size;
  launch(oprf_add_corrections_kernel,
         {(num_blocks + 255) / 256, 256, 0, st, gpu_index},
         static_cast<uint64_t *>(lwe_out),
         static_cast<const uint64_t *>(corrections), big_n, num_blocks);
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
  const PbsParams p{lwe_dimension, glwe_dimension, polynomial_size,
                    pbs_base_log, pbs_level_count, std::max(grouping_factor, 1u)};
  const uint64_t T = compact_lists_total(num_lwes_per_compact_list,
                                         num_compact_lists,
                                         compact_lwe_dimension);
  const PbsScratch &s = pbs_scratch(buffer, p.type(), "expand", p, 2 * T);
  B200_PANIC_IF_FALSE(casting_ksk && (!casting_to_big || computing_ksk),
                      "Cuda error (expand): missing keyswitching key");
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
  launch(compact_unpack_index_kernel,
         {(samples + 255) / 256, 256, 0, st, gpu_index}, in_idx, out_idx,
         samples);
  launch_pbs(st, gpu_index, static_cast<uint64_t *>(lwe_array_out), out_idx,
             static_cast<const uint64_t *>(lut_vector),
             static_cast<const uint64_t *>(lut_indexes), small, in_idx,
             bootstrapping_key, p, samples, 1, 0, s.centered_ms);
  B200_CHECK(cudaFreeAsync(ws, st));
}

void b200_cpk_encrypt_zeros_from_seeds_64_async(
    void *stream, uint32_t gpu_index, void *lwe_flattened_compact_array_out,
    void const *compact_public_key, const uint8_t *seeds, uint32_t num_seeds,
    const uint64_t *entries, uint32_t num_entries, uint32_t lwe_dimension,
    uint32_t noise_bound_log2, bool accumulate) {
  set_device(gpu_index);
  cpk_encrypt_zeros(static_cast<cudaStream_t>(stream), gpu_index,
                    static_cast<uint64_t *>(lwe_flattened_compact_array_out),
                    static_cast<const uint64_t *>(compact_public_key), seeds,
                    num_seeds, entries, num_entries, lwe_dimension,
                    noise_bound_log2, accumulate);
}

void b200_rerand_64_async(void *stream, uint32_t gpu_index, void *lwe_array,
                          void const *lwe_flattened_compact_array_in,
                          const uint32_t *num_lwes_per_compact_list,
                          uint32_t num_compact_lists,
                          uint32_t compact_lwe_dimension, void const *ksk,
                          uint32_t ksk_base_log, uint32_t ksk_level_count,
                          uint32_t lwe_dimension) {
  set_device(gpu_index);
  B200_PANIC_IF_FALSE(ksk || lwe_dimension == compact_lwe_dimension,
                      "Cuda error (rerand): without a keyswitching key the "
                      "ciphertexts (dimension %u) must be under the compact "
                      "key (dimension %u)", lwe_dimension,
                      compact_lwe_dimension);
  const uint64_t T = compact_lists_total(num_lwes_per_compact_list,
                                         num_compact_lists,
                                         compact_lwe_dimension);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint64_t exp_words = T * (compact_lwe_dimension + 1);
  const uint64_t out_words = T * ((uint64_t)lwe_dimension + 1);
  uint64_t *ws = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(
      &ws, (exp_words + (ksk ? out_words : 0)) * sizeof(uint64_t),
      workspace_pool(gpu_index), st));
  compact_expand(st, gpu_index, ws,
                 static_cast<const uint64_t *>(lwe_flattened_compact_array_in),
                 num_lwes_per_compact_list, num_compact_lists,
                 compact_lwe_dimension);
  uint64_t *zeros = ws;
  if (ksk) {
    zeros = ws + exp_words;
    cuda_keyswitch_lwe_ciphertext_vector_64_64_async(
        stream, gpu_index, zeros, nullptr, ws, nullptr, ksk,
        compact_lwe_dimension, lwe_dimension, ksk_base_log, ksk_level_count,
        (uint32_t)T);
  }
  const uint64_t blocks = std::min<uint64_t>((out_words + 255) / 256, 65535u);
  launch(rerand_add_kernel, {(unsigned)blocks, 256, 0, st, gpu_index},
         static_cast<uint64_t *>(lwe_array), zeros, out_words);
  B200_CHECK(cudaFreeAsync(ws, st));
}

// ===========================================================================
// packing keyswitch and ciphertext-list compression (compression.cuh)
// ===========================================================================
// The scratch buffer is the per-LWE GLWE rows the keyswitch writes before the
// pack-in-GLWE sum: num_lwes * (k + 1) * N words.
uint64_t scratch_cuda_packing_keyswitch_lwe_list_to_glwe_64_async(
    void *stream, uint32_t gpu_index, int8_t **fp_ks_buffer,
    uint32_t lwe_dimension, uint32_t glwe_dimension, uint32_t polynomial_size,
    uint32_t num_lwes, bool allocate_gpu_memory) {
  (void)lwe_dimension;
  set_device(gpu_index);
  const uint64_t bytes = (uint64_t)num_lwes * (glwe_dimension + 1) *
                         polynomial_size * sizeof(uint64_t);
  *fp_ks_buffer = nullptr;
  if (allocate_gpu_memory && bytes)
    B200_CHECK(cudaMallocAsync(reinterpret_cast<void **>(fp_ks_buffer), bytes,
                               static_cast<cudaStream_t>(stream)));
  return bytes;
}

void cuda_packing_keyswitch_lwe_list_to_glwe_64_async(
    void *stream, uint32_t gpu_index, void *glwe_array_out,
    void const *lwe_array_in, void const *fp_ksk_array, int8_t *fp_ks_buffer,
    uint32_t input_lwe_dimension, uint32_t output_glwe_dimension,
    uint32_t output_polynomial_size, uint32_t base_log, uint32_t level_count,
    uint32_t num_lwes) {
  set_device(gpu_index);
  check_polynomial_size(output_polynomial_size);
  B200_PANIC_IF_FALSE(num_lwes <= output_polynomial_size,
                      "Cuda error (packing keyswitch): %u LWEs do not fit in "
                      "one GLWE of N = %u", num_lwes, output_polynomial_size);
  if (num_lwes == 0)
    return;
  B200_PANIC_IF_FALSE(fp_ks_buffer, "Cuda error (packing keyswitch): the "
                                    "scratch buffer was not allocated");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint32_t k = output_glwe_dimension, N = output_polynomial_size;
  uint64_t *rows = reinterpret_cast<uint64_t *>(fp_ks_buffer);
  keyswitch_64(stream, gpu_index, rows, nullptr, lwe_array_in, nullptr,
               fp_ksk_array, input_lwe_dimension, (k + 1) * N, k * N, base_log,
               level_count, num_lwes);
  launch(pack_glwe_kernel,
         {dim3((k + 1) * N / PACK_THREADS, 1), PACK_THREADS, 0, st, gpu_index},
         static_cast<uint64_t *>(glwe_array_out), rows, k, N, num_lwes,
         num_lwes, 0);
}

void cleanup_cuda_packing_keyswitch_lwe_list_to_glwe_64(
    void *stream, uint32_t gpu_index, int8_t **fp_ks_buffer,
    bool gpu_memory_allocated) {
  set_device(gpu_index);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (gpu_memory_allocated && *fp_ks_buffer)
    B200_CHECK(cudaFreeAsync(*fp_ks_buffer, st));
  *fp_ks_buffer = nullptr;
  B200_CHECK(cudaStreamSynchronize(st));
}

static void check_compression_layout(uint32_t lwe_per_glwe, uint32_t N,
                                     uint32_t storage_log_modulus) {
  check_polynomial_size(N);
  B200_PANIC_IF_FALSE(lwe_per_glwe >= 1 && lwe_per_glwe <= N,
                      "Cuda error (compression): lwe_per_glwe %u must be in "
                      "[1, N = %u]", lwe_per_glwe, N);
  B200_PANIC_IF_FALSE(storage_log_modulus >= 1 && storage_log_modulus <= 64,
                      "Cuda error (compression): storage_log_modulus %u must "
                      "be in [1, 64]", storage_log_modulus);
}

void b200_compress_lwe_ciphertexts_64_async(
    void *stream, uint32_t gpu_index, void *packed_out, void const *lwe_array_in,
    uint32_t num_lwes, uint32_t lwe_dimension, uint64_t scale,
    void const *packing_ksk, uint32_t glwe_dimension, uint32_t polynomial_size,
    uint32_t base_log, uint32_t level_count, uint32_t lwe_per_glwe,
    uint32_t storage_log_modulus) {
  set_device(gpu_index);
  check_compression_layout(lwe_per_glwe, polynomial_size, storage_log_modulus);
  if (num_lwes == 0)
    return;
  const uint32_t num_glwes = (num_lwes + lwe_per_glwe - 1) / lwe_per_glwe;
  B200_PANIC_IF_FALSE(num_glwes <= 65535u, "Cuda error (compression): %u "
                      "GLWEs are too many for one call", num_glwes);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint32_t k = glwe_dimension, N = polynomial_size;
  const uint64_t in_words = (uint64_t)num_lwes * (lwe_dimension + 1);
  const uint64_t row_words = (uint64_t)num_lwes * (k + 1) * N;
  uint64_t *ws = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(&ws, (in_words + row_words) * sizeof(uint64_t),
                                     workspace_pool(gpu_index), st));
  uint64_t *scaled = ws, *rows = ws + in_words;
  const uint64_t blocks = std::min<uint64_t>((in_words + 255) / 256, 65535u);
  launch(compression_scale_kernel, {(unsigned)blocks, 256, 0, st, gpu_index},
         scaled, static_cast<const uint64_t *>(lwe_array_in), in_words, scale);
  keyswitch_64(stream, gpu_index, rows, nullptr, scaled, nullptr, packing_ksk,
               lwe_dimension, (k + 1) * N, k * N, base_log, level_count,
               num_lwes);
  launch(pack_glwe_kernel,
         {dim3((k + 1) * N / PACK_THREADS, num_glwes), PACK_THREADS, 0, st,
          gpu_index},
         static_cast<uint64_t *>(packed_out), rows, k, N, num_lwes,
         lwe_per_glwe, storage_log_modulus);
  B200_CHECK(cudaFreeAsync(ws, st));
}

void b200_decompress_lwe_ciphertexts_64_async(
    void *stream, uint32_t gpu_index, void *lwe_out, void const *packed_in,
    uint32_t num_lwes_in_list, const uint32_t *indexes, uint32_t num_indexes,
    uint32_t compression_glwe_dimension, uint32_t compression_polynomial_size,
    uint32_t lwe_per_glwe, uint32_t storage_log_modulus, void const *lut_vector,
    void const *bootstrapping_key, int8_t *buffer, uint32_t glwe_dimension,
    uint32_t polynomial_size, uint32_t base_log, uint32_t level_count,
    uint32_t grouping_factor) {
  set_device(gpu_index);
  check_compression_layout(lwe_per_glwe, compression_polynomial_size,
                           storage_log_modulus);
  check_polynomial_size(polynomial_size);
  const uint32_t big_n = compression_glwe_dimension * compression_polynomial_size;
  const PbsParams p{big_n, glwe_dimension, polynomial_size, base_log,
                    level_count, std::max(grouping_factor, 1u)};
  pbs_scratch(buffer, p.type(), "decompression", p, num_indexes);
  if (num_indexes == 0)
    return;
  // trivial PBS indexes, one all-zero LUT index per sample, then the list
  // indexes: one stream-ordered copy (staged from pageable memory)
  std::vector<uint64_t> h_idx(3 * (size_t)num_indexes, 0);
  for (uint32_t r = 0; r < num_indexes; r++) {
    B200_PANIC_IF_FALSE(indexes[r] < num_lwes_in_list,
                        "Cuda error (decompression): index %u out of range "
                        "for a list of %u ciphertexts", indexes[r],
                        num_lwes_in_list);
    h_idx[r] = r;
    h_idx[2 * (size_t)num_indexes + r] = indexes[r];
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint64_t lwe_words = (uint64_t)num_indexes * (big_n + 1);
  uint64_t *ws = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(
      &ws, (lwe_words + h_idx.size()) * sizeof(uint64_t),
      workspace_pool(gpu_index), st));
  uint64_t *extracted = ws, *iota = ws + lwe_words;
  uint64_t *lut_idx = iota + num_indexes, *list_idx = lut_idx + num_indexes;
  B200_CHECK(cudaMemcpyAsync(iota, h_idx.data(), h_idx.size() * sizeof(uint64_t),
                             cudaMemcpyHostToDevice, st));
  launch(unpack_extract_kernel,
         {dim3((big_n + 1 + 255) / 256, std::min<uint32_t>(num_indexes, 65535u)),
          256, 0, st, gpu_index},
         extracted, static_cast<const uint64_t *>(packed_in), list_idx,
         num_indexes, compression_glwe_dimension, compression_polynomial_size,
         lwe_per_glwe, storage_log_modulus);
  // no centered-mean correction: the extracted words are exact multiples of
  // 2^(64 - storage_log_modulus) and must not move (as in the grouped OPRF)
  launch_pbs(st, gpu_index, static_cast<uint64_t *>(lwe_out), iota,
             static_cast<const uint64_t *>(lut_vector), lut_idx, extracted, iota,
             bootstrapping_key, p, num_indexes, 1, 0, 0);
  B200_CHECK(cudaFreeAsync(ws, st));
}

void b200_apply_noise_squashing_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_array_in, uint32_t num_blocks, uint32_t input_lwe_dimension,
    uint32_t message_modulus, void const *ksk, uint32_t ks_base_log,
    uint32_t ks_level_count, void const *lut_vector,
    void const *bootstrapping_key, int8_t *buffer, uint32_t lwe_dimension,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t pbs_base_log,
    uint32_t pbs_level_count) {
  set_device(gpu_index);
  pbs128_instance(glwe_dimension, polynomial_size, pbs_level_count,
                  pbs_base_log);
  const uint32_t packed = (num_blocks + 1) / 2;
  const PbsParams p{lwe_dimension, glwe_dimension, polynomial_size,
                    pbs_base_log, pbs_level_count, 1};
  const PbsScratch &s =
      pbs_scratch(buffer, p.type(), "noise squashing", p, packed, true);
  if (num_blocks == 0)
    return;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint64_t big_words = (uint64_t)packed * (input_lwe_dimension + 1);
  const uint64_t small_words = (uint64_t)packed * (lwe_dimension + 1);
  uint64_t *ws = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(&ws, (big_words + small_words) * sizeof(uint64_t),
                                     workspace_pool(gpu_index), st));
  uint64_t *pairs = ws, *small = ws + big_words;
  launch(squash_pack_pairs_kernel,
         {(unsigned)((big_words + 255) / 256), 256, 0, st, gpu_index}, pairs,
         static_cast<const uint64_t *>(lwe_array_in), input_lwe_dimension + 1,
         num_blocks, (uint64_t)message_modulus);
  keyswitch_64(stream, gpu_index, small, nullptr, pairs, nullptr, ksk,
               input_lwe_dimension, lwe_dimension + 1, lwe_dimension,
               ks_base_log, ks_level_count, packed);
  launch_pbs128(st, gpu_index, static_cast<u128 *>(lwe_array_out),
                static_cast<const u128 *>(lut_vector), small,
                static_cast<const ddc *>(bootstrapping_key), lwe_dimension,
                glwe_dimension, polynomial_size, pbs_base_log, pbs_level_count,
                packed, s.centered_ms);
  B200_CHECK(cudaFreeAsync(ws, st));
}

void b200_apply_noise_squashing_multi_bit_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out,
    void const *lwe_array_in, uint32_t num_blocks, uint32_t input_lwe_dimension,
    uint32_t message_modulus, void const *ksk, uint32_t ks_base_log,
    uint32_t ks_level_count, void const *lut_vector,
    void const *bootstrapping_key, int8_t *buffer, uint32_t lwe_dimension,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t grouping_factor,
    uint32_t pbs_base_log, uint32_t pbs_level_count) {
  set_device(gpu_index);
  pbs128_mb_instance(glwe_dimension, polynomial_size, pbs_level_count,
                     pbs_base_log, grouping_factor);
  check_mb_lwe_dimension(lwe_dimension, grouping_factor);
  const uint32_t packed = (num_blocks + 1) / 2;
  const PbsParams p{lwe_dimension, glwe_dimension, polynomial_size,
                    pbs_base_log, pbs_level_count, grouping_factor};
  pbs_scratch(buffer, p.type(), "multi-bit noise squashing", p, packed, true);
  if (num_blocks == 0)
    return;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint64_t big_words = (uint64_t)packed * (input_lwe_dimension + 1);
  const uint64_t small_words = (uint64_t)packed * (lwe_dimension + 1);
  uint64_t *ws = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(&ws, (big_words + small_words) * sizeof(uint64_t),
                                     workspace_pool(gpu_index), st));
  uint64_t *pairs = ws, *small = ws + big_words;
  launch(squash_pack_pairs_kernel,
         {(unsigned)((big_words + 255) / 256), 256, 0, st, gpu_index}, pairs,
         static_cast<const uint64_t *>(lwe_array_in), input_lwe_dimension + 1,
         num_blocks, (uint64_t)message_modulus);
  keyswitch_64(stream, gpu_index, small, nullptr, pairs, nullptr, ksk,
               input_lwe_dimension, lwe_dimension + 1, lwe_dimension,
               ks_base_log, ks_level_count, packed);
  launch_pbs128_mb(st, gpu_index, static_cast<u128 *>(lwe_array_out), nullptr,
                   static_cast<const u128 *>(lut_vector), small, nullptr,
                   static_cast<const ddc *>(bootstrapping_key), lwe_dimension,
                   glwe_dimension, polynomial_size, grouping_factor,
                   pbs_base_log, pbs_level_count, packed);
  B200_CHECK(cudaFreeAsync(ws, st));
}

// ===========================================================================
// u128 packing keyswitch and noise-squashing compression (keyswitch128.cuh)
// ===========================================================================
static void check_decomposition_128(uint32_t base_log, uint32_t level_count) {
  B200_PANIC_IF_FALSE(base_log >= 1 && base_log <= 63 && level_count >= 1 &&
                          base_log * level_count <= 128,
                      "Cuda error (128-bit packing keyswitch): base_log %u, "
                      "level_count %u: need 1 <= base_log <= 63, "
                      "level_count >= 1, base_log * level_count <= 128",
                      base_log, level_count);
}

// the packing keyswitch of `count` u128 LWEs into rows of (k + 1) N words
static void keyswitch_128(cudaStream_t st, uint32_t gpu_index, u128 *rows,
                          const void *lwe_in, const void *ksk, uint32_t n_in,
                          uint32_t k, uint32_t N, uint32_t base_log,
                          uint32_t level_count, uint32_t count) {
  const uint32_t out_len = (k + 1) * N, col_tiles = (out_len + KS128_TO - 1) / KS128_TO;
  auto *in = static_cast<const u128 *>(lwe_in);
  auto *key = static_cast<const u128 *>(ksk);
  if (count < 64)
    launch(keyswitch128_kernel<1>, {dim3((count + 15) / 16, col_tiles), 256, 0, st, gpu_index},
           rows, in, key, n_in, out_len, k * N, base_log, level_count, count);
  else
    launch(keyswitch128_kernel<4>, {dim3((count + 63) / 64, col_tiles), 256, 0, st, gpu_index},
           rows, in, key, n_in, out_len, k * N, base_log, level_count, count);
  t_last_ks_kernel = "ks128";
}

void scratch_cuda_packing_keyswitch_lwe_list_to_glwe_128_async(
    void *stream, uint32_t gpu_index, int8_t **fp_ks_buffer,
    uint32_t lwe_dimension, uint32_t glwe_dimension, uint32_t polynomial_size,
    uint32_t num_lwes, bool allocate_gpu_memory) {
  (void)lwe_dimension;
  set_device(gpu_index);
  const uint64_t bytes = (uint64_t)num_lwes * (glwe_dimension + 1) *
                         polynomial_size * sizeof(u128);
  *fp_ks_buffer = nullptr;
  if (allocate_gpu_memory && bytes)
    B200_CHECK(cudaMallocAsync(reinterpret_cast<void **>(fp_ks_buffer), bytes,
                               static_cast<cudaStream_t>(stream)));
}

void cuda_packing_keyswitch_lwe_list_to_glwe_128_async(
    void *stream, uint32_t gpu_index, void *glwe_array_out,
    void const *lwe_array_in, void const *fp_ksk_array, int8_t *fp_ks_buffer,
    uint32_t input_lwe_dimension, uint32_t output_glwe_dimension,
    uint32_t output_polynomial_size, uint32_t base_log, uint32_t level_count,
    uint32_t num_lwes) {
  set_device(gpu_index);
  check_polynomial_size(output_polynomial_size);
  check_decomposition_128(base_log, level_count);
  B200_PANIC_IF_FALSE(num_lwes <= output_polynomial_size,
                      "Cuda error (128-bit packing keyswitch): %u LWEs do not "
                      "fit in one GLWE of N = %u", num_lwes,
                      output_polynomial_size);
  if (num_lwes == 0)
    return;
  B200_PANIC_IF_FALSE(fp_ks_buffer, "Cuda error (128-bit packing keyswitch): "
                                    "the scratch buffer was not allocated");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint32_t k = output_glwe_dimension, N = output_polynomial_size;
  u128 *rows = reinterpret_cast<u128 *>(fp_ks_buffer);
  keyswitch_128(st, gpu_index, rows, lwe_array_in, fp_ksk_array,
                input_lwe_dimension, k, N, base_log, level_count, num_lwes);
  launch(pack128_glwe_kernel,
         {dim3((k + 1) * N / PACK128_THREADS, 1), PACK128_THREADS, 0, st, gpu_index},
         static_cast<u128 *>(glwe_array_out), rows, k, N, num_lwes, num_lwes,
         false);
}

void cleanup_cuda_packing_keyswitch_lwe_list_to_glwe_128(
    void *stream, uint32_t gpu_index, int8_t **fp_ks_buffer,
    bool gpu_memory_allocated) {
  cleanup_cuda_packing_keyswitch_lwe_list_to_glwe_64(stream, gpu_index,
                                                     fp_ks_buffer,
                                                     gpu_memory_allocated);
}

static void check_lwe_per_glwe(uint32_t lwe_per_glwe, uint32_t N) {
  check_polynomial_size(N);
  B200_PANIC_IF_FALSE(lwe_per_glwe >= 1 && lwe_per_glwe <= N,
                      "Cuda error (noise-squashing compression): lwe_per_glwe "
                      "%u must be in [1, N = %u]", lwe_per_glwe, N);
}

void b200_compress_lwe_ciphertexts_128_async(
    void *stream, uint32_t gpu_index, void *packed_out, void const *lwe_array_in,
    uint32_t num_lwes, uint32_t lwe_dimension, void const *packing_ksk,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t base_log,
    uint32_t level_count, uint32_t lwe_per_glwe) {
  set_device(gpu_index);
  check_lwe_per_glwe(lwe_per_glwe, polynomial_size);
  check_decomposition_128(base_log, level_count);
  if (num_lwes == 0)
    return;
  const uint32_t num_glwes = (num_lwes + lwe_per_glwe - 1) / lwe_per_glwe;
  B200_PANIC_IF_FALSE(num_glwes <= 65535u, "Cuda error (noise-squashing "
                      "compression): %u GLWEs are too many for one call",
                      num_glwes);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint32_t k = glwe_dimension, N = polynomial_size;
  u128 *rows = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(
      reinterpret_cast<void **>(&rows),
      (uint64_t)num_lwes * (k + 1) * N * sizeof(u128), workspace_pool(gpu_index),
      st));
  keyswitch_128(st, gpu_index, rows, lwe_array_in, packing_ksk, lwe_dimension,
                k, N, base_log, level_count, num_lwes);
  launch(pack128_glwe_kernel,
         {dim3((k + 1) * N / PACK128_THREADS, num_glwes), PACK128_THREADS, 0, st,
          gpu_index},
         static_cast<u128 *>(packed_out), rows, k, N, num_lwes, lwe_per_glwe,
         true);
  B200_CHECK(cudaFreeAsync(rows, st));
}

void b200_decompress_lwe_ciphertexts_128_async(
    void *stream, uint32_t gpu_index, void *lwe_out, void const *packed_in,
    uint32_t num_lwes_in_list, const uint32_t *indexes, uint32_t num_indexes,
    uint32_t glwe_dimension, uint32_t polynomial_size, uint32_t lwe_per_glwe) {
  set_device(gpu_index);
  check_lwe_per_glwe(lwe_per_glwe, polynomial_size);
  if (num_indexes == 0)
    return;
  std::vector<uint64_t> h_idx(num_indexes);
  for (uint32_t r = 0; r < num_indexes; r++) {
    B200_PANIC_IF_FALSE(indexes[r] < num_lwes_in_list,
                        "Cuda error (noise-squashing decompression): index %u "
                        "out of range for a list of %u ciphertexts",
                        indexes[r], num_lwes_in_list);
    h_idx[r] = indexes[r];
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint64_t *idx = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(reinterpret_cast<void **>(&idx),
                                     h_idx.size() * sizeof(uint64_t),
                                     workspace_pool(gpu_index), st));
  B200_CHECK(cudaMemcpyAsync(idx, h_idx.data(), h_idx.size() * sizeof(uint64_t),
                             cudaMemcpyHostToDevice, st));
  const uint32_t big_n = glwe_dimension * polynomial_size;
  launch(unpack_extract128_kernel,
         {dim3((big_n + 1 + 255) / 256, std::min<uint32_t>(num_indexes, 65535u)),
          256, 0, st, gpu_index},
         static_cast<u128 *>(lwe_out), static_cast<const u128 *>(packed_in), idx,
         num_indexes, glwe_dimension, polynomial_size, lwe_per_glwe);
  B200_CHECK(cudaFreeAsync(idx, st));
}

// ===========================================================================
// bit circuits (bit_circuit.cuh; tfhe-rs_b200/bit_circuit.py)
// ===========================================================================
static uint64_t lincomb_outputs(uint32_t num_rows, uint32_t num_shared_rows,
                                uint32_t num_instances) {
  B200_PANIC_IF_FALSE(num_shared_rows <= num_rows && num_instances >= 1,
                      "Cuda error (linear combination): %u shared rows of %u, "
                      "%u instances", num_shared_rows, num_rows, num_instances);
  const uint64_t outs = num_shared_rows +
                        (uint64_t)(num_rows - num_shared_rows) * num_instances;
  B200_PANIC_IF_FALSE(outs < (1ull << 31), "Cuda error (linear combination): "
                      "%llu output rows are too many for one launch",
                      (unsigned long long)outs);
  return outs;
}

static void linear_combination(cudaStream_t st, uint32_t gpu_index,
                               uint64_t *out, const uint64_t *pool,
                               uint32_t lwe_dimension, uint32_t num_shared_slots,
                               uint32_t num_instances, uint32_t num_rows,
                               uint32_t num_shared_rows,
                               const uint32_t *row_offsets,
                               const uint32_t *term_slots,
                               const int64_t *term_coefs, const uint64_t *body) {
  const uint64_t outs = lincomb_outputs(num_rows, num_shared_rows, num_instances);
  if (outs == 0)
    return;
  launch(lwe_linear_combination_kernel,
         {(unsigned)outs, LINCOMB_THREADS, 0, st, gpu_index}, out, pool,
         lwe_dimension + 1, num_shared_slots, num_instances, num_shared_rows,
         row_offsets, term_slots, term_coefs, body);
}

void b200_lwe_linear_combination_64_async(
    void *stream, uint32_t gpu_index, void *lwe_array_out, void const *pool,
    uint32_t lwe_dimension, uint32_t num_shared_slots, uint32_t num_instances,
    uint32_t num_rows, uint32_t num_shared_rows, void const *row_offsets,
    void const *term_slots, void const *term_coefs,
    void const *body_constants) {
  set_device(gpu_index);
  linear_combination(static_cast<cudaStream_t>(stream), gpu_index,
                     static_cast<uint64_t *>(lwe_array_out),
                     static_cast<const uint64_t *>(pool), lwe_dimension,
                     num_shared_slots, num_instances, num_rows, num_shared_rows,
                     static_cast<const uint32_t *>(row_offsets),
                     static_cast<const uint32_t *>(term_slots),
                     static_cast<const int64_t *>(term_coefs),
                     static_cast<const uint64_t *>(body_constants));
}

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
    uint32_t pbs_base_log, uint32_t pbs_level_count, uint32_t grouping_factor) {
  set_device(gpu_index);
  check_polynomial_size(polynomial_size);
  B200_PANIC_IF_FALSE(big_lwe_dimension == glwe_dimension * polynomial_size,
                      "Cuda error (bit circuit): big LWE dimension %u is not "
                      "k * N = %u", big_lwe_dimension,
                      glwe_dimension * polynomial_size);
  const PbsParams p{lwe_dimension, glwe_dimension, polynomial_size,
                    pbs_base_log, pbs_level_count, std::max(grouping_factor, 1u)};
  // output rows of every layer, and the widest
  std::vector<uint64_t> outs(num_layers);
  uint64_t widest = 0;
  for (uint32_t L = 0; L < num_layers; L++) {
    B200_PANIC_IF_FALSE(layer_rows[L] <= layer_rows[L + 1],
                        "Cuda error (bit circuit): layer %u ends before it "
                        "starts", L);
    outs[L] = lincomb_outputs(layer_rows[L + 1] - layer_rows[L],
                              layer_shared_rows[L], num_instances);
    widest = std::max(widest, outs[L]);
  }
  const PbsScratch &s = pbs_scratch(buffer, p.type(), "bit circuit", p, widest);
  if (widest == 0)
    return;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint64_t *ws = nullptr;
  B200_CHECK(cudaMallocFromPoolAsync(
      &ws, widest * (big_lwe_dimension + lwe_dimension + 2) * sizeof(uint64_t),
      workspace_pool(gpu_index), st));
  uint64_t *big = ws, *small = ws + widest * (big_lwe_dimension + 1);
  uint64_t *d_pool = static_cast<uint64_t *>(pool);
  const uint64_t *lut_idx = static_cast<const uint64_t *>(lut_indexes);
  const uint64_t *out_idx = static_cast<const uint64_t *>(output_indexes);
  uint64_t out_base = 0;
  for (uint32_t L = 0; L < num_layers; L++) {
    if (outs[L] == 0)
      continue;
    // 1. linear step into the staging rows (reads the pool only)
    linear_combination(
        st, gpu_index, big, d_pool, big_lwe_dimension, num_shared_slots,
        num_instances, layer_rows[L + 1] - layer_rows[L], layer_shared_rows[L],
        static_cast<const uint32_t *>(row_offsets) + layer_rows[L],
        static_cast<const uint32_t *>(term_slots),
        static_cast<const int64_t *>(term_coefs),
        static_cast<const uint64_t *>(body_constants) +
            (uint64_t)layer_rows[L] * num_instances);
    // 2. keyswitch (the LWE keyswitch's own kernel choice)
    keyswitch_64(stream, gpu_index, small, nullptr, big, nullptr, ksk,
                 big_lwe_dimension, lwe_dimension + 1, lwe_dimension,
                 ks_base_log, ks_level_count, (uint32_t)outs[L]);
    // 3. PBS scattering straight into the pool
    launch_pbs(st, gpu_index, d_pool, out_idx + out_base,
               static_cast<const uint64_t *>(lut_vector), lut_idx + out_base,
               small, static_cast<const uint64_t *>(input_indexes),
               bootstrapping_key, p, (uint32_t)outs[L], 1, 0,
               p.grouping > 1 ? 0 : s.centered_ms);
    out_base += outs[L];
  }
  B200_CHECK(cudaFreeAsync(ws, st));
}

uint64_t b200_kernel_launch_count(void) {
  return g_launches.load(std::memory_order_relaxed);
}

const char *b200_last_pbs_kernel(void) { return t_last_pbs_kernel; }

const char *b200_last_keyswitch_kernel(void) { return t_last_ks_kernel; }

int b200_pbs_uses_fast_path(uint32_t lwe_dimension, uint32_t glwe_dimension,
                            uint32_t polynomial_size, uint32_t level_count) {
  return pbs_route(PbsParams{lwe_dimension, glwe_dimension, polynomial_size, 0,
                             level_count, 1}) == PbsRoute::N2048;
}

const char *b200_version(void) { return "tfhe-rs_b200 0.1 (sm_90a)"; }

// ===========================================================================
// zk-cuda-backend C ABI (include/tfhe_b200_zk.h)
// ===========================================================================
void affine_to_projective_g1_wrapper(G1ProjectivePoint *proj, const G1Point *affine) {
  if (affine->infinity) {
    g1_projective_point_at_infinity_wrapper(proj);
    return;
  }
  proj->X = affine->x, proj->Y = affine->y;
  zk::fp_one(proj->Z);
}

void affine_to_projective_g2_wrapper(G2ProjectivePoint *proj, const G2Point *affine) {
  if (affine->infinity) {
    g2_projective_point_at_infinity_wrapper(proj);
    return;
  }
  proj->X = affine->x, proj->Y = affine->y;
  zk::fp_one(proj->Z);
}

void projective_to_affine_g1_wrapper(G1Point *affine, const G1ProjectivePoint *proj) {
  if (zk::fp_is_zero(proj->Z)) {
    g1_point_at_infinity_wrapper(affine);
    return;
  }
  Fp zi;
  zk::fp_inv(zi, proj->Z);
  zk::fp_mul(affine->x, proj->X, zi);
  zk::fp_mul(affine->y, proj->Y, zi);
  affine->infinity = false;
}

void projective_to_affine_g2_wrapper(G2Point *affine, const G2ProjectivePoint *proj) {
  if (zk::fp_is_zero(proj->Z)) {
    g2_point_at_infinity_wrapper(affine);
    return;
  }
  Fp2 zi;
  zk::fp_inv(zi, proj->Z);
  zk::fp_mul(affine->x, proj->X, zi);
  zk::fp_mul(affine->y, proj->Y, zi);
  affine->infinity = false;
}

void g1_point_at_infinity_wrapper(G1Point *point) {
  std::memset(point, 0, sizeof(*point));
  point->infinity = true;
}

void g2_point_at_infinity_wrapper(G2Point *point) {
  std::memset(point, 0, sizeof(*point));
  point->infinity = true;
}

void g1_projective_point_at_infinity_wrapper(G1ProjectivePoint *point) { std::memset(point, 0, sizeof(*point)); }

void g2_projective_point_at_infinity_wrapper(G2ProjectivePoint *point) { std::memset(point, 0, sizeof(*point)); }

bool g1_is_infinity_wrapper(const G1Point *point) { return point->infinity; }

bool g2_is_infinity_wrapper(const G2Point *point) { return point->infinity; }

void g1_msm_unmanaged_wrapper_async(cudaStream_t stream, uint32_t gpu_index, G1ProjectivePoint *h_result,
                                    const G1Point *d_points, const Scalar *d_scalars, uint32_t n,
                                    G1ProjectivePoint *d_scratch) {
  msm_unmanaged(stream, gpu_index, h_result, d_points, d_scalars, n, d_scratch);
}

void g2_msm_unmanaged_wrapper_async(cudaStream_t stream, uint32_t gpu_index, G2ProjectivePoint *h_result,
                                    const G2Point *d_points, const Scalar *d_scalars, uint32_t n,
                                    G2ProjectivePoint *d_scratch) {
  msm_unmanaged(stream, gpu_index, h_result, d_points, d_scalars, n, d_scratch);
}

size_t pippenger_scratch_size_g1_wrapper(uint32_t n, uint32_t gpu_index) {
  return msm_scratch_size<G1Point>(n, gpu_index);
}

size_t pippenger_scratch_size_g2_wrapper(uint32_t n, uint32_t gpu_index) {
  return msm_scratch_size<G2Point>(n, gpu_index);
}

void g1_msm_managed_wrapper(cudaStream_t stream, uint32_t gpu_index, G1ProjectivePoint *result,
                            const G1Point *points, const Scalar *scalars, uint32_t n, bool points_in_montgomery,
                            uint64_t *size_tracker) {
  msm_managed(stream, gpu_index, result, points, scalars, n, points_in_montgomery, size_tracker);
}

void g2_msm_managed_wrapper(cudaStream_t stream, uint32_t gpu_index, G2ProjectivePoint *result,
                            const G2Point *points, const Scalar *scalars, uint32_t n, bool points_in_montgomery,
                            uint64_t *size_tracker) {
  msm_managed(stream, gpu_index, result, points, scalars, n, points_in_montgomery, size_tracker);
}

void g1_from_montgomery_wrapper(G1Point *result, const G1Point *point) {
  B200_PANIC_IF_FALSE(result && point && result != point, "g1_from_montgomery: bad pointers");
  if (point->infinity) {
    g1_point_at_infinity_wrapper(result);
    return;
  }
  zk::fp_from_montgomery(result->x, point->x);
  zk::fp_from_montgomery(result->y, point->y);
  result->infinity = false;
}

void g2_from_montgomery_wrapper(G2Point *result, const G2Point *point) {
  B200_PANIC_IF_FALSE(result && point && result != point, "g2_from_montgomery: bad pointers");
  if (point->infinity) {
    g2_point_at_infinity_wrapper(result);
    return;
  }
  zk::fp_from_montgomery(result->x, point->x);
  zk::fp_from_montgomery(result->y, point->y);
  result->infinity = false;
}

void fp_to_montgomery_wrapper(Fp *result, const Fp *value) {
  B200_PANIC_IF_FALSE(result && value && result != value, "fp_to_montgomery: bad pointers");
  zk::fp_to_montgomery(*result, *value);
}

void fp_from_montgomery_wrapper(Fp *result, const Fp *value) {
  B200_PANIC_IF_FALSE(result && value && result != value, "fp_from_montgomery: bad pointers");
  zk::fp_from_montgomery(*result, *value);
}

void g1_projective_from_montgomery_normalized_wrapper(G1ProjectivePoint *result, const G1ProjectivePoint *point) {
  projective_normalized(result, point);
}

void g2_projective_from_montgomery_normalized_wrapper(G2ProjectivePoint *result, const G2ProjectivePoint *point) {
  projective_normalized(result, point);
}

bool is_on_curve_g1_wrapper(const G1Point *point) { return on_curve_normal(point); }

bool is_on_curve_g2_wrapper(const G2Point *point) { return on_curve_normal(point); }

void scalar_modulus_limbs_wrapper(uint64_t *limbs) {
  B200_PANIC_IF_FALSE(limbs != nullptr, "scalar_modulus_limbs: limbs is null");
  for (int i = 0; i < 5; i++)
    limbs[i] = zk::r_limb(i);
}

const char *b200_last_msm_config(void) { return t_last_msm_config; }

double b200_last_msm_combine_us(void) { return t_last_msm_combine_us; }

} // extern "C"
#pragma GCC visibility pop
