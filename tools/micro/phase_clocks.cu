// tools/micro/phase_clocks.cu -- where do the cycles of ONE CMUX step go?
// Runs the blind-rotation loop of the shipped two-CTA N = 2048 instance
// (pbs_n2048_k1_l1_v6_kernel<2, true, 2, 1>, lane-pair layout) -- the kernel's
// own p22_lanepair_loop, with a probe that reads clock64() between phases --
// for exchange 2 through the warp's own rows (x2m_*, X2 = 1, the shipped one)
// and through half-warp shuffles (x2h_*, X2 = 0), on a synthetic accumulator
// and mask.  Every SM runs 1 or 2 CTAs; the tool prints the average cycles per
// phase of warp 0 of CTA 0.  The clock reads order the phases of a warp, so the
// sum is a little above the step time of the kernel.  Measurement tool only
// (not part of the library).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I../../tfhe-rs_b200/csrc -o phase_clocks phase_clocks.cu
//   ./phase_clocks <CTAs per SM: 1 or 2>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "pbs_n2048.cuh"
using namespace b200;

#define NPH 16
__device__ __forceinline__ long long clk() {
  long long c;
  asm volatile("mov.u64 %0, %%clock64;" : "=l"(c)::"memory");
  return c;
}

// cycles per phase, summed over the steps: 32-bit sums (918 steps of a few
// thousand cycles) keep the loop free of spills
struct ClockProbe {
  uint32_t acc[NPH] = {};
  long long t0;
  __device__ __forceinline__ void begin() { t0 = clk(); }
  __device__ __forceinline__ void lap(int p) {
    const long long t1 = clk();
    acc[p] += (uint32_t)(t1 - t0);
    t0 = t1;
  }
};

template <int X2>
__global__ void __launch_bounds__(128, 2)
timed_lanepair(const cplx *__restrict__ bsk, const Fft1024Tables *__restrict__ tables,
               uint32_t n, uint32_t base_log, unsigned long long *out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using Smem = P22SmemV6<2, true>;
  Smem &sm = *reinterpret_cast<Smem *>(smem_raw);
  const int tid = threadIdx.x;
  const int t = p22lp_t(tid);
  if (tid == 0) { mbar_init(&sm.bar, 1); mbar_fence_init(); }
  for (uint32_t i = tid; i < n + 8; i += 128)
    sm.a_hat[i] = (uint16_t)(1 + ((i * 2654435761u + blockIdx.x * 40503u) % 4095u));
  for (uint32_t j = tid; j < 2 * P22_N; j += 128)
    sm.acc[j >> 11][j & (P22_N - 1)] = j * 2654435761u + blockIdx.x;
  cplx tw2[3], tw3[15];
#pragma unroll
  for (int e = 0; e < 3; e++) tw2[e] = tables->pass2[x1h_q(t)][e];
#pragma unroll
  for (int e = 0; e < 15; e++) tw3[e] = tables->pass3[t][e];
  __syncthreads();
  if (tid == 0) p22_ring_issue(&sm.ring[0][0], &sm.bar, bsk, 0);
  __syncthreads();
  ClockProbe probe;
  p22_lanepair_loop<X2>(sm, bsk, n, base_log, tw2, tw3, probe);
  if (tid == 0 && blockIdx.x == 0)
    for (int p = 0; p < NPH; p++) out[p] = (unsigned long long)probe.acc[p];
  if (sm.acc[0][tid] == 0x12345678u) out[NPH] = 1; // keep results live
}

template <int X2>
static int run(const char *label, int ctas, int sms, const cplx *bsk, const Fft1024Tables *dt, uint32_t n,
               unsigned long long *out) {
  const int smem = (int)sizeof(P22SmemV6<2, true>);
  cudaFuncSetAttribute(timed_lanepair<X2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  for (int rep = 0; rep < 2; rep++) {
    timed_lanepair<X2><<<ctas * sms, 128, smem>>>(bsk, dt, n, 23, out);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return 1; }
  }
  unsigned long long h[NPH + 1];
  cudaMemcpy(h, out, sizeof(h), cudaMemcpyDeviceToHost);
  const char *names[14] = {"digits (rotate + decompose)", "fwd pass 1", "exchange 1 (+ CTA barrier)", "fwd pass 2",
                           "exchange 2", "fwd pass 3", "own-row key load + key wait", "MAC", "inv pass 3",
                           "inv exchange 2", "inv pass 2", "inv exchange 1 (+ CTA barrier, TMA issue)", "inv pass 1",
                           "accumulator update (+ CTA barrier)"};
  unsigned long long tot = 0;
  for (int p = 0; p < 14; p++) tot += h[p];
  printf("%s, %d CTA(s) per SM: %.0f cycles per CMUX step (warp 0 of CTA 0)\n", label, ctas, (double)tot / n);
  for (int p = 0; p < 14; p++) printf("  %-44s %7.0f  %5.1f %%\n", names[p], (double)h[p] / n, 100.0 * h[p] / tot);
  return 0;
}

int main(int argc, char **argv) {
  const uint32_t n = 918;
  const int ctas = argc > 1 ? atoi(argv[1]) : 2;
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  Fft1024Tables *host = new Fft1024Tables;
  b200_fill_fft1024_tables(host);
  Fft1024Tables *dt;
  cudaMalloc(&dt, sizeof(*host));
  cudaMemcpy(dt, host, sizeof(*host), cudaMemcpyHostToDevice);
  cudaMemcpyToSymbol(c_fft1024_pass1, host->pass1, sizeof(host->pass1));
  const size_t words = (size_t)n * 4 * P22_M;
  std::vector<cplx> h(words);
  for (size_t i = 0; i < words; i++) { h[i].re = 1e-9 * (double)((i * 2654435761u) % 1000); h[i].im = -h[i].re; }
  cplx *bsk; cudaMalloc(&bsk, words * sizeof(cplx));
  cudaMemcpy(bsk, h.data(), words * sizeof(cplx), cudaMemcpyHostToDevice);
  unsigned long long *out; cudaMalloc(&out, (NPH + 1) * 8); cudaMemset(out, 0, (NPH + 1) * 8);
  if (run<0>("lane-pair, exchange 2 through half-warp shuffles (x2h)", ctas, sms, bsk, dt, n, out)) return 1;
  if (run<1>("lane-pair, exchange 2 through the warp's rows (x2m)", ctas, sms, bsk, dt, n, out)) return 1;
  return 0;
}
