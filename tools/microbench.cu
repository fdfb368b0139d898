// Pipe-throughput microbenchmark for the integer-multiplier question behind the MSM roofline:
// how many IMAD / IMAD.WIDE / IMAD.HI / DFMA warp-instructions per clock per SM does H100 issue,
// and do DFMA and IMAD overlap?  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o microbench microbench.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#define ITER 4096
#define CHAINS 8

__global__ void k_imad_lo(uint32_t* out, uint32_t a, uint32_t b) {
  uint32_t x[CHAINS];
  for (int i = 0; i < CHAINS; i++) x[i] = threadIdx.x + i;
  for (int it = 0; it < ITER; it++)
#pragma unroll
    for (int i = 0; i < CHAINS; i++) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(x[i]) : "r"(a), "r"(b));
  uint32_t s = 0; for (int i = 0; i < CHAINS; i++) s += x[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void k_imad_hi(uint32_t* out, uint32_t a, uint32_t b) {
  uint32_t x[CHAINS];
  for (int i = 0; i < CHAINS; i++) x[i] = threadIdx.x + i + 0x80000000u;
  for (int it = 0; it < ITER; it++)
#pragma unroll
    for (int i = 0; i < CHAINS; i++) asm volatile("mad.hi.u32 %0, %0, %1, %2;" : "+r"(x[i]) : "r"(a), "r"(b));
  uint32_t s = 0; for (int i = 0; i < CHAINS; i++) s += x[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void k_imad_wide(uint32_t* out, uint32_t a, uint32_t b) {
  uint64_t x[CHAINS];
  for (int i = 0; i < CHAINS; i++) x[i] = threadIdx.x + i;
  for (int it = 0; it < ITER; it++)
#pragma unroll
    for (int i = 0; i < CHAINS; i++) {
      uint32_t lo = (uint32_t)x[i];
      asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(x[i]) : "r"(lo), "r"(a));
    }
  uint64_t s = 0; for (int i = 0; i < CHAINS; i++) s += x[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = (uint32_t)s ^ (uint32_t)(s >> 32) ^ b;
}
// the actual pattern in the field multiplication: mad.lo.cc / madc.hi.cc chains
__global__ void k_imad_chain(uint32_t* out, uint32_t a, uint32_t b) {
  uint32_t x[CHAINS];
  for (int i = 0; i < CHAINS; i++) x[i] = threadIdx.x + i;
  for (int it = 0; it < ITER; it++) {
    asm volatile("mad.lo.cc.u32 %0, %1, %2, %0;" : "+r"(x[0]) : "r"(a), "r"(b));
#pragma unroll
    for (int i = 1; i < CHAINS - 1; i += 2) {
      asm volatile("madc.hi.cc.u32 %0, %1, %2, %0;" : "+r"(x[i]) : "r"(a), "r"(b));
      asm volatile("madc.lo.cc.u32 %0, %1, %2, %0;" : "+r"(x[i + 1]) : "r"(a + i), "r"(b));
    }
    asm volatile("madc.hi.u32 %0, %1, %2, %0;" : "+r"(x[CHAINS - 1]) : "r"(a), "r"(b));
  }
  uint32_t s = 0; for (int i = 0; i < CHAINS; i++) s += x[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void k_dfma(uint32_t* out, double a, double b) {
  double x[CHAINS];
  for (int i = 0; i < CHAINS; i++) x[i] = threadIdx.x + i;
  for (int it = 0; it < ITER; it++)
#pragma unroll
    for (int i = 0; i < CHAINS; i++) asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(x[i]) : "d"(a), "d"(b));
  double s = 0; for (int i = 0; i < CHAINS; i++) s += x[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = (uint32_t)s;
}
__global__ void k_mix_dfma_imad(uint32_t* out, double a, double b, uint32_t ia, uint32_t ib) {
  double x[CHAINS]; uint64_t y[CHAINS];
  for (int i = 0; i < CHAINS; i++) { x[i] = threadIdx.x + i; y[i] = threadIdx.x + i; }
  for (int it = 0; it < ITER; it++)
#pragma unroll
    for (int i = 0; i < CHAINS; i++) {
      asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(x[i]) : "d"(a), "d"(b));
      uint32_t lo = (uint32_t)y[i];
      asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(y[i]) : "r"(lo), "r"(ia));
    }
  double s = 0; uint64_t t = 0; for (int i = 0; i < CHAINS; i++) { s += x[i]; t += y[i]; }
  out[blockIdx.x * blockDim.x + threadIdx.x] = (uint32_t)s + (uint32_t)t + ib;
}
__global__ void k_iadd3(uint32_t* out, uint32_t a, uint32_t b) {
  uint32_t x[CHAINS];
  for (int i = 0; i < CHAINS; i++) x[i] = threadIdx.x + i;
  for (int it = 0; it < ITER; it++)
#pragma unroll
    for (int i = 0; i < CHAINS; i++) asm volatile("add.u32 %0, %0, %1;" : "+r"(x[i]) : "r"(a));
  uint32_t s = b; for (int i = 0; i < CHAINS; i++) s += x[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <class F> float timeit(F f) {
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  f(); cudaDeviceSynchronize();
  cudaEventRecord(e0); f(); cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1); return ms;
}

int main() {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  int sms = p.multiProcessorCount;
  int clk_khz = 0; cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
  printf("device %s, %d SMs, nominal %d MHz\n", p.name, sms, clk_khz / 1000);
  uint32_t* out; cudaMalloc(&out, (size_t)sms * 8 * 1024 * 4);
  for (int warps_per_sm : {4, 8, 16, 32}) {
    int threads = 256, blocks = sms * warps_per_sm * 32 / threads;
    double ops = (double)blocks * threads * ITER * CHAINS;  // lane-ops
    auto rep = [&](const char* name, float ms, double per_iter) {
      double lane_per_s = ops * per_iter / (ms * 1e-3);
      printf("  %-22s warps/SM=%2d  %8.3f ms  %7.2f Tlane-op/s  = %6.1f lane-op/clk/SM at the nominal clock\n", name,
             warps_per_sm, ms, lane_per_s / 1e12, lane_per_s / sms / (clk_khz * 1e3));
    };
    rep("IMAD lo", timeit([&] { k_imad_lo<<<blocks, threads>>>(out, 3, 5); }), 1);
    rep("IMAD.HI", timeit([&] { k_imad_hi<<<blocks, threads>>>(out, 3, 5); }), 1);
    rep("IMAD.WIDE", timeit([&] { k_imad_wide<<<blocks, threads>>>(out, 3, 5); }), 1);
    rep("mad.lo/hi.cc chain", timeit([&] { k_imad_chain<<<blocks, threads>>>(out, 3, 5); }), 1);
    rep("DFMA", timeit([&] { k_dfma<<<blocks, threads>>>(out, 1.0000001, 0.5); }), 1);
    rep("DFMA+IMAD.WIDE (each)", timeit([&] { k_mix_dfma_imad<<<blocks, threads>>>(out, 1.0000001, 0.5, 3, 5); }), 1);
    rep("IADD", timeit([&] { k_iadd3<<<blocks, threads>>>(out, 3, 5); }), 1);
  }
  return 0;
}
