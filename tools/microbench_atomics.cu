// Micro-benchmark for a counting-sort front of the MSM (the question: can 2 x 16.7 M global atomics on 32 K counters
// beat the two CUB onesweep passes?).  m entries with pseudo-random 15-bit keys:
//   (a) histogram: red.global.add on hist[key]                       (no return value)
//   (b) scatter:   pos = atomicAdd(&cursor[key], 1); out[pos] = val  (return value + scattered 4-byte store)
//   (c) the same two with every key equal (fully skewed input)
//   (d) block-local shared-memory histogram of 32 K bins (128 KB) flushed with global reds
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o build/microbench_atomics tools/microbench_atomics.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t mix(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}

__global__ void k_hist(uint32_t m, uint32_t nb_mask, int skew, uint32_t* hist) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const uint32_t key = skew ? (i & 15u) : (mix(i) & nb_mask);
  atomicAdd(hist + key, 1u);
}

__global__ void k_scatter(uint32_t m, uint32_t nb_mask, int skew, uint32_t* cursor, uint32_t* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const uint32_t key = skew ? (i & 15u) : (mix(i) & nb_mask);
  const uint32_t pos = atomicAdd(cursor + key, 1u);
  out[pos] = i;
}

__global__ void __launch_bounds__(1024) k_hist_smem(uint32_t m, uint32_t nb, uint32_t* hist) {
  extern __shared__ uint32_t sh[];
  for (uint32_t k = threadIdx.x; k < nb; k += blockDim.x) sh[k] = 0;
  __syncthreads();
  const uint32_t per = (m + gridDim.x - 1) / gridDim.x;
  const uint32_t lo = blockIdx.x * per, hi = min(m, lo + per);
  for (uint32_t i = lo + threadIdx.x; i < hi; i += blockDim.x) atomicAdd(sh + (mix(i) & (nb - 1)), 1u);
  __syncthreads();
  for (uint32_t k = threadIdx.x; k < nb; k += blockDim.x)
    if (sh[k]) atomicAdd(hist + k, sh[k]);
}

int main() {
  const uint32_t m = 16u << 20, nb = 1u << 15;
  uint32_t *hist, *cursor, *out;
  cudaMalloc(&hist, nb * 4); cudaMalloc(&cursor, nb * 4); cudaMalloc(&out, (size_t)m * 4);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  auto timeit = [&](const char* what, auto fn) {
    float best = 1e9f;
    for (int r = 0; r < 5; r++) {
      cudaMemset(hist, 0, nb * 4);
      fn(true);                                   // prepare (untimed)
      cudaDeviceSynchronize();
      cudaEventRecord(e0);
      fn(false);
      cudaEventRecord(e1);
      cudaEventSynchronize(e1);
      float ms; cudaEventElapsedTime(&ms, e0, e1);
      if (ms < best) best = ms;
    }
    printf("%-58s %8.3f ms\n", what, best);
  };
  const uint32_t blocks = (m + 255) / 256;
  // cursor = exclusive offsets of a uniform distribution (m / nb per bucket) so that scatter writes stay in range
  uint32_t* h = new uint32_t[nb];
  auto set_cursor = [&](int skew) {
    if (skew) { for (uint32_t k = 0; k < nb; k++) h[k] = k < 16 ? k * (m / 16) : 0; }
    else {
      // exact counts of mix() keys
      uint32_t* cnt = new uint32_t[nb]();
      for (uint32_t i = 0; i < m; i++) { uint32_t x = i; x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16; cnt[x & (nb - 1)]++; }
      uint32_t acc = 0;
      for (uint32_t k = 0; k < nb; k++) { h[k] = acc; acc += cnt[k]; }
      delete[] cnt;
    }
    cudaMemcpy(cursor, h, nb * 4, cudaMemcpyHostToDevice);
  };
  for (int skew = 0; skew < 2; skew++) {
    timeit(skew ? "(c) histogram, 16 distinct keys" : "(a) histogram, 16.7 M reds on 32 K counters",
           [&](bool prep) { if (!prep) k_hist<<<blocks, 256>>>(m, nb - 1, skew, hist); });
    timeit(skew ? "(c) scatter, 16 distinct keys" : "(b) scatter, 16.7 M atomics with return + 4-byte stores",
           [&](bool prep) { if (prep) set_cursor(skew); else k_scatter<<<blocks, 256>>>(m, nb - 1, skew, cursor, out); });
  }
  cudaFuncSetAttribute(k_hist_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(nb * 4));
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  for (int g : {sms, 2 * sms}) {
    char what[96]; snprintf(what, sizeof(what), "(d) shared-memory histogram, %d blocks x 1024 threads + flush", g);
    timeit(what, [&](bool prep) { if (!prep) k_hist_smem<<<g, 1024, nb * 4>>>(m, nb, hist); });
  }
  cudaError_t e = cudaDeviceSynchronize();
  printf("status: %s\n", cudaGetErrorString(e));
  return e != cudaSuccess;
}
