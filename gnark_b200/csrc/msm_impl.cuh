// sm_90a kernels + stream-ordered host driver for the bucket MSM (see msm.cuh for
// the algorithm and the reference call sites it replaces).
#pragma once
#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include "internal.h"
#include "msm.cuh"
#include "points_decode.cuh"

namespace gb200 {

#define GB_CUDA_TRY(x)                                   \
  do {                                                   \
    cudaError_t e_ = (x);                                \
    if (e_ != cudaSuccess) return e_;                    \
  } while (0)

// ---------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------
// idx: null (bases table_off + i) or the checked index list of an indexed MSM (bases idx[i])
template <class Fr>
__global__ void __launch_bounds__(256) k_msm_decompose(MsmPlan pl, const Fr* __restrict__ scalars,
                                                       uint32_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                       const uint32_t* __restrict__ idx) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < pl.n) msm_decompose_one<Fr>(pl, i, scalars, keys, vals, idx);
}

// batched MSM: one thread per (item, scalar), entry g = b * n + i.  kStrided = false: the items' scalars are back to back
// (scalar_stride = n), the index folds to g and the kernel keeps the registers of the unstrided read
template <class Fr, bool kStrided>
__global__ void __launch_bounds__(256) k_msm_decompose_batch(MsmPlan pl, const Fr* __restrict__ scalars,
                                                             uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (!kStrided) pl.scalar_stride = pl.n;
  if (g < pl.n * pl.batch) msm_decompose_batch_one<Fr>(pl, g, scalars, keys, vals);
}

// off[b] = first sorted position with key >= b, for b in [0, nb]
static __global__ void k_msm_bucket_offsets(const uint32_t* __restrict__ skeys, uint32_t m, uint32_t nb,
                                     uint32_t* __restrict__ off) {
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > nb) return;
  uint32_t lo = 0, hi = m;
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(skeys + mid) < b) lo = mid + 1; else hi = mid;
  }
  off[b] = lo;
}

static __global__ void k_msm_task_counts(const uint32_t* __restrict__ off, uint32_t nb, uint32_t task_len,
                                  uint32_t* __restrict__ ntasks) {
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > nb) return;
  ntasks[b] = b == nb ? 0u : (off[b + 1] - off[b] + task_len - 1) / task_len;
}

// one thread per task: partial[t] = sum of <= task_len consecutive entries of one bucket
// Resident blocks per SM asked of ptxas (register cap 65536 / (128 k)); 1 = the compiler's own allocation.
// 64-byte coordinates (Fp2 over 8 limbs, BN254 G2): left alone ptxas takes over 200 registers = 2 blocks / SM; capped at
// 168 registers (3 blocks / SM) a few spills buy a third resident block, which keeps the IMAD pipe busier while
// one block waits on its gathers.  96-byte coordinates (Fp2 over 12 limbs, BW6-761 Fp) already spill at 255
// registers = 2 blocks / SM and are left alone.
#ifndef GB200_ACC_MIN_BLOCKS_64
#define GB200_ACC_MIN_BLOCKS_64 3
#endif
template <class F>
__global__ void __launch_bounds__(128, sizeof(F) == 64 ? GB200_ACC_MIN_BLOCKS_64 : 1) k_msm_accumulate(MsmPlan pl, const Affine<F>* __restrict__ table,
                                                        const uint32_t* __restrict__ svals,
                                                        const uint32_t* __restrict__ off,
                                                        const uint32_t* __restrict__ task_off,
                                                        XYZZ<F>* __restrict__ partial) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t nb = pl.total_buckets;
  if (t >= __ldg(task_off + nb)) return;
  // bucket of task t: largest b with task_off[b] <= t
  uint32_t lo = 0, hi = nb;
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo + 1) >> 1);
    if (__ldg(task_off + mid) <= t) lo = mid; else hi = mid - 1;
  }
  const uint32_t b = lo;
  const uint32_t j = t - __ldg(task_off + b);
  const uint32_t begin = __ldg(off + b) + j * pl.task_len;
  uint32_t end = begin + pl.task_len;
  const uint32_t bend = __ldg(off + b + 1);
  if (end > bend) end = bend;
  partial[t] = msm_accumulate_range<F>(table, svals, begin, end);
}

// one thread per bucket: sum of its task partials.  Buckets with more than MSM_HEAVY partials
// (skewed witnesses: many equal small scalars; a short top window) are queued for the
// block-cooperative kernel below instead of being summed serially.
constexpr uint32_t MSM_HEAVY = 48;   // below this a single thread's serial sum beats the warp tree (measured)
template <class F>
__global__ void __launch_bounds__(128) k_msm_combine(MsmPlan pl, const uint32_t* __restrict__ task_off,
                                                     const XYZZ<F>* __restrict__ partial,
                                                     XYZZ<F>* __restrict__ buckets, uint32_t* __restrict__ heavy_count,
                                                     uint32_t* __restrict__ heavy_list) {
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= pl.total_buckets) return;
  const uint32_t t0 = task_off[b], t1 = task_off[b + 1];
  if (t1 - t0 > MSM_HEAVY) {
    heavy_list[atomicAdd(heavy_count, 1u)] = b;
    return;
  }
  XYZZ<F> acc = XYZZ<F>::inf();
  if (t0 < t1) acc = partial[t0];
  for (uint32_t t = t0 + 1; t < t1; t++) acc.add(partial[t]);
  buckets[b] = acc;
}

// one WARP per heavy bucket (grid-stride over the queue): lanes stride the partials, then a
// 5-level tree through shared memory
template <class F>
__global__ void __launch_bounds__(128) k_msm_combine_heavy(const uint32_t* __restrict__ task_off,
                                                           const XYZZ<F>* __restrict__ partial,
                                                           XYZZ<F>* __restrict__ buckets,
                                                           const uint32_t* __restrict__ heavy_count,
                                                           const uint32_t* __restrict__ heavy_list) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  XYZZ<F>* sm = reinterpret_cast<XYZZ<F>*>(smem_raw) + (threadIdx.x & ~31u);
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warps_per_block = blockDim.x >> 5;
  const uint32_t warp = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  const uint32_t nwarps = gridDim.x * warps_per_block;
  const uint32_t nh = *heavy_count;
  for (uint32_t i = warp; i < nh; i += nwarps) {
    const uint32_t b = heavy_list[i];
    const uint32_t t0 = task_off[b], t1 = task_off[b + 1];
    XYZZ<F> acc = XYZZ<F>::inf();
    for (uint32_t t = t0 + lane; t < t1; t += 32) acc.add(partial[t]);
    sm[lane] = acc;
    __syncwarp();
    for (uint32_t w = 16; w > 0; w >>= 1) {
      if (lane < w) {
        XYZZ<F> a = sm[lane];
        a.add(sm[lane + w]);
        sm[lane] = a;
      }
      __syncwarp();
    }
    if (lane == 0) buckets[b] = sm[0];
    __syncwarp();
  }
}

// one thread per (set, chunk): weighted running sum of `chunk` buckets
template <class F>
__global__ void __launch_bounds__(128) k_msm_reduce_chunks(MsmPlan pl, uint32_t chunks_per_set,
                                                           const XYZZ<F>* __restrict__ buckets,
                                                           XYZZ<F>* __restrict__ chunk_sums) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= chunks_per_set * (uint32_t)pl.nsets) return;
  const uint32_t s = g / chunks_per_set, t = g % chunks_per_set;
  const uint32_t lo = t * pl.chunk;
  uint32_t hi = lo + pl.chunk;
  if (hi > pl.set_size) hi = pl.set_size;
  chunk_sums[g] = msm_reduce_chunk<F>(buckets + (size_t)s * pl.set_size, lo, hi);
}

// The tail is a chain of dependent point additions (microseconds each on an otherwise idle SM), so its cost is its DEPTH: the
// chunk sums of a set are added as a pure tree - block (slice, set) reduces one slice of them in shared memory, one entry
// per thread where the slice allows, k_msm_finish adds the slice sums - 12 levels for 4096 chunk sums.
template <class F>
__global__ void __launch_bounds__(256) k_msm_set_sum(uint32_t chunks_per_set, const XYZZ<F>* __restrict__ chunk_sums,
                              XYZZ<F>* __restrict__ slice_sums) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  XYZZ<F>* sm = reinterpret_cast<XYZZ<F>*>(smem_raw);
  const uint32_t s = blockIdx.y, slices = gridDim.x;
  const uint32_t per = (chunks_per_set + slices - 1) / slices;
  const uint32_t lo = blockIdx.x * per;
  const uint32_t hi = lo + per < chunks_per_set ? lo + per : chunks_per_set;
  const XYZZ<F>* src = chunk_sums + (size_t)s * chunks_per_set;
  XYZZ<F> acc = XYZZ<F>::inf();
  for (uint32_t k = lo + threadIdx.x; k < hi; k += blockDim.x) acc.add(src[k]);
  sm[threadIdx.x] = acc;
  __syncthreads();
  for (uint32_t w = blockDim.x >> 1; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      XYZZ<F> a = sm[threadIdx.x];
      a.add(sm[threadIdx.x + w]);
      sm[threadIdx.x] = a;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) slice_sums[(size_t)s * slices + blockIdx.x] = sm[0];
}

// slice sums -> set sums (warp w takes sets w, w + warps, ...: a 5-level tree over at most 32 slices), then Horner over
// the sets on one thread; result in gnark Jacobian layout.  set_totals: nsets entries of scratch (per block).
// kBatch: block b finishes MSM b of a batch - its nsets sets follow those of the blocks before it, it writes out[b] - so the
// items' Horner sums run in parallel.  A single MSM takes the other instantiation, which carries no item offsets (its
// registers are at the 255 cap on the wide curves, and the offsets would add spills).
template <class F, bool kBatch>
__global__ void __launch_bounds__(256) k_msm_finish(int nsets, int c, uint32_t slices, const XYZZ<F>* __restrict__ slice_sums,
                                                    XYZZ<F>* __restrict__ set_totals, Jacobian<F>* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  if (kBatch) {
    slice_sums += (size_t)blockIdx.x * nsets * slices;
    set_totals += (size_t)blockIdx.x * nsets;
    out += blockIdx.x;
  }
  XYZZ<F>* sm = reinterpret_cast<XYZZ<F>*>(smem_raw) + (threadIdx.x & ~31u);
  const uint32_t lane = threadIdx.x & 31u;
  for (int s = (int)(threadIdx.x >> 5); s < nsets; s += (int)(blockDim.x >> 5)) {
    sm[lane] = lane < slices ? slice_sums[(size_t)s * slices + lane] : XYZZ<F>::inf();
    __syncwarp();
    for (uint32_t w = 16; w > 0; w >>= 1) {
      if (lane < w && lane + w < slices) {
        XYZZ<F> a = sm[lane];
        a.add(sm[lane + w]);
        sm[lane] = a;
      }
      __syncwarp();
    }
    if (lane == 0) set_totals[s] = sm[0];
    __syncwarp();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    XYZZ<F> r = nsets > 0 ? msm_horner<F>(set_totals, nsets, c) : XYZZ<F>::inf();
    *out = r.to_jacobian();
  }
}

// Multi-GPU combine (SURVEY.md 8e; the reference sums its chunk results on the host, icicle.go:383-411): gathered holds
// `world` rows of `count` Jacobian points (row r = rank r's partial results, the layout ncclAllGather produces);
// out[k] = sum over ranks of gathered[r][k].  One thread per result point: the world-1 additions of one point are
// serial anyway, and `count` is the number of MSMs folded at once (5 for a Groth16 proof, K for a stream of MSMs).
template <class F>
__global__ void __launch_bounds__(64) k_points_fold(const Jacobian<F>* __restrict__ gathered, uint32_t world, uint32_t count,
                                                    Jacobian<F>* __restrict__ out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  XYZZ<F> acc = XYZZ<F>::from_jacobian(gathered[k]);
  for (uint32_t r = 1; r < world; r++) acc.add(XYZZ<F>::from_jacobian(gathered[(size_t)r * count + k]));
  out[k] = acc.to_jacobian();
}

// one thread per point of a serialised slice (points_decode.cuh); status[0] = first non-zero DECODE_* code seen,
// status[1] = index of a point that failed
template <class F, class FB>
__global__ void __launch_bounds__(128) k_points_decode(const uint8_t* __restrict__ bytes, size_t n, size_t stride, int compressed,
                                                       DecodeConsts<FB> k, Affine<F>* __restrict__ out,
                                                       uint32_t* __restrict__ status) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<F> a = Affine<F>::inf();
  const int rc = decode_point<F, FB>(bytes + i * stride, compressed, k, a);
  out[i] = a;
  if (rc != DECODE_OK && atomicCAS(status, 0u, (uint32_t)rc) == 0u) status[1] = (uint32_t)i;
}

// table precompute (built once per table upload): slab w holds 2^(c*w) * P_i.
// pass 1: doubling chains, XYZZ results to a scratch buffer [w-1][chunk];
// pass 2: one inversion per point (Montgomery's trick over its nwin-1 outputs), affine results.
constexpr int MSM_MAX_WINDOWS = 64;
template <class F>
__global__ void __launch_bounds__(128) k_msm_precompute_dbl(uint32_t cnt, int nwin, int c, const Affine<F>* __restrict__ src,
                                                            XYZZ<F>* __restrict__ tmp) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cnt) return;
  XYZZ<F> q = XYZZ<F>::from_affine(src[i]);
  for (int w = 1; w < nwin; w++) {
    for (int k = 0; k < c; k++) q.dbl();
    tmp[(size_t)(w - 1) * cnt + i] = q;
  }
}
template <class F>
__global__ void __launch_bounds__(128) k_msm_precompute_affine(uint32_t cnt, uint32_t n, uint32_t first, int nwin,
                                                               const Affine<F>* __restrict__ src,
                                                               const XYZZ<F>* __restrict__ tmp, Affine<F>* __restrict__ table) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cnt) return;
  table[first + i] = src[i];
  F pre[MSM_MAX_WINDOWS];
  F acc = F::one();
  for (int w = 1; w < nwin; w++) {
    pre[w] = acc;
    const F zzz = tmp[(size_t)(w - 1) * cnt + i].zzz;
    if (!zzz.is_zero()) acc = acc * zzz;
  }
  F inv = acc.inverse();
  for (int w = nwin - 1; w >= 1; w--) {
    const XYZZ<F> q = tmp[(size_t)(w - 1) * cnt + i];
    Affine<F> a = Affine<F>::inf();
    if (!q.zzz.is_zero()) {
      const F zi3 = inv * pre[w];       // 1 / zzz_w
      inv = inv * q.zzz;
      const F zi2 = (zi3 * q.zz).sqr(); // (zz/zzz)^2 = 1 / zz
      a.x = q.x * zi2;
      a.y = q.y * zi3;
    }
    table[(size_t)w * n + first + i] = a;
  }
}

// d_src: n affine points (may be slab 0 of d_table itself); d_table: [nwin][n] affine points
template <class F>
cudaError_t msm_precompute_enqueue(cudaStream_t st, uint32_t n, int nwin, int c, const Affine<F>* d_src, Affine<F>* d_table) {
  if (n == 0) return cudaSuccess;
  if (nwin > MSM_MAX_WINDOWS) return cudaErrorInvalidValue;
  const uint32_t chunk = n < (1u << 18) ? n : (1u << 18);
  XYZZ<F>* tmp = nullptr;
  if (nwin > 1) GB_CUDA_TRY(cudaMallocAsync(&tmp, (size_t)(nwin - 1) * chunk * sizeof(XYZZ<F>), st));
  for (uint32_t first = 0; first < n; first += chunk) {
    const uint32_t cnt = n - first < chunk ? n - first : chunk;
    if (nwin > 1) k_msm_precompute_dbl<F><<<(cnt + 127) / 128, 128, 0, st>>>(cnt, nwin, c, d_src + first, tmp);
    k_msm_precompute_affine<F><<<(cnt + 127) / 128, 128, 0, st>>>(cnt, n, first, nwin, d_src + first, tmp, d_table);
  }
  GB_CUDA_TRY(cudaGetLastError());
  if (tmp) GB_CUDA_TRY(cudaFreeAsync(tmp, st));
  return cudaSuccess;
}

// ---------------------------------------------------------------------------
// workspace + driver
// ---------------------------------------------------------------------------
constexpr int MSM_NUM_EVENTS = 8;
constexpr uint32_t MSM_SET_SLICES = 32;   // upper bound of the blocks k_msm_set_sum spends on one bucket set
template <class F>
struct MsmLayout {
  size_t m;            // entries
  size_t max_tasks;
  uint32_t chunks_per_set;
  size_t cub_bytes;
  // offsets into the workspace
  size_t o_keys0, o_keys1, o_vals0, o_vals1, o_off, o_ntasks, o_task_off, o_partial, o_buckets, o_chunks, o_sets, o_heavy, o_cub, total;
};

inline size_t gb_align(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

template <class F>
cudaError_t msm_layout(const MsmPlan& pl, MsmLayout<F>& L) {
  L.m = (size_t)pl.n * pl.batch * pl.nwin;
  L.max_tasks = L.m / pl.task_len + pl.total_buckets + 1;
  L.chunks_per_set = (pl.set_size + pl.chunk - 1) / pl.chunk;
  size_t sort_bytes = 0, scan_bytes = 0;
  int end_bit = 1;
  while ((1ull << end_bit) <= pl.total_buckets) end_bit++;
  GB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                              (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)L.m, 0, end_bit));
  GB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                            (int)pl.total_buckets + 1));
  L.cub_bytes = sort_bytes > scan_bytes ? sort_bytes : scan_bytes;
  size_t o = 0;
  L.o_keys0 = o; o += gb_align(L.m * 4);
  L.o_keys1 = o; o += gb_align(L.m * 4);
  L.o_vals0 = o; o += gb_align(L.m * 4);
  L.o_vals1 = o; o += gb_align(L.m * 4);
  L.o_off = o; o += gb_align(((size_t)pl.total_buckets + 2) * 4);
  L.o_ntasks = o; o += gb_align(((size_t)pl.total_buckets + 2) * 4);
  L.o_task_off = o; o += gb_align(((size_t)pl.total_buckets + 2) * 4);
  L.o_partial = o; o += gb_align(L.max_tasks * sizeof(XYZZ<F>));
  L.o_buckets = o; o += gb_align((size_t)pl.total_buckets * sizeof(XYZZ<F>));
  L.o_chunks = o; o += gb_align((size_t)L.chunks_per_set * pl.nsets * sizeof(XYZZ<F>));
  L.o_sets = o; o += gb_align((size_t)pl.nsets * (MSM_SET_SLICES + 1) * sizeof(XYZZ<F>));   // slice sums, then set totals
  L.o_heavy = o; o += gb_align((L.max_tasks / MSM_HEAVY + 2) * 4);  // [0] = count, [1..] = bucket ids
  L.o_cub = o; o += gb_align(L.cub_bytes);
  L.total = o;
  return cudaSuccess;
}

// largest power-of-two block that fits `budget` bytes of XYZZ<F> in shared memory
template <class F>
inline int msm_set_sum_threads(size_t budget = 160 * 1024) {
  int t = 256;  // __launch_bounds__ of k_msm_set_sum (register budget: up to 255 regs/thread)
  while ((size_t)t * sizeof(XYZZ<F>) > budget) t >>= 1;
  return t;
}

// Enqueue a full MSM on `stream`.  d_scalars: n Fr elements (Montgomery) on device; batch * n, item-major, for a plan of
// msm_make_batch_plan.  d_out: one Jacobian<F> on device per item.  ws must hold msm_layout().total bytes.  d_idx
// (optional, single MSMs only): n checked table indices, scalar i then multiplies base d_idx[i] instead of base table_off + i.
template <class Fr, class F>
cudaError_t msm_enqueue(cudaStream_t stream, const MsmPlan& pl, const Affine<F>* d_table, const Fr* d_scalars,
                        Jacobian<F>* d_out, void* ws, const MsmLayout<F>& L, cudaEvent_t* ev = nullptr,
                        const MsmPipe* pipe = nullptr, const uint32_t* d_idx = nullptr) {
  // pipe (optional, internal.h): the accumulate kernel and the latency-bound reduction kernels that follow it are
  // enqueued on their own streams (forked with events), so that in a pipeline of MSMs the next MSM's DRAM-bound
  // front overlaps this one's multiplier-bound accumulate, and the tail overlaps both instead of idling most of the SMs.
  // ev (optional, MSM_NUM_EVENTS entries): stage boundaries for the step profile
  // (the reference's ICICLE_STEP_PROFILE timers, icicle.go:72-75,1088-1094)
#define GB_EV(k) do { if (ev) GB_CUDA_TRY(cudaEventRecord(ev[k], stream)); } while (0)
  unsigned char* w = reinterpret_cast<unsigned char*>(ws);
  uint32_t* keys0 = (uint32_t*)(w + L.o_keys0);
  uint32_t* keys1 = (uint32_t*)(w + L.o_keys1);
  uint32_t* vals0 = (uint32_t*)(w + L.o_vals0);
  uint32_t* vals1 = (uint32_t*)(w + L.o_vals1);
  uint32_t* off = (uint32_t*)(w + L.o_off);
  uint32_t* ntasks = (uint32_t*)(w + L.o_ntasks);
  uint32_t* task_off = (uint32_t*)(w + L.o_task_off);
  XYZZ<F>* partial = (XYZZ<F>*)(w + L.o_partial);
  XYZZ<F>* buckets = (XYZZ<F>*)(w + L.o_buckets);
  XYZZ<F>* chunks = (XYZZ<F>*)(w + L.o_chunks);
  XYZZ<F>* sets = (XYZZ<F>*)(w + L.o_sets);
  void* cub_tmp = w + L.o_cub;
  size_t cub_bytes = L.cub_bytes;
  const uint32_t nb = pl.total_buckets;

  if (pl.n == 0) {
    // empty sum = infinity
    // nsets = 0: the point at infinity
    if (pl.batch > 1) k_msm_finish<F, true><<<pl.batch, 32, 32 * sizeof(XYZZ<F>), stream>>>(0, pl.c, 1, sets, sets, d_out);
    else k_msm_finish<F, false><<<1, 32, 32 * sizeof(XYZZ<F>), stream>>>(0, pl.c, 1, sets, sets, d_out);
    return cudaGetLastError();
  }
  GB_EV(0);
  if (pl.batch > 1 && pl.scalar_stride != pl.n)
    k_msm_decompose_batch<Fr, true><<<(unsigned)((L.m / pl.nwin + 255) / 256), 256, 0, stream>>>(pl, d_scalars, keys0, vals0);
  else if (pl.batch > 1)
    k_msm_decompose_batch<Fr, false><<<(unsigned)((L.m / pl.nwin + 255) / 256), 256, 0, stream>>>(pl, d_scalars, keys0, vals0);
  else
    k_msm_decompose<Fr><<<(pl.n + 255) / 256, 256, 0, stream>>>(pl, d_scalars, keys0, vals0, d_idx);
  GB_EV(1);
  int end_bit = 1;
  while ((1ull << end_bit) <= nb) end_bit++;
  GB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(cub_tmp, cub_bytes, keys0, keys1, vals0, vals1, (int)L.m, 0, end_bit,
                                              stream));
  GB_EV(2);
  k_msm_bucket_offsets<<<(nb + 1 + 255) / 256, 256, 0, stream>>>(keys1, (uint32_t)L.m, nb, off);
  k_msm_task_counts<<<(nb + 1 + 255) / 256, 256, 0, stream>>>(off, nb, pl.task_len, ntasks);
  cub_bytes = L.cub_bytes;
  GB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, ntasks, task_off, (int)nb + 1, stream));
  GB_EV(3);
  if (pipe && pipe->acc) {
    GB_CUDA_TRY(cudaEventRecord(pipe->front_ev, stream));
    GB_CUDA_TRY(cudaStreamWaitEvent(pipe->acc, pipe->front_ev, 0));
    stream = pipe->acc;
  }
  k_msm_accumulate<F><<<(unsigned)((L.max_tasks + 127) / 128), 128, 0, stream>>>(pl, d_table, vals1, off, task_off, partial);
  GB_EV(4);
  if (pipe && pipe->acc_ev) GB_CUDA_TRY(cudaEventRecord(pipe->acc_ev, stream));
  if (pipe && pipe->tail) {
    GB_CUDA_TRY(cudaStreamWaitEvent(pipe->tail, pipe->acc_ev, 0));
    stream = pipe->tail;
  }
  uint32_t* heavy = (uint32_t*)(w + L.o_heavy);
  GB_CUDA_TRY(cudaMemsetAsync(heavy, 0, 4, stream));
  k_msm_combine<F><<<(nb + 127) / 128, 128, 0, stream>>>(pl, task_off, partial, buckets, heavy, heavy + 1);
  {
    const int ht = 128;  // 4 warps = 4 buckets in flight per block
    const size_t hsmem = (size_t)ht * sizeof(XYZZ<F>);
    GB_CUDA_TRY(cudaFuncSetAttribute(k_msm_combine_heavy<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hsmem));
    int dev = 0, sms = 132;    // two blocks per SM (132 on H100 SXM)
    GB_CUDA_TRY(cudaGetDevice(&dev));
    GB_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    k_msm_combine_heavy<F><<<sms * 2, ht, hsmem, stream>>>(task_off, partial, buckets, heavy, heavy + 1);
  }
  GB_EV(5);
  const uint32_t nchunks = L.chunks_per_set * (uint32_t)pl.nsets;
  k_msm_reduce_chunks<F><<<(nchunks + 127) / 128, 128, 0, stream>>>(pl, L.chunks_per_set, buckets, chunks);
  GB_EV(6);
  int st = msm_set_sum_threads<F>();
  while (st > 32 && (uint32_t)st > L.chunks_per_set) st >>= 1;
  uint32_t slices = (L.chunks_per_set + (uint32_t)st - 1) / (uint32_t)st;       // one chunk sum per thread where 32 slices allow
  if (slices > MSM_SET_SLICES) slices = MSM_SET_SLICES;
  const size_t smem = (size_t)st * sizeof(XYZZ<F>);
  GB_CUDA_TRY(cudaFuncSetAttribute(k_msm_set_sum<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // a grid's y dimension stops at 65535 sets; a large batch of MSMs has more, which go in further launches
  for (uint32_t s0 = 0; s0 < (uint32_t)pl.nsets; s0 += 65535u) {
    const uint32_t rows = (uint32_t)pl.nsets - s0 < 65535u ? (uint32_t)pl.nsets - s0 : 65535u;
    k_msm_set_sum<F><<<dim3(slices, rows), st, smem, stream>>>(L.chunks_per_set, chunks + (size_t)s0 * L.chunks_per_set,
                                                               sets + (size_t)s0 * slices);
  }
  const int item_sets = pl.nsets / (int)pl.batch;
  const int fw = item_sets < 8 ? (item_sets > 0 ? item_sets : 1) : 8;             // warps of a finish block
  const size_t fsmem = (size_t)fw * 32 * sizeof(XYZZ<F>);
  XYZZ<F>* set_totals = sets + (size_t)pl.nsets * MSM_SET_SLICES;
  if (pl.batch > 1) {
    GB_CUDA_TRY(cudaFuncSetAttribute(k_msm_finish<F, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem));
    k_msm_finish<F, true><<<pl.batch, 32 * fw, fsmem, stream>>>(item_sets, pl.c, slices, sets, set_totals, d_out);
  } else {
    GB_CUDA_TRY(cudaFuncSetAttribute(k_msm_finish<F, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem));
    k_msm_finish<F, false><<<1, 32 * fw, fsmem, stream>>>(item_sets, pl.c, slices, sets, set_totals, d_out);
  }
  GB_EV(7);
#undef GB_EV
  return cudaGetLastError();
}

}  // namespace gb200
