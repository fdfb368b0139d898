// sm_90a NTT kernels + device domain + stream-ordered drivers (see ntt.cuh for the
// conventions and the reference call sites), plus the fused Groth16 quotient
// pipeline computeH (backend/groth16/bn254/prove.go:346-389, GPU twin
// backend/accelerated/icicle/groth16/bn254/icicle.go:1391-1488).
#pragma once
#include <cuda_runtime.h>

#include <cstdlib>

#include "msm_impl.cuh"  // GB_CUDA_TRY, gb_align
#include "ntt.cuh"

namespace gb200 {

// out[k] = scale * base^k, k < n.   pw[j] = base^(2^j)
template <class Fr>
__global__ void __launch_bounds__(256) k_powers(const Fr* __restrict__ pw, Fr scale, uint32_t n, Fr* __restrict__ out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  Fr acc = scale;
  uint32_t e = k;
  for (int j = 0; e; j++, e >>= 1)
    if (e & 1) acc = acc * pw[j];
  out[k] = acc;
}

// Read-only table element (twiddle, coset factor) as 16-byte loads.  Left to the compiler, `tw[k]` feeding a product
// is split into one 4-byte load per limb (8 LDG.32 per twiddle, each a separate 32-lane gather); two LDG.128 fetch the
// same sectors with a quarter of the requests.
template <class Fr>
__device__ __forceinline__ Fr ntt_ldg(const Fr* __restrict__ p) {
  static_assert(sizeof(Fr) % 16 == 0 && Fr::N % 4 == 0, "Fr is a whole number of 16-byte words");
  Fr v;
  const uint4* q = reinterpret_cast<const uint4*>(p);
#pragma unroll
  for (int k = 0; k < Fr::N / 4; k++) {
    const uint4 x = __ldg(q + k);
    v.l[4 * k] = x.x; v.l[4 * k + 1] = x.y; v.l[4 * k + 2] = x.z; v.l[4 * k + 3] = x.w;
  }
  return v;
}

// One pass: tile of 2^(S+cb) elements in shared memory (limb-major), blockDim = tile/2.  kBatch: blockIdx.y selects the
// vector of a batch (vector b at data + b * 2^logn); tables and the pre / post indices are those of the vector.  A single
// transform takes the other instantiation, whose registers the vector offset would raise (BN254: 62 -> 64, the cap).
template <class Fr, bool kBatch>
__global__ void __launch_bounds__(1 << (NTT_MAX_TILE_LOG - 1))
k_ntt_pass(NttPass p, int logn, int dit, const Fr* __restrict__ tw, Fr* __restrict__ data,
                           const Fr* __restrict__ pre, int pre_bitrev, const Fr* __restrict__ post, int post_bitrev,
                           int use_const, Fr post_const) {
  constexpr int N = Fr::N;
  extern __shared__ __align__(16) uint32_t sm[];
  const uint32_t tile_elems = 1u << (p.S + p.cb);
  const uint32_t half = tile_elems >> 1;
  const uint32_t t = threadIdx.x;
  const uint32_t tile = blockIdx.x;
  if (kBatch) data += (size_t)blockIdx.y << logn;

  // load (+ optional pre-scale)
#pragma unroll
  for (int r = 0; r < 2; r++) {
    const uint32_t e = t + r * half;
    const uint32_t gi = ntt_tile_index(p, tile, e);
    Fr v = data[gi];
    if (pre) v = v * ntt_ldg(pre + (pre_bitrev ? ntt_bitrev(gi, logn) : gi));
#pragma unroll
    for (int l = 0; l < N; l++) sm[l * tile_elems + e] = v.l[l];
  }
  __syncthreads();

  for (int k = 0; k < p.S; k++) {
    const int s = dit ? k : p.S - 1 - k;
    const int lb = p.cb + s;
    const int beta = p.lo_bit + s;
    const uint32_t lo = ((t >> lb) << (lb + 1)) | (t & ((1u << lb) - 1u));
    const uint32_t hi = lo | (1u << lb);
    Fr a, b;
#pragma unroll
    for (int l = 0; l < N; l++) { a.l[l] = sm[l * tile_elems + lo]; b.l[l] = sm[l * tile_elems + hi]; }
    if (beta == 0) {
      // index bit 0: every twiddle is w^0 = 1 (block-uniform branch), the butterfly is (a + b, a - b)
      const Fr d = a - b;
      a = a + b;
      b = d;
    } else {
      const Fr w = ntt_ldg(tw + ntt_twiddle_index(logn, ntt_tile_index(p, tile, lo), beta));
      if (dit) ntt_bfly_dit(a, b, w); else ntt_bfly_dif(a, b, w);
    }
#pragma unroll
    for (int l = 0; l < N; l++) { sm[l * tile_elems + lo] = a.l[l]; sm[l * tile_elems + hi] = b.l[l]; }
    // (between two stages on local bits <= 5 a warp only touches its own 64 slots and __syncwarp() would do; it was
    // not faster than the block barrier)
    __syncthreads();
  }

  // store (+ optional post-scale)
#pragma unroll
  for (int r = 0; r < 2; r++) {
    const uint32_t e = t + r * half;
    const uint32_t gi = ntt_tile_index(p, tile, e);
    Fr v;
#pragma unroll
    for (int l = 0; l < N; l++) v.l[l] = sm[l * tile_elems + e];
    if (post) v = v * ntt_ldg(post + (post_bitrev ? ntt_bitrev(gi, logn) : gi));
    else if (use_const) v = v * post_const;
    data[gi] = v;
  }
}

// n == 1 degenerate transform: only scaling applies, to each of the `batch` one-element vectors
template <class Fr>
__global__ void __launch_bounds__(256) k_ntt_scale1(Fr* data, Fr c, size_t batch) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < batch) data[i] = data[i] * c;
}

template <class Fr>
struct NttDomainDev {
  int dev = 0;
  int logn = 0;
  uint32_t n = 0;
  Fr gen, gen_inv, coset, coset_inv, ninv;
  Fr* tw = nullptr;    // w^k,  k < n/2
  Fr* itw = nullptr;   // w^-k
  Fr* cos = nullptr;   // g^j,  j < n
  Fr* icos = nullptr;  // g^-j / n
  NttPlan plan;
  // PLONK: 1 / (c w^j - 1), j < n, for the coset c the last constraint pass on this handle ran on (precomputedDenominators,
  // backend/plonk/bn254/prove.go:1002-1007).  The prover keeps one handle per coset of the quotient domain, so after the
  // first proof this is a pure cache (n elements of HBM per handle; GB200_PLONK_DEN_CACHE=0 computes it per call)
  Fr* den_inv = nullptr;
  Fr den_coset;
  bool den_valid = false;

  size_t table_bytes() const { return ((size_t)(n > 1 ? n / 2 : 1) * 2 + (size_t)n * 2) * sizeof(Fr); }

  static cudaError_t powers(cudaStream_t st, const Fr& base, const Fr& scale, uint32_t n, Fr* out, Fr* d_pw) {
    Fr pw[32];
    Fr b = base;
    for (int j = 0; j < 32; j++) { pw[j] = b; b = b.sqr(); }
    GB_CUDA_TRY(cudaMemcpyAsync(d_pw, pw, sizeof(pw), cudaMemcpyHostToDevice, st));
    k_powers<Fr><<<(n + 255) / 256, 256, 0, st>>>(d_pw, scale, n, out);
    GB_CUDA_TRY(cudaGetLastError());
    return cudaStreamSynchronize(st);  // pw is a stack buffer
  }

  cudaError_t init(cudaStream_t st, int logn_, const Fr* gen_mont, const Fr* coset_mont) {
    logn = logn_;
    n = 1u << logn;
    // Tile = 2^8 elements (128 threads, 8 KiB of shared memory per block): a pass is a chain of barrier-separated phases
    // (load, one stage per barrier, store), so SMALL blocks - many resident per SM - overlap one block's loads and
    // barriers with another's butterflies.  Measured on H100 SXM (400 W power limit; tools/sweep_ntt.py, ms per transform):
    //   tile            2^11    2^10    2^9     2^8     2^7
    //   BN254 2^20      0.316   0.292   0.255   0.238   0.248     (2^11: one 1024-thread block per SM)
    //   BN254 2^24      6.17    5.55    5.39    4.94    5.18
    //   BLS12-381 2^22  1.55    1.31    1.17    1.15    1.14
    // although the smaller tiles need more passes (2^20: 2 passes at 2^11, 3 at 2^9 / 2^8).  GB200_NTT_TILE_LOG (6..11) overrides.
    int tile_log = NTT_DEFAULT_TILE_LOG;
    if (const char* e = getenv("GB200_NTT_TILE_LOG")) { const int v = atoi(e); if (v >= 6 && v <= NTT_MAX_TILE_LOG) tile_log = v; }
    plan = ntt_make_plan(logn, tile_log);
    gen = gen_mont ? *gen_mont : NttDomainHost<Fr>::default_generator(logn);
    coset = coset_mont ? *coset_mont : NttDomainHost<Fr>::default_coset();
    gen_inv = gen.inverse();
    coset_inv = coset.inverse();
    Fr nn = Fr::one();
    for (int k = 0; k < logn; k++) nn = nn.dbl();
    ninv = nn.inverse();
    const uint32_t half = n > 1 ? n / 2 : 1;
    Fr* d_pw = nullptr;
    GB_CUDA_TRY(cudaMalloc(&d_pw, 32 * sizeof(Fr)));
    GB_CUDA_TRY(cudaMalloc(&tw, half * sizeof(Fr)));
    GB_CUDA_TRY(cudaMalloc(&itw, half * sizeof(Fr)));
    GB_CUDA_TRY(cudaMalloc(&cos, (size_t)n * sizeof(Fr)));
    GB_CUDA_TRY(cudaMalloc(&icos, (size_t)n * sizeof(Fr)));
    GB_CUDA_TRY(powers(st, gen, Fr::one(), half, tw, d_pw));
    GB_CUDA_TRY(powers(st, gen_inv, Fr::one(), half, itw, d_pw));
    GB_CUDA_TRY(powers(st, coset, Fr::one(), n, cos, d_pw));
    GB_CUDA_TRY(powers(st, coset_inv, ninv, n, icos, d_pw));
    return cudaFree(d_pw);
  }
  void destroy() {
    cudaFree(tw); cudaFree(itw); cudaFree(cos); cudaFree(icos); cudaFree(den_inv);
    tw = itw = cos = icos = den_inv = nullptr;
    den_valid = false;
  }
};

// a grid's y dimension stops at 65535: larger batches of vectors go in further launches
constexpr size_t NTT_MAX_GRID_Y = 65535;

// Enqueue `batch` transforms, in place on device data (batch * n elements, vector b at data + b * n).
template <class Fr>
cudaError_t ntt_enqueue(cudaStream_t st, const NttDomainDev<Fr>& d, Fr* data, bool inverse, int decimation,
                        bool on_coset, size_t batch = 1) {
  const Fr* T = inverse ? d.itw : d.tw;
  const bool dit = decimation == NTT_DIT;
  if (batch == 0) return cudaSuccess;
  if (d.logn == 0) {
    if (inverse) {
      const size_t threads = batch < 256 ? batch : 256;
      k_ntt_scale1<Fr><<<(unsigned)((batch + threads - 1) / threads), (unsigned)threads, 0, st>>>(data, d.ninv, batch);
    }
    return cudaGetLastError();
  }
  for (int pi = 0; pi < d.plan.npasses; pi++) {
    const NttPass& p = dit ? d.plan.pass[pi] : d.plan.pass[d.plan.npasses - 1 - pi];
    const bool first = pi == 0, last = pi == d.plan.npasses - 1;
    const Fr* pre = nullptr; int pre_br = 0;
    const Fr* post = nullptr; int post_br = 0; int use_const = 0;
    if (first && !inverse && on_coset) { pre = d.cos; pre_br = dit ? 1 : 0; }
    if (last && inverse) {
      if (on_coset) { post = d.icos; post_br = dit ? 0 : 1; }
      else use_const = 1;
    }
    const uint32_t tile_elems = 1u << (p.S + p.cb);
    const uint32_t ntiles = d.n >> (p.S + p.cb);
    const size_t smem = (size_t)tile_elems * sizeof(Fr);
    const int max_smem = (int)(NTT_MAX_TILE_LOG >= 11 ? (sizeof(Fr) << NTT_MAX_TILE_LOG) : smem);
    if (batch == 1) {
      GB_CUDA_TRY(cudaFuncSetAttribute(k_ntt_pass<Fr, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
      k_ntt_pass<Fr, false><<<ntiles, tile_elems / 2, smem, st>>>(p, d.logn, dit ? 1 : 0, T, data, pre, pre_br, post, post_br,
                                                                  use_const, d.ninv);
      GB_CUDA_TRY(cudaGetLastError());
      continue;
    }
    GB_CUDA_TRY(cudaFuncSetAttribute(k_ntt_pass<Fr, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    for (size_t b0 = 0; b0 < batch; b0 += NTT_MAX_GRID_Y) {
      const unsigned rows = (unsigned)(batch - b0 < NTT_MAX_GRID_Y ? batch - b0 : NTT_MAX_GRID_Y);
      k_ntt_pass<Fr, true><<<dim3(ntiles, rows), tile_elems / 2, smem, st>>>(p, d.logn, dit ? 1 : 0, T, data + b0 * d.n, pre,
                                                                             pre_br, post, post_br, use_const, d.ninv);
      GB_CUDA_TRY(cudaGetLastError());
    }
  }
  return cudaSuccess;
}

// a[i] = (a[i]*b[i] - c[i]) * den      (prove.go:377-383; ICICLE: 3 VecOps icicle.go:1455-1461)
// (the batched computeH runs it over the k * n elements of the k items' a, b and c)
template <class Fr>
__global__ void __launch_bounds__(256) k_h_pointwise(uint32_t n, Fr* __restrict__ a, const Fr* __restrict__ b,
                                                     const Fr* __restrict__ c, Fr den) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = (a[i] * b[i] - c[i]) * den;
}

// 1 / (g^n - 1) of the coset g: the vanishing polynomial's inverse on the coset
template <class Fr>
Fr compute_h_den(const NttDomainDev<Fr>& d) {
  Fr gn = d.coset;
  for (int k = 0; k < d.logn; k++) gn = gn.sqr();
  return (gn - Fr::one()).inverse();
}

// computeH on device.  a, b, c: n-element device vectors (already zero padded);
// on return a holds h in bit-reversed order (Montgomery), b and c are clobbered.
template <class Fr>
cudaError_t compute_h_enqueue(cudaStream_t st, const NttDomainDev<Fr>& d, Fr* a, Fr* b, Fr* c) {
  Fr* v[3] = {a, b, c};
  for (int k = 0; k < 3; k++) {
    GB_CUDA_TRY(ntt_enqueue<Fr>(st, d, v[k], true, NTT_DIF, false));
    GB_CUDA_TRY(ntt_enqueue<Fr>(st, d, v[k], false, NTT_DIT, true));
  }
  k_h_pointwise<Fr><<<(d.n + 255) / 256, 256, 0, st>>>(d.n, a, b, c, compute_h_den(d));
  GB_CUDA_TRY(cudaGetLastError());
  return ntt_enqueue<Fr>(st, d, a, true, NTT_DIF, true);
}

// computeH of `batch` proofs on one domain.  abc: [3][batch][n] device vectors (A of every item, then B, then C,
// already zero padded); on return h of item b is at abc + b * n, bit-reversed, exactly as compute_h_enqueue leaves a.
// batch * n must fit the pointwise kernel's 32-bit index (checked by the caller).
template <class Fr>
cudaError_t compute_h_batch_enqueue(cudaStream_t st, const NttDomainDev<Fr>& d, Fr* abc, size_t batch) {
  if (batch == 0) return cudaSuccess;
  GB_CUDA_TRY(ntt_enqueue<Fr>(st, d, abc, true, NTT_DIF, false, 3 * batch));
  GB_CUDA_TRY(ntt_enqueue<Fr>(st, d, abc, false, NTT_DIT, true, 3 * batch));
  const uint32_t kn = (uint32_t)(batch * d.n);
  k_h_pointwise<Fr><<<(kn + 255) / 256, 256, 0, st>>>(kn, abc, abc + (size_t)kn, abc + 2 * (size_t)kn, compute_h_den(d));
  GB_CUDA_TRY(cudaGetLastError());
  return ntt_enqueue<Fr>(st, d, abc, true, NTT_DIF, true, batch);
}

}  // namespace gb200
