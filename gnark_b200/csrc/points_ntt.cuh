// Radix-2 NTT over the points of a group (G1): the KZG SRS conversion between monomial form [tau^k]G and the Lagrange
// basis [L_i(tau)]G.  Reference call sites: gnark-crypto's kzg.ToLagrangeG1 (as used at
// std/recursion/plonk/verifier_test.go:370), whose in-tree statement is backend/groth16/<curve>/mpcsetup/lagrange.go:21-41
// (lagrangeCoeffsG1) and :132-169 (the DIF recursion); test/unsafekzg/kzgsrs.go:184-198 takes the trapdoor shortcut.
//
//   inverse = 1:  out[i] = (1/n) sum_k w^(-ik) in[k]        (monomial -> Lagrange)
//   inverse = 0:  out[k] = sum_i w^(ik) in[i]               (Lagrange -> monomial)
//
// Natural order in and out, canonical affine results.  Same conventions as the Fr NTT (ntt.cuh): DIF stages on the
// domain's tables w^k / w^-k (k < n/2), butterfly (a, b) -> (a + b, (a - b) * w^j) with j = ntt_twiddle_index, then a
// bit-reversed read.  A butterfly is two XYZZ additions and one variable-base scalar multiplication by a full-width Fr
// scalar (thousands of Fp products), against 4 XYZZ points of memory traffic: every stage is compute-bound, so the device
// path is one launch per stage with one thread per butterfly, no shared-memory tiling.
// The per-thread logic is HD: tests/emu/points_ntt_emu.cpp runs it on the CPU.
#pragma once
#include "curve.cuh"
#include "fixed_base.cuh"   // FB_CHUNK, xyzz_batch_to_affine
#include "ntt.cuh"
#ifdef __CUDACC__
#include "msm_impl.cuh"     // GB_CUDA_TRY, AsyncBuf
#endif

namespace gb200 {

// k * p, k an Fr element in Montgomery form: MSB-first double-and-add over the canonical scalar.  While the accumulator
// is still infinity its doublings and the first addition cost nothing (XYZZ::dbl / add return early), so the work is
// (top bit) doublings + (popcount - 1) additions.  p = infinity or k = 0 gives infinity.
template <class Fr, class F>
HD XYZZ<F> points_ntt_mul(const XYZZ<F>& p, const Fr& k_mont) {
  const Fr k = k_mont.from_mont();
  XYZZ<F> acc = XYZZ<F>::inf();
  if (p.is_inf()) return acc;
  for (int bit = Fr::Params::BITS - 1; bit >= 0; bit--) {
    acc.dbl();
    if ((k.l[bit >> 5] >> (bit & 31)) & 1u) acc.add(p);
  }
  return acc;
}

// butterfly t (< n/2) of the DIF stage on index bit beta, in place on d[]: (a, b) -> (a + b, (a - b) * tw[j])
template <class Fr, class F>
HD void points_ntt_butterfly(XYZZ<F>* d, const Fr* tw, int logn, int beta, uint32_t t) {
  const uint32_t lo = ((t >> beta) << (beta + 1)) | (t & ((1u << beta) - 1u));
  const uint32_t hi = lo | (1u << beta);
  const XYZZ<F> b = d[hi];
  XYZZ<F> a = d[lo], diff = a;
  diff.add(b.neg());
  a.add(b);
  const uint32_t j = ntt_twiddle_index(logn, lo, beta);
  d[lo] = a;
  d[hi] = j ? points_ntt_mul<Fr, F>(diff, tw[j]) : diff;
}

// output i after the DIF stages: the point at bitrev(i), times 1/n for the inverse transform
template <class Fr, class F>
HD XYZZ<F> points_ntt_output(const XYZZ<F>* d, int logn, uint32_t i, bool scale, const Fr& ninv) {
  const XYZZ<F> p = d[ntt_bitrev(i, logn)];
  return scale ? points_ntt_mul<Fr, F>(p, ninv) : p;
}

#ifdef __CUDACC__
constexpr int PNTT_OUT_THREADS = 64;   // a multiple of FB_CHUNK
static_assert(PNTT_OUT_THREADS % FB_CHUNK == 0, "whole batched inversions per block");

template <class F>
__global__ void __launch_bounds__(256) k_pntt_load(const Affine<F>* __restrict__ in, uint32_t n, XYZZ<F>* __restrict__ d) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) d[i] = XYZZ<F>::from_affine(in[i]);
}
template <class Fr, class F>
__global__ void __launch_bounds__(128) k_pntt_stage(XYZZ<F>* __restrict__ d, const Fr* __restrict__ tw, int logn, int beta) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < (1u << (logn - 1))) points_ntt_butterfly<Fr, F>(d, tw, logn, beta, t);
}
// scale (inverse only), bit-reverse permutation and affine conversion: one thread per output point for the scalar
// multiplication, then one thread per FB_CHUNK of the block's points for the batched inversion
template <class Fr, class F>
__global__ void __launch_bounds__(PNTT_OUT_THREADS) k_pntt_output(const XYZZ<F>* __restrict__ d, int logn, int scale, Fr ninv,
                                                                 Affine<F>* __restrict__ out) {
  __shared__ __align__(16) unsigned char sm[PNTT_OUT_THREADS * sizeof(XYZZ<F>)];
  XYZZ<F>* s = reinterpret_cast<XYZZ<F>*>(sm);
  const uint32_t n = 1u << logn;
  const uint32_t base = blockIdx.x * PNTT_OUT_THREADS;
  if (base + threadIdx.x < n) s[threadIdx.x] = points_ntt_output<Fr, F>(d, logn, base + threadIdx.x, scale != 0, ninv);
  __syncthreads();
  const uint32_t first = base + threadIdx.x * FB_CHUNK;
  if (threadIdx.x * FB_CHUNK < PNTT_OUT_THREADS && first < n)
    xyzz_batch_to_affine<F>(s + threadIdx.x * FB_CHUNK, out + first, n - first < FB_CHUNK ? n - first : FB_CHUNK);
}

// In place on 2^logn device points.  tw: the domain's w^k (forward) or w^-k (inverse) table, k < n/2.  The XYZZ work
// buffer comes from the stream-ordered pool.
template <class Fr, class F>
cudaError_t points_ntt_enqueue(cudaStream_t st, int logn, const Fr* tw, const Fr& ninv, bool inverse, Affine<F>* pts) {
  if (logn == 0) return cudaSuccess;   // the one-point transform is the identity
  const uint32_t n = 1u << logn, half = n / 2;
  AsyncBuf work;
  GB_CUDA_TRY(work.alloc((size_t)n * sizeof(XYZZ<F>), st));
  XYZZ<F>* d = reinterpret_cast<XYZZ<F>*>(work.p);
  k_pntt_load<F><<<(n + 255) / 256, 256, 0, st>>>(pts, n, d);
  for (int beta = logn - 1; beta >= 0; beta--)
    k_pntt_stage<Fr, F><<<(half + 127) / 128, 128, 0, st>>>(d, tw, logn, beta);
  k_pntt_output<Fr, F><<<(n + PNTT_OUT_THREADS - 1) / PNTT_OUT_THREADS, PNTT_OUT_THREADS, 0, st>>>(d, logn, inverse ? 1 : 0,
                                                                                                  ninv, pts);
  GB_CUDA_TRY(cudaGetLastError());
  return work.release_on(st);
}
#endif  // __CUDACC__

}  // namespace gb200
