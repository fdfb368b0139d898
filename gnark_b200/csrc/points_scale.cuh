// Variable-base scaling of a point vector by powers of one scalar: out[i] = (c * t^i) * P[i], in place on n affine points
// of one group.  It is the whole of a Groth16 MPC contribution (backend/groth16/<curve>/mpcsetup): phase 1's
// SrsCommons.update (phase1.go:104-147) scales [tau^i], [alpha tau^i] and [beta tau^i] with (c, t) = (tau', tau'),
// (alpha', tau') and (beta', tau'); phase 2's update (phase2.go:110-135) scales Z, PKK and each SigmaCKK[j] by one
// scalar (t = 1).  gnark runs these one ScalarMultiplication at a time.
//
// The scalars c * t^i are built on the device by the kernel behind b200_vec_scale_powers (k_scale_powers) applied to a
// vector of ones.  Each point then gets one thread running an MSB-first double-and-add over the canonical scalar, with
// mixed additions of the affine input: no table, so nothing indexed at run time.  On an H100 it ran 25-43 % faster than
// signed 4- and 5-bit windows (odd multiples P .. 7P or P .. 15P in XYZZ, Booth-recoded digits, about half the additions)
// on every curve and group (DESIGN.md §7, "Groth16 MPC contributions"), so the simple loop is the kernel.  The results go to affine through one batched inversion per FB_CHUNK points of a block
// (xyzz_batch_to_affine, as k_pntt_output does), so no n-sized XYZZ buffer is needed.
// The per-thread logic is HD: tests/emu/points_scale_emu.cpp runs it on the CPU.
#pragma once
#include "curve.cuh"
#include "fixed_base.cuh"   // FB_CHUNK, xyzz_batch_to_affine

namespace gb200 {

// k * p, k an Fr element in Montgomery form.  p = infinity or k = 0 gives infinity; p is not checked to be on the curve.
// The doublings before the top set bit and the first addition cost nothing (acc is still infinity).
template <class Fr, class F>
HD XYZZ<F> points_scale_mul(const Affine<F>& p, const Fr& k_mont) {
  XYZZ<F> acc = XYZZ<F>::inf();
  if (p.is_inf()) return acc;
  const Fr k = k_mont.from_mont();
  for (int bit = Fr::Params::BITS - 1; bit >= 0; bit--) {
    acc.dbl();
    if ((k.l[bit >> 5] >> (bit & 31)) & 1u) acc.add_mixed(p);
  }
  return acc;
}

constexpr int PS_THREADS = 64;   // a multiple of FB_CHUNK
static_assert(PS_THREADS % FB_CHUNK == 0, "whole batched inversions per block");
// 32-bit point indices in the kernel (the C ABI refuses larger n)
constexpr size_t PS_MAX_POINTS = 0xffffffffull;

#ifdef __CUDACC__
// the vector of ones that k_scale_powers turns into c * t^i
template <class Fr>
__global__ void __launch_bounds__(256) k_points_scale_ones(Fr* __restrict__ k, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) k[i] = Fr::one();
}

// one thread per point for the multiplication, then one thread per FB_CHUNK of the block's points for the batched
// inversion; in place (a block reads its points before the barrier and writes only its own points after it)
template <class Fr, class F>
__global__ void __launch_bounds__(PS_THREADS) k_points_scale(Affine<F>* __restrict__ pts, const Fr* __restrict__ k,
                                                            uint32_t n) {
  __shared__ __align__(16) unsigned char sm[PS_THREADS * sizeof(XYZZ<F>)];
  XYZZ<F>* s = reinterpret_cast<XYZZ<F>*>(sm);
  const uint32_t base = blockIdx.x * PS_THREADS;
  if (base + threadIdx.x < n) s[threadIdx.x] = points_scale_mul<Fr, F>(pts[base + threadIdx.x], k[base + threadIdx.x]);
  __syncthreads();
  const uint32_t first = base + threadIdx.x * FB_CHUNK;
  if (threadIdx.x * FB_CHUNK < PS_THREADS && first < n)
    xyzz_batch_to_affine<F>(s + threadIdx.x * FB_CHUNK, pts + first, n - first < FB_CHUNK ? n - first : FB_CHUNK);
}
#endif  // __CUDACC__

}  // namespace gb200
