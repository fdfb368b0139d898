// CPU emulation of the group-element NTT (points_ntt.cuh) on G1 of the four curves (TEST ONLY).
// The same per-thread logic as the device kernels - load, one DIF stage after another over the butterflies, the scaled
// bit-reversed read, the batched affine conversion in FB_CHUNK groups - compiled for the host with the PTX carry chains
// emulated, on the twiddle tables NttDomainHost builds exactly as the device domain does.
// Used by tests/test_points_ntt_emulation.py; NOT loaded by the product.
#include <cstdint>
#include <vector>

#include "points_ntt.cuh"

using namespace gb200;

namespace {

template <class Fr, class F>
int points_ntt_emu(void* pts_, int logn, int inverse) {
  Affine<F>* pts = reinterpret_cast<Affine<F>*>(pts_);
  if (logn < 0 || logn > 20) return -1;
  if (logn == 0) return 0;
  NttDomainHost<Fr> dom;
  dom.init(logn, nullptr, nullptr, false);
  const uint32_t n = 1u << logn;
  std::vector<XYZZ<F>> d(n), s(n);
  for (uint32_t i = 0; i < n; i++) d[i] = XYZZ<F>::from_affine(pts[i]);                 // k_pntt_load
  const Fr* tw = inverse ? dom.itw.data() : dom.tw.data();
  for (int beta = logn - 1; beta >= 0; beta--)                                            // k_pntt_stage
    for (uint32_t t = 0; t < n / 2; t++) points_ntt_butterfly<Fr, F>(d.data(), tw, logn, beta, t);
  for (uint32_t i = 0; i < n; i++) s[i] = points_ntt_output<Fr, F>(d.data(), logn, i, inverse != 0, dom.ninv);
  for (uint32_t first = 0; first < n; first += FB_CHUNK)                                  // k_pntt_output
    xyzz_batch_to_affine<F>(s.data() + first, pts + first, n - first < (uint32_t)FB_CHUNK ? n - first : FB_CHUNK);
  return 0;
}

template <class Fr, class F>
int points_ntt_mul_emu(const void* p, const void* k, void* out) {
  *reinterpret_cast<Affine<F>*>(out) =
      points_ntt_mul<Fr, F>(XYZZ<F>::from_affine(*reinterpret_cast<const Affine<F>*>(p)), *reinterpret_cast<const Fr*>(k))
          .to_affine();
  return 0;
}

}  // namespace

extern "C" int emu_points_ntt(int curve, void* points_affine, int logn, int inverse) {
  switch (curve) {
    case 0: return points_ntt_emu<bn254_fr, bn254_fp>(points_affine, logn, inverse);
    case 1: return points_ntt_emu<bls12_381_fr, bls12_381_fp>(points_affine, logn, inverse);
    case 2: return points_ntt_emu<bls12_377_fr, bls12_377_fp>(points_affine, logn, inverse);
    case 3: return points_ntt_emu<bw6_761_fr, bw6_761_fp>(points_affine, logn, inverse);
  }
  return -1;
}

// the twiddle multiplication alone: out = k * p (p affine, k Montgomery), affine
extern "C" int emu_points_ntt_mul(int curve, const void* point_affine, const void* k_mont, void* out_affine) {
  switch (curve) {
    case 0: return points_ntt_mul_emu<bn254_fr, bn254_fp>(point_affine, k_mont, out_affine);
    case 1: return points_ntt_mul_emu<bls12_381_fr, bls12_381_fp>(point_affine, k_mont, out_affine);
    case 2: return points_ntt_mul_emu<bls12_377_fr, bls12_377_fp>(point_affine, k_mont, out_affine);
    case 3: return points_ntt_mul_emu<bw6_761_fr, bw6_761_fp>(point_affine, k_mont, out_affine);
  }
  return -1;
}
