// CPU emulation of b200_points_scale (points_scale.cuh) on G1 and G2 of the four curves (TEST ONLY).
// The scalars c * t^i as k_scale_powers leaves them on a vector of ones (c times the product of the squarings t^(2^j)
// over the set bits of i), then the per-thread multiplication and the per-block batched affine conversion of
// k_points_scale, compiled for the host with the PTX carry chains emulated.
// Used by tests/test_points_scale_emulation.py; NOT loaded by the product.
#include <cstdint>
#include <vector>

#include "points_scale.cuh"

using namespace gb200;

namespace {

template <class Fr, class F>
int points_scale_emu(void* pts_, size_t n, const void* c_, const void* t_) {
  Affine<F>* pts = reinterpret_cast<Affine<F>*>(pts_);
  const Fr c = *reinterpret_cast<const Fr*>(c_);
  Fr pw[64];
  Fr b = t_ ? *reinterpret_cast<const Fr*>(t_) : Fr::one();
  for (int j = 0; j < 64; j++) { pw[j] = b; b = b.sqr(); }
  std::vector<XYZZ<F>> s(PS_THREADS);
  for (size_t base = 0; base < n; base += PS_THREADS) {
    const uint32_t cnt = (uint32_t)(n - base < (size_t)PS_THREADS ? n - base : (size_t)PS_THREADS);
    for (uint32_t i = 0; i < cnt; i++) {
      Fr k = Fr::one() * c;                                    // k_points_scale_ones, then k_scale_powers
      size_t e = base + i;
      for (int j = 0; e; j++, e >>= 1)
        if (e & 1) k = k * pw[j];
      s[i] = points_scale_mul<Fr, F>(pts[base + i], k);
    }
    for (uint32_t first = 0; first < cnt; first += FB_CHUNK)
      xyzz_batch_to_affine<F>(s.data() + first, pts + base + first, cnt - first < (uint32_t)FB_CHUNK ? cnt - first : FB_CHUNK);
  }
  return 0;
}

template <class Fr, class F>
int points_scale_mul_emu(const void* p, const void* k, void* out) {
  *reinterpret_cast<Affine<F>*>(out) =
      points_scale_mul<Fr, F>(*reinterpret_cast<const Affine<F>*>(p), *reinterpret_cast<const Fr*>(k)).to_affine();
  return 0;
}

}  // namespace

// points[i] <- (c * t^i) * points[i], i < n; t null: t = 1
extern "C" int emu_points_scale(int curve, int group, void* points_affine, size_t n, const void* c_mont,
                                const void* t_mont) {
  const int key = curve * 2 + (group - 1);
  switch (group == 1 || group == 2 ? key : -1) {
    case 0: return points_scale_emu<bn254_fr, bn254_fp>(points_affine, n, c_mont, t_mont);
    case 1: return points_scale_emu<bn254_fr, bn254_fp2>(points_affine, n, c_mont, t_mont);
    case 2: return points_scale_emu<bls12_381_fr, bls12_381_fp>(points_affine, n, c_mont, t_mont);
    case 3: return points_scale_emu<bls12_381_fr, bls12_381_fp2>(points_affine, n, c_mont, t_mont);
    case 4: return points_scale_emu<bls12_377_fr, bls12_377_fp>(points_affine, n, c_mont, t_mont);
    case 5: return points_scale_emu<bls12_377_fr, bls12_377_fp2>(points_affine, n, c_mont, t_mont);
    case 6: case 7: return points_scale_emu<bw6_761_fr, bw6_761_fp>(points_affine, n, c_mont, t_mont);  // G2 over Fp
  }
  return -1;
}

// the per-thread multiplication alone: out = k * p (p affine, k Montgomery), affine
extern "C" int emu_points_scale_mul(int curve, int group, const void* point_affine, const void* k_mont, void* out_affine) {
  const int key = curve * 2 + (group - 1);
  switch (group == 1 || group == 2 ? key : -1) {
    case 0: return points_scale_mul_emu<bn254_fr, bn254_fp>(point_affine, k_mont, out_affine);
    case 1: return points_scale_mul_emu<bn254_fr, bn254_fp2>(point_affine, k_mont, out_affine);
    case 2: return points_scale_mul_emu<bls12_381_fr, bls12_381_fp>(point_affine, k_mont, out_affine);
    case 3: return points_scale_mul_emu<bls12_381_fr, bls12_381_fp2>(point_affine, k_mont, out_affine);
    case 4: return points_scale_mul_emu<bls12_377_fr, bls12_377_fp>(point_affine, k_mont, out_affine);
    case 5: return points_scale_mul_emu<bls12_377_fr, bls12_377_fp2>(point_affine, k_mont, out_affine);
    case 6: case 7: return points_scale_mul_emu<bw6_761_fr, bw6_761_fp>(point_affine, k_mont, out_affine);
  }
  return -1;
}
