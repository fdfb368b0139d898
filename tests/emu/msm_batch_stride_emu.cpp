// CPU emulation of the batched MSM's decompose with a scalar stride (TEST ONLY): msm.cuh's msm_decompose_batch_one,
// compiled for the host, writes the keys and values of `batch` items whose n scalars start scalar_stride apart - the
// form the batched Groth16 prover uses for the n - 1 scalars of each n-long h and for the private tail of each wire
// vector.  Next to it the decompose of items stored back to back, as the batch read them before it had a stride (entry
// g reads scalars[g]).  Used by tests/test_gpu_groth16_batch.py; NOT loaded by the product.
#include <cstddef>
#include <cstdint>

#include "msm.cuh"

using namespace gb200;

namespace {

template <class Fr>
int decompose(uint32_t table_stride, uint32_t off, const void* scalars_, uint32_t n, uint32_t batch, uint32_t scalar_stride,
              int c, int precomp, int back_to_back, uint32_t* keys, uint32_t* vals) {
  const Fr* scalars = reinterpret_cast<const Fr*>(scalars_);
  const MsmPlan pl = msm_make_batch_plan(batch, n, table_stride, off, Fr::Params::BITS, c, precomp, 1, 1, scalar_stride);
  const uint32_t item_sets = (uint32_t)pl.nsets / pl.batch;
  for (uint32_t g = 0; g < n * batch; g++) {
    if (back_to_back) {
      const uint32_t b = g / pl.n, i = g - b * pl.n;
      msm_decompose_digits<Fr>(pl, scalars[g], pl.table_off + i, b * item_sets, g, (size_t)pl.batch * pl.n, keys, vals);
    } else {
      msm_decompose_batch_one<Fr>(pl, g, scalars, keys, vals);
    }
  }
  return 0;
}

}  // namespace

// scalar_stride 0 stands for n (msm_make_batch_plan's default)
extern "C" int emu_decompose_batch(int curve, uint32_t table_stride, uint32_t off, const void* scalars, uint32_t n,
                                   uint32_t batch, uint32_t scalar_stride, int c, int precomp, int back_to_back,
                                   uint32_t* keys, uint32_t* vals) {
#define GB_EMU_DEC(FR) decompose<FR>(table_stride, off, scalars, n, batch, scalar_stride, c, precomp, back_to_back, keys, vals)
  switch (curve) {
    case 0: return GB_EMU_DEC(bn254_fr);
    case 1: return GB_EMU_DEC(bls12_381_fr);
    case 2: return GB_EMU_DEC(bls12_377_fr);
    case 3: return GB_EMU_DEC(bw6_761_fr);
  }
#undef GB_EMU_DEC
  return -1;
}
