// CPU emulation of the BATCHED bucket MSM (TEST ONLY): out[b] = sum_i scalars[b * n + i] * (base table_off + i of a
// caller-built table), b < batch.  msm.cuh's per-thread logic compiled for the host with the PTX carry chains emulated:
// the batched decompose (msm_decompose_batch_one: keys in the item's own bucket sets, entries laid out [w][b][i]), then
// the sort, accumulate, combine and chunk reduction over all batch * nsets sets at once, as the device runs them, and one
// Horner per item over its own sets.  Used by tests/test_msm_batch_emulation.py; NOT loaded by the product.
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <vector>

#include "msm.cuh"

using namespace gb200;

namespace {

template <class Fr, class F>
int msm_emu_batch(const void* table_, uint32_t stride, uint32_t table_off, const void* scalars_, uint32_t n, uint32_t batch,
                  int c, int precomp, uint32_t task_len, uint32_t chunk, void* out_jac, uint32_t* keys_out,
                  uint32_t* vals_out) {
  const Affine<F>* table = reinterpret_cast<const Affine<F>*>(table_);
  const Fr* scalars = reinterpret_cast<const Fr*>(scalars_);
  const MsmPlan pl = msm_make_batch_plan(batch, n, stride, table_off, Fr::Params::BITS, c, precomp, task_len, chunk);
  // 1 decompose: one (item, scalar) per thread of k_msm_decompose_batch
  const size_t m = (size_t)n * batch * pl.nwin;
  std::vector<uint32_t> keys(m), vals(m);
  for (uint32_t g = 0; g < n * batch; g++) msm_decompose_batch_one<Fr>(pl, g, scalars, keys.data(), vals.data());
  if (keys_out) std::copy(keys.begin(), keys.end(), keys_out);
  if (vals_out) std::copy(vals.begin(), vals.end(), vals_out);
  // 2 sort by bucket key (stable, as the radix sort), bucket offsets by search
  std::vector<uint32_t> order(m);
  std::iota(order.begin(), order.end(), 0u);
  std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return keys[x] < keys[y]; });
  std::vector<uint32_t> skeys(m), svals(m);
  for (size_t k = 0; k < m; k++) { skeys[k] = keys[order[k]]; svals[k] = vals[order[k]]; }
  std::vector<uint32_t> off(pl.total_buckets + 1);
  for (uint32_t b = 0; b <= pl.total_buckets; b++)
    off[b] = (uint32_t)(std::lower_bound(skeys.begin(), skeys.end(), b) - skeys.begin());
  // 3 accumulate in tasks of <= task_len entries, 4 combine the task partials of each bucket
  std::vector<XYZZ<F>> buckets(pl.total_buckets);
  for (uint32_t b = 0; b < pl.total_buckets; b++) {
    XYZZ<F> acc = XYZZ<F>::inf();
    for (uint32_t s = off[b]; s < off[b + 1]; s += pl.task_len)
      acc.add(msm_accumulate_range<F>(table, svals.data(), s, std::min(off[b + 1], s + pl.task_len)));
    buckets[b] = acc;
  }
  // 5 reduce: chunked weighted sums of every set of the batch, then Horner over each item's own sets
  std::vector<XYZZ<F>> set_sums(pl.nsets);
  for (int s = 0; s < pl.nsets; s++) {
    XYZZ<F> tot = XYZZ<F>::inf();
    for (uint32_t lo = 0; lo < pl.set_size; lo += pl.chunk)
      tot.add(msm_reduce_chunk<F>(buckets.data() + (size_t)s * pl.set_size, lo, std::min(pl.set_size, lo + pl.chunk)));
    set_sums[s] = tot;
  }
  const int item_sets = pl.nsets / (int)batch;
  Jacobian<F>* out = reinterpret_cast<Jacobian<F>*>(out_jac);
  for (uint32_t b = 0; b < batch; b++)
    out[b] = msm_horner<F>(set_sums.data() + (size_t)b * item_sets, item_sets, c).to_jacobian();
  return 0;
}

// the single MSM's decompose (msm_decompose_one), for the batch = 1 comparison
template <class Fr>
int decompose_single(uint32_t stride, uint32_t table_off, const void* scalars, uint32_t n, int c, int precomp,
                     uint32_t* keys, uint32_t* vals) {
  const MsmPlan pl = msm_make_plan(n, stride, table_off, Fr::Params::BITS, c, precomp, 1, 1);
  for (uint32_t i = 0; i < n; i++) msm_decompose_one<Fr>(pl, i, reinterpret_cast<const Fr*>(scalars), keys, vals);
  return 0;
}

}  // namespace

// keys_out / vals_out (nullable): the batch * n * nwin entries of the decompose, before the sort
extern "C" int emu_msm_batch(int curve, int group, const void* table, uint32_t stride, uint32_t off, const void* scalars,
                             uint32_t n, uint32_t batch, int c, int precomp, uint32_t task_len, uint32_t chunk, void* out_jac,
                             uint32_t* keys_out, uint32_t* vals_out) {
#define GB_EMU_BATCH(FR, FP) \
  msm_emu_batch<FR, FP>(table, stride, off, scalars, n, batch, c, precomp, task_len, chunk, out_jac, keys_out, vals_out)
  switch (curve * 2 + (group - 1)) {
    case 0: return GB_EMU_BATCH(bn254_fr, bn254_fp);
    case 1: return GB_EMU_BATCH(bn254_fr, bn254_fp2);
    case 2: return GB_EMU_BATCH(bls12_381_fr, bls12_381_fp);
    case 3: return GB_EMU_BATCH(bls12_381_fr, bls12_381_fp2);
    case 4: return GB_EMU_BATCH(bls12_377_fr, bls12_377_fp);
    case 5: return GB_EMU_BATCH(bls12_377_fr, bls12_377_fp2);
    case 6:
    case 7: return GB_EMU_BATCH(bw6_761_fr, bw6_761_fp);
  }
#undef GB_EMU_BATCH
  return -1;
}

extern "C" int emu_decompose_single(int curve, uint32_t stride, uint32_t off, const void* scalars, uint32_t n, int c,
                                    int precomp, uint32_t* keys, uint32_t* vals) {
  switch (curve) {
    case 0: return decompose_single<bn254_fr>(stride, off, scalars, n, c, precomp, keys, vals);
    case 1: return decompose_single<bls12_381_fr>(stride, off, scalars, n, c, precomp, keys, vals);
    case 2: return decompose_single<bls12_377_fr>(stride, off, scalars, n, c, precomp, keys, vals);
    case 3: return decompose_single<bw6_761_fr>(stride, off, scalars, n, c, precomp, keys, vals);
  }
  return -1;
}
