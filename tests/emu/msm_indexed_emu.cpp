// CPU emulation of the INDEXED bucket MSM (TEST ONLY): sum_i scalars[i] * (point idx[i] of a caller-built table).
// msm.cuh's per-thread logic compiled for the host with the PTX carry chains emulated, on a table laid out as the
// device keeps it: `count` points per slab, nwin slabs of 2^(c*w) * P_i when precomp, one slab otherwise - the slab
// index w * count + idx[i] of msm_decompose_one with an index list.  Every index is first checked with msm_index_ok,
// as b200_msm_indexed does before it enqueues the MSM.  Used by tests/test_msm_indexed_emulation.py; NOT loaded by the
// product.
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <vector>

#include "msm.cuh"

using namespace gb200;

namespace {

template <class Fr, class F>
int msm_emu_indexed(const void* table_, uint32_t count, const uint32_t* idx, const void* scalars_, uint32_t n, int c,
                    int precomp, uint32_t task_len, uint32_t chunk, void* out_jac) {
  const Affine<F>* table = reinterpret_cast<const Affine<F>*>(table_);
  const Fr* scalars = reinterpret_cast<const Fr*>(scalars_);
  const MsmPlan pl = msm_make_plan(n, count, 0, Fr::Params::BITS, c, precomp, task_len, chunk);
  // 1 decompose through the index list
  const size_t m = (size_t)n * pl.nwin;
  std::vector<uint32_t> keys(m), vals(m);
  for (uint32_t i = 0; i < n; i++) msm_decompose_one<Fr>(pl, i, scalars, keys.data(), vals.data(), idx);
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
  // 5 reduce: chunked weighted sums per set, then Horner over the sets
  std::vector<XYZZ<F>> set_sums(pl.nsets);
  for (int s = 0; s < pl.nsets; s++) {
    XYZZ<F> tot = XYZZ<F>::inf();
    for (uint32_t lo = 0; lo < pl.set_size; lo += pl.chunk)
      tot.add(msm_reduce_chunk<F>(buckets.data() + (size_t)s * pl.set_size, lo, std::min(pl.set_size, lo + pl.chunk)));
    set_sums[s] = tot;
  }
  *reinterpret_cast<Jacobian<F>*>(out_jac) = msm_horner<F>(set_sums.data(), pl.nsets, c).to_jacobian();
  return 0;
}

}  // namespace

// returns 1 with the lowest invalid position in *bad (and reads no point) when an index is not below `count`
extern "C" int emu_msm_table_indexed(int curve, int group, const void* table, uint32_t count, const uint32_t* idx,
                                     const void* scalars, uint32_t n, int c, int precomp, uint32_t task_len, uint32_t chunk,
                                     void* out_jac, uint32_t* bad) {
  for (uint32_t i = 0; i < n; i++)
    if (!msm_index_ok(idx, i, count)) { *bad = i; return 1; }
  switch (curve * 2 + (group - 1)) {
    case 0: return msm_emu_indexed<bn254_fr, bn254_fp>(table, count, idx, scalars, n, c, precomp, task_len, chunk, out_jac);
    case 1: return msm_emu_indexed<bn254_fr, bn254_fp2>(table, count, idx, scalars, n, c, precomp, task_len, chunk, out_jac);
    case 2: return msm_emu_indexed<bls12_381_fr, bls12_381_fp>(table, count, idx, scalars, n, c, precomp, task_len, chunk, out_jac);
    case 3: return msm_emu_indexed<bls12_381_fr, bls12_381_fp2>(table, count, idx, scalars, n, c, precomp, task_len, chunk, out_jac);
    case 4: return msm_emu_indexed<bls12_377_fr, bls12_377_fp>(table, count, idx, scalars, n, c, precomp, task_len, chunk, out_jac);
    case 5: return msm_emu_indexed<bls12_377_fr, bls12_377_fp2>(table, count, idx, scalars, n, c, precomp, task_len, chunk, out_jac);
    case 6:
    case 7: return msm_emu_indexed<bw6_761_fr, bw6_761_fp>(table, count, idx, scalars, n, c, precomp, task_len, chunk, out_jac);
  }
  return -1;
}
