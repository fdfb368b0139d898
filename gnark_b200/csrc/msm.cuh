// Pippenger bucket MSM - per-thread logic (host/device) shared by the sm_90a
// kernels in msm_impl.cuh and by the CPU emulation used in the "not gpu" tests.
//
// Replaces gnark-crypto's G1Jac/G2Jac.MultiExp at the reference's call sites
// backend/groth16/bn254/prove.go:194,207,227,237,283 and ICICLE's Msm/G2Msm at
// backend/accelerated/icicle/groth16/bn254/icicle.go:397,451.
//
// Pipeline (one stream, no host sync until the result copy):
//   1 decompose   scalar (Montgomery Fr, as gnark stores it) -> canonical ->
//                 signed c-bit digits; one (bucket key, table index|sign) entry
//                 per non-zero digit.
//   2 sort        entries by bucket key (radix sort), bucket offsets by search.
//   3 accumulate  tasks of <= TASK_LEN consecutive entries of one bucket:
//                 gather affine point, conditional negate, XYZZ mixed add.  (the
//                 dominant kernel: W*(sizeof(affine)+4) B and ~10 Fp-mul per scalar-mul)
//   4 combine     partial sums of a bucket -> bucket sum.
//   5 reduce      sum_k (k+1)*B_k per bucket set by chunked running sums, then a
//                 tree sum; Horner over bucket sets when there is more than one.
//
// Table modes.  PRECOMP: the device table holds 2^(c*w)*P_i for every window w
// (layout [w][i], built once at table upload - HBM capacity traded for the
// removal of the serial 2^c-doubling Horner tail and of W-1 bucket reductions):
// all windows share ONE bucket set.  PLAIN: table = the n points; W bucket sets.
#pragma once
#include "curve.cuh"

namespace gb200 {

struct MsmPlan {
  uint32_t n;             // scalars in this call
  uint32_t table_stride;  // points per window slab of the table
  uint32_t table_off;     // offset of the first base inside a slab
  int c;                  // window bits
  int nwin;               // windows per scalar
  int precomp;            // 1: table has nwin slabs, single bucket set
  int nsets;              // bucket sets (1 or nwin)
  uint32_t set_size;      // buckets per set = 2^(c-1)
  uint32_t total_buckets; // nsets * set_size ; also the "no entry" key
  uint32_t task_len;      // max entries per accumulate task
  uint32_t chunk;         // buckets per level-1 reduction chunk
  uint32_t batch;         // MSMs over the same bases (1 = a single MSM); nsets and total_buckets count every item's sets
  uint32_t scalar_stride; // batch: scalars between the first scalars of consecutive items (>= n)
};

HD int msm_num_windows(int scalar_bits, int c) { return scalar_bits / c + 1; }

HD MsmPlan msm_make_plan(uint32_t n, uint32_t table_stride, uint32_t table_off, int scalar_bits, int c,
                         int precomp, uint32_t task_len, uint32_t chunk) {
  MsmPlan p;
  p.n = n; p.table_stride = table_stride; p.table_off = table_off; p.c = c;
  p.nwin = msm_num_windows(scalar_bits, c);
  p.precomp = precomp;
  p.nsets = precomp ? 1 : p.nwin;
  p.set_size = 1u << (c - 1);
  p.total_buckets = (uint32_t)p.nsets * p.set_size;
  p.task_len = task_len;
  p.chunk = chunk;
  p.batch = 1;
  p.scalar_stride = n;
  return p;
}

// `batch` MSMs of n scalars each over the same bases: one pipeline whose bucket sets are the items' sets side by side
// (item b owns sets [b * nsets_item, (b + 1) * nsets_item)); sort, offsets, accumulate, combine and the chunk reduction
// work on any number of contiguous sets and need nothing else.  Item b's scalars start at scalar b * scalar_stride, so
// the items can be the first n elements of longer vectors (the n - 1 of an n-long h, the tail of a wire vector);
// 0 stands for n (items back to back).
HD MsmPlan msm_make_batch_plan(uint32_t batch, uint32_t n, uint32_t table_stride, uint32_t table_off, int scalar_bits, int c,
                               int precomp, uint32_t task_len, uint32_t chunk, uint32_t scalar_stride = 0) {
  MsmPlan p = msm_make_plan(n, table_stride, table_off, scalar_bits, c, precomp, task_len, chunk);
  p.batch = batch;
  p.scalar_stride = scalar_stride ? scalar_stride : n;
  p.nsets *= (int)batch;
  p.total_buckets = (uint32_t)p.nsets * p.set_size;
  return p;
}

// ---- 0. index check (indexed MSMs) -------------------------------------------
// an index list may address the table only through checked entries: position i is valid when it names one of the
// table's `count` points (not slab entries: the slab offset is added by the decompose)
HD bool msm_index_ok(const uint32_t* idx, uint32_t i, uint32_t count) { return idx[i] < count; }

// ---- 1. decompose ----------------------------------------------------------
// Digits of one scalar (Montgomery form) whose base is table index `base`: the entry of window w goes to slot
// slot0 + w * win_stride, its key lies in bucket set set0 + (precomp ? 0 : w).  val = table index | sign<<31.
template <class Fr>
HD void msm_decompose_digits(const MsmPlan& pl, const Fr& scalar, uint32_t base, uint32_t set0, size_t slot0,
                             size_t win_stride, uint32_t* keys, uint32_t* vals) {
  constexpr int N = Fr::N;
  const Fr s = scalar.from_mont();
  uint32_t carry = 0;
  const uint32_t half = pl.set_size;  // 2^(c-1)
  const uint32_t mask = (pl.c == 32) ? 0xffffffffu : ((1u << pl.c) - 1u);
  for (int w = 0; w < pl.nwin; w++) {
    const int bit = w * pl.c;
    const int limb = bit >> 5, sh = bit & 31;
    uint32_t raw = 0;
    if (limb < N) {
      raw = s.l[limb] >> sh;
      if (sh + pl.c > 32 && limb + 1 < N) raw |= s.l[limb + 1] << (32 - sh);
    }
    raw &= mask;
    uint32_t d = raw + carry;
    uint32_t neg = 0;
    carry = 0;
    if (d >= half && w != pl.nwin - 1) {
      // digit d - 2^c < 0 ; |digit| = 2^c - d  (<= 2^(c-1))
      d = (1u << pl.c) - d; neg = 1; carry = 1;
    }
    const size_t slot = (size_t)w * win_stride + slot0;
    if (d == 0) {
      keys[slot] = pl.total_buckets;
      vals[slot] = 0;
    } else {
      const uint32_t set = set0 + (pl.precomp ? 0u : (uint32_t)w);
      keys[slot] = set * pl.set_size + (d - 1);
      const uint32_t ti = (pl.precomp ? (uint32_t)w * pl.table_stride : 0u) + base;
      vals[slot] = ti | (neg << 31);
    }
  }
}

// keys/vals are laid out [w][i] (coalesced per window).  The base of scalar i is table_off + i, or idx[i] when an index
// list is given (checked by msm_index_ok before the MSM is enqueued).
template <class Fr>
HD void msm_decompose_one(const MsmPlan& pl, uint32_t i, const Fr* scalars, uint32_t* keys, uint32_t* vals,
                          const uint32_t* idx = nullptr) {
  msm_decompose_digits<Fr>(pl, scalars[i], idx ? idx[i] : pl.table_off + i, 0u, i, pl.n, keys, vals);
}

// Batched MSM (msm_make_batch_plan): entry g = b * n + i is scalar i of item b, read at b * scalar_stride + i (32-bit:
// the caller keeps batch * scalar_stride below 2^32), base table_off + i as in the single MSM, keys in the item's own sets.
// Entries are laid out [w][b][i], so every window stays coalesced; with batch = 1 they are exactly msm_decompose_one's.
template <class Fr>
HD void msm_decompose_batch_one(const MsmPlan& pl, uint32_t g, const Fr* scalars, uint32_t* keys, uint32_t* vals) {
  const uint32_t b = g / pl.n, i = g - b * pl.n;
  const uint32_t item_sets = (uint32_t)pl.nsets / pl.batch;
  msm_decompose_digits<Fr>(pl, scalars[b * pl.scalar_stride + i], pl.table_off + i, b * item_sets, g, (size_t)pl.batch * pl.n,
                           keys, vals);
}

// ---- 3. accumulate ---------------------------------------------------------
template <class F>
HD Affine<F> msm_load_point(const Affine<F>* table, uint32_t val) {
  Affine<F> p = table[val & 0x7fffffffu];
  if (val >> 31) p.y = p.y.neg();
  return p;
}

template <class F>
HD XYZZ<F> msm_accumulate_range(const Affine<F>* table, const uint32_t* vals, uint32_t begin, uint32_t end) {
  XYZZ<F> acc = XYZZ<F>::inf();
  for (uint32_t e = begin; e < end; e++) acc.add_mixed(msm_load_point(table, vals[e]));
  return acc;
}

// entries [begin, end) of task t (false: t is past the last task); the same arithmetic as k_msm_accumulate
HD bool msm_task_bounds(const MsmPlan& pl, const uint32_t* off, const uint32_t* task_off, uint32_t t, uint32_t& begin,
                        uint32_t& end) {
  const uint32_t nb = pl.total_buckets;
  if (t >= task_off[nb]) return false;
  uint32_t lo = 0, hi = nb;
  while (lo < hi) {     // bucket of task t: largest b with task_off[b] <= t
    const uint32_t mid = lo + ((hi - lo + 1) >> 1);
    if (task_off[mid] <= t) lo = mid; else hi = mid - 1;
  }
  const uint32_t j = t - task_off[lo];
  begin = off[lo] + j * pl.task_len;
  end = begin + pl.task_len;
  if (end > off[lo + 1]) end = off[lo + 1];
  return true;
}

// ---- 5. reduce -------------------------------------------------------------
// chunk t of a set covers buckets [lo, hi) (set-local, weight of bucket k is k+1):
// returns sum_k (k+1) * B_k over the chunk.
template <class F>
HD XYZZ<F> msm_reduce_chunk(const XYZZ<F>* set_buckets, uint32_t lo, uint32_t hi) {
  XYZZ<F> run = XYZZ<F>::inf();   // sum_{j >= k} B_j
  XYZZ<F> acc = XYZZ<F>::inf();   // sum (k - lo + 1) B_k
  for (uint32_t k = hi; k-- > lo;) {
    run.add(set_buckets[k]);
    acc.add(run);
  }
  if (lo) acc.add(xyzz_mul_small(run, lo));
  return acc;
}

// Horner over bucket sets: sum_w 2^(c*w) * S_w
template <class F>
HD XYZZ<F> msm_horner(const XYZZ<F>* set_sums, int nsets, int c) {
  XYZZ<F> acc = set_sums[nsets - 1];
  for (int w = nsets - 2; w >= 0; w--) {
    for (int k = 0; k < c; k++) acc.dbl();
    acc.add(set_sums[w]);
  }
  return acc;
}

// ---- table precompute ------------------------------------------------------
// Jacobian-free: produce 2^c * P in affine with one inversion (used by the
// emulation / tiny tables; the kernel batches inversions, see msm_impl.cuh)
template <class F>
HD Affine<F> msm_shift_point(const Affine<F>& p, int c) {
  XYZZ<F> q = XYZZ<F>::from_affine(p);
  for (int k = 0; k < c; k++) q.dbl();
  return q.to_affine();
}

}  // namespace gb200
