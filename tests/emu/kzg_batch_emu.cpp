// CPU emulation of the batched polynomial kernels behind the KZG entry points (TEST ONLY): plonk.cuh's per-thread
// steps (poly_eval_chunk, syndiv_pre_chunk / syndiv_post_chunk / syndiv_zero_chunk, poly_fold_coeff) and the point
// tables (kzg_pow_len, kzg_pow_tables) compiled for the host with the PTX carry chains emulated, driven over the grid the
// device launches: one row per polynomial (blockIdx.y), 2048-coefficient eval / division blocks, and the per-row sum scan
// of scan_enqueue<Fr, 1, true> - 1024-element blocks, block totals scanned per row, recursively.  Used by
// tests/test_kzg_emulation.py; NOT loaded by the product.
#include <cstdint>
#include <vector>

#include "plonk.cuh"

using namespace gb200;

namespace {

constexpr size_t EVAL_BLOCK = 256 * EVAL_E;
constexpr size_t SCAN_BLOCK = (size_t)SCAN_THREADS * SCAN_E;

// k_scan_block<Fr, 1, true> on block blk of one row: its inclusive (or exclusive) prefix, its total to block_sums[blk]
template <class Fr>
void scan_block(Fr* data, size_t n, size_t blk, Fr* block_sums, bool exclusive) {
  Fr acc = Fr::zero();
  for (size_t i = blk * SCAN_BLOCK; i < (blk + 1) * SCAN_BLOCK; i++) {
    const Fr v = i < n ? data[i] : Fr::zero();
    if (i < n) data[i] = exclusive ? acc : acc + v;
    acc = acc + v;
  }
  if (block_sums) block_sums[blk] = acc;
}

// scan_enqueue<Fr, 1, true>(data, n, exclusive, rows)
template <class Fr>
void scan_rows(Fr* data, size_t n, bool exclusive, size_t rows) {
  if (n == 0) return;
  const size_t nblocks = (n + SCAN_BLOCK - 1) / SCAN_BLOCK;
  if (nblocks == 1) {
    for (size_t r = 0; r < rows; r++) scan_block<Fr>(data + r * n, n, 0, nullptr, exclusive);
    return;
  }
  std::vector<Fr> sums(rows * nblocks);
  for (size_t r = 0; r < rows; r++)
    for (size_t b = 0; b < nblocks; b++) scan_block<Fr>(data + r * n, n, b, sums.data() + r * nblocks, exclusive);
  scan_rows<Fr>(sums.data(), nblocks, true, rows);
  // k_scan_fix<Fr, 1, true>
  for (size_t r = 0; r < rows; r++)
    for (size_t b = 1; b < nblocks; b++)
      for (size_t i = b * SCAN_BLOCK; i < (b + 1) * SCAN_BLOCK && i < n; i++)
        data[r * n + i] = sums[r * nblocks + b] + data[r * n + i];
}

template <class Fr>
int eval_batch(const void* polys_, size_t n, size_t batch, const void* points, void* values_) {
  const Fr* polys = reinterpret_cast<const Fr*>(polys_);
  Fr* values = reinterpret_cast<Fr*>(values_);
  if (n == 0) {
    for (size_t b = 0; b < batch; b++) values[b] = Fr::zero();
    return 0;
  }
  const uint32_t len = kzg_pow_len(n);
  std::vector<Fr> pw(batch * len);
  kzg_pow_tables<Fr>(reinterpret_cast<const Fr*>(points), batch, len, false, pw.data());
  const size_t nblocks = (n + EVAL_BLOCK - 1) / EVAL_BLOCK;
  for (size_t b = 0; b < batch; b++) {
    const Fr* row_pw = pw.data() + b * len;
    std::vector<Fr> sums(nblocks);
    for (size_t blk = 0; blk < nblocks; blk++) {   // k_poly_eval_partial<Fr, true>
      Fr s = Fr::zero();
      for (size_t t = 0; t < 256; t++) s = s + poly_eval_chunk<Fr>(polys + b * n, n, row_pw, row_pw[0], (blk * 256 + t) * EVAL_E);
      sums[blk] = s;
    }
    Fr v = Fr::zero();                               // k_sum_reduce<Fr, true>
    for (size_t blk = 0; blk < nblocks; blk++) v = v + sums[blk];
    values[b] = v;
  }
  return 0;
}

template <class Fr>
int div_batch(const void* polys_, size_t n, size_t batch, const void* points, void* q_, void* values_) {
  const Fr* c = reinterpret_cast<const Fr*>(polys_);
  Fr* q = reinterpret_cast<Fr*>(q_);
  Fr* values = reinterpret_cast<Fr*>(values_);
  if (n == 0) {
    for (size_t b = 0; b < batch; b++) values[b] = Fr::zero();
    return 0;
  }
  const uint32_t len = kzg_pow_len(n);
  std::vector<Fr> pw(2 * batch * len);
  kzg_pow_tables<Fr>(reinterpret_cast<const Fr*>(points), batch, len, true, pw.data());
  const Fr* pwi = pw.data() + batch * len;
  std::vector<Fr> t(batch * n);
  const size_t nb = (n + EVAL_BLOCK - 1) / EVAL_BLOCK;
  for (size_t b = 0; b < batch; b++)                 // k_syndiv_pre<Fr, true>
    for (size_t th = 0; th < nb * 256; th++)
      syndiv_pre_chunk<Fr>(c + b * n, n, pwi + b * len, pwi[b * len], t.data() + b * n, th * EVAL_E);
  scan_rows<Fr>(t.data(), n, false, batch);
  for (size_t b = 0; b < batch; b++) {               // k_syndiv_post<Fr, true>
    const Fr* row_pw = pw.data() + b * len;
    for (size_t th = 0; th < nb * 256; th++) {
      if (row_pw[0].is_zero()) syndiv_zero_chunk<Fr>(c + b * n, n, q + b * n, values + b, th * EVAL_E);
      else syndiv_post_chunk<Fr>(t.data() + b * n, n, row_pw, row_pw[0], q + b * n, values + b, th * EVAL_E);
    }
  }
  return 0;
}

template <class Fr>
int fold(const void* polys, size_t n, size_t batch, const void* gamma, void* out) {
  for (size_t j = 0; j < n; j++)
    reinterpret_cast<Fr*>(out)[j] =
        poly_fold_coeff<Fr>(reinterpret_cast<const Fr*>(polys), n, batch, *reinterpret_cast<const Fr*>(gamma), j);
  return 0;
}

}  // namespace

#define GB_EMU_CURVE(CALL)                     \
  switch (curve) {                             \
    case 0: { using Fr = bn254_fr; return CALL; }      \
    case 1: { using Fr = bls12_381_fr; return CALL; }  \
    case 2: { using Fr = bls12_377_fr; return CALL; }  \
    case 3: { using Fr = bw6_761_fr; return CALL; }    \
  }                                            \
  return -1;

extern "C" int emu_poly_eval_batch(int curve, const void* polys, size_t n, size_t batch, const void* points, void* values) {
  GB_EMU_CURVE(eval_batch<Fr>(polys, n, batch, points, values))
}
// q: batch * n fr.Elements (row b: the quotient, top coefficient 0), values: batch
extern "C" int emu_poly_div_batch(int curve, const void* polys, size_t n, size_t batch, const void* points, void* q,
                                  void* values) {
  GB_EMU_CURVE(div_batch<Fr>(polys, n, batch, points, q, values))
}
extern "C" int emu_poly_fold(int curve, const void* polys, size_t n, size_t batch, const void* gamma, void* out) {
  GB_EMU_CURVE(fold<Fr>(polys, n, batch, gamma, out))
}
extern "C" uint32_t emu_kzg_pow_len(size_t n) { return kzg_pow_len(n); }
