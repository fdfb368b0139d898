// KZG on the device (declared in include/gnark_b200.h): evaluation of a batch of polynomials, kzg.Open of a batch
// (one batched division by (X - z_b), one batched MSM of the quotients) and the H of kzg.BatchOpenSinglePoint (the
// gamma-fold, one division, one MSM).  Commitments need nothing here: a batch of them is b200_msm_batch on the SRS.
// Every call is synchronous and synchronises once, when its results come down.
#include "capi_common.h"

namespace gb200 {

// The refusals of a quotient MSM over srs[0, n - 1) for `batch` polynomials of n coefficients, checked before anything
// is allocated: a G2 table, n - 1 beyond the table, batch * n * sizeof(fr.Element) beyond size_t, the batched MSM's
// index limits.  *c: the MSM window: a precomputed table's own, else that of an n-point MSM (the polynomial's length,
// not n - 1: on an SRS of 2^k points the quotient MSM then takes the window b200_msm takes on it).
static int32_t kzg_check(const char* what, const b200_table_s* t, size_t n, size_t batch, size_t msm_batch, int* c) {
  const std::string w(what);
  if (t->group != 1) return set_error(w + ": the SRS table holds G2 points; KZG opens over a G1 table");
  const size_t m = n ? n - 1 : 0;
  if (m > t->n)
    return set_error(w + ": n - 1 = " + std::to_string(m) + " quotient coefficients exceed the SRS's " +
                     std::to_string(t->n) + " points");
  const NttOps* fr = get_ntt_ops(t->curve);
  if (!fr) return set_error(w + ": unsupported curve");
  if ((unsigned __int128)batch * n * fr->fr_bytes > (unsigned __int128)SIZE_MAX)
    return set_error(w + ": batch * n overflows");
  *c = t->precomp ? t->c : msm_window_with_limit(n, t->ops->scalar_bits);
  if (m && msm_batch) {
    const size_t most = msm_max_batch(t, m, *c);
    if (msm_batch > most)
      return set_error(w + ": batch * (n - 1) * windows must stay below 2^31 and batch * bucket sets * 2^(c-1) below 2^31 - 1; "
                       "at most " + std::to_string(most) + " items of this n fit - split the batch");
  }
  return 0;
}

// `batch` MSMs of m scalars each over srs[0, m): item b's scalars at d_scalars + b * stride
static cudaError_t kzg_msm(DeviceCtx* ctx, Staging& st, const b200_table_s* t, size_t m, size_t batch, size_t stride, int c,
                           const void* d_scalars, void* d_out) {
  const int nwin = msm_num_windows(t->ops->scalar_bits, c);
  uint32_t task_len, chunk;
  msm_tuning(m, batch, nwin, c, t->precomp, t->ops->acc_blocks_per_sm(), &task_len, &chunk);
  size_t ws_bytes = 0;    // m = 0 writes `batch` points at infinity and needs no workspace
  if (m) {
    cudaError_t e = t->ops->ws_bytes((uint32_t)m, (uint32_t)batch, (uint32_t)t->n, c, t->precomp, task_len, chunk, &ws_bytes);
    if (e != cudaSuccess) return e;
  }
  void* ws;
  cudaError_t e = st.scratch(ws_bytes, &ws);
  if (e != cudaSuccess) return e;
  return t->ops->run(ctx->stream, (uint32_t)m, (uint32_t)batch, (uint32_t)t->n, 0, c, t->precomp, task_len, chunk,
                     t->d_points, d_scalars, d_out, ws, nullptr, nullptr, nullptr, (uint32_t)stride);
}

}  // namespace gb200

using namespace gb200;

extern "C" {

int32_t b200_poly_eval_batch(int32_t dev, int32_t curve, const void* polys, size_t n, size_t batch, int32_t polys_on_dev,
                             const void* points_mont, void* values_host) {
  GUARD_BEGIN
  const NttOps* fr = get_ntt_ops(curve);
  if (!fr) return set_error("poly_eval_batch: unsupported curve");
  if (!points_mont || !values_host || (batch && n && !polys)) return set_error("poly_eval_batch: null argument");
  if ((unsigned __int128)batch * n * fr->fr_bytes > (unsigned __int128)SIZE_MAX)
    return set_error("poly_eval_batch: batch * n overflows");
  if (batch == 0) return 0;
  GB_DEVICE(ctx, dev);
  int32_t rc = msm_join(ctx); if (rc) return rc;
  Staging st(ctx);
  const void* d_polys;
  void* d_values;
  CK(st.in(polys, batch * n * fr->fr_bytes, polys_on_dev, &d_polys));
  CK(st.out(values_host, batch * fr->fr_bytes, false, &d_values));
  return st.finish("poly_eval_batch", fr->poly_eval_batch(ctx->stream, d_polys, n, batch, points_mont, d_values));
  GUARD_END
}

int32_t b200_kzg_open_batch(b200_table_t srs, const void* polys, size_t n, size_t batch, int32_t polys_on_dev,
                            const void* points_mont, void* values_host, void* proofs_jac_host) {
  GUARD_BEGIN
  if (!srs) return set_error("kzg_open_batch: null table");
  if (!points_mont || !values_host || !proofs_jac_host || (batch && n && !polys))
    return set_error("kzg_open_batch: null argument");
  int c = 0;
  int32_t rc = kzg_check("kzg_open_batch", srs, n, batch, batch, &c); if (rc) return rc;
  if (batch == 0) return 0;
  const NttOps* fr = get_ntt_ops(srs->curve);
  const size_t fb = fr->fr_bytes;
  GB_DEVICE(ctx, srs->dev);
  rc = msm_join(ctx); if (rc) return rc;
  Staging st(ctx);
  const void* d_polys;
  void *d_values, *d_proofs, *d_q;
  CK(st.in(polys, batch * n * fb, polys_on_dev, &d_polys));
  CK(st.out(values_host, batch * fb, false, &d_values));
  CK(st.out(proofs_jac_host, batch * srs->ops->jac_bytes, false, &d_proofs));
  CK(st.scratch(batch * n * fb, &d_q));
  cudaError_t e = fr->poly_div_linear_batch(ctx->stream, d_polys, n, batch, points_mont, d_q, d_values);
  if (e == cudaSuccess) e = kzg_msm(ctx, st, srs, n ? n - 1 : 0, batch, n, c, d_q, d_proofs);
  return st.finish("kzg_open_batch", e);
  GUARD_END
}

int32_t b200_kzg_fold_open(b200_table_t srs, const void* polys, size_t n, size_t batch, int32_t polys_on_dev,
                           const void* z_mont, const void* gamma_mont, void* proof_jac_host) {
  GUARD_BEGIN
  if (!srs) return set_error("kzg_fold_open: null table");
  if (!z_mont || !gamma_mont || !proof_jac_host || (batch && n && !polys)) return set_error("kzg_fold_open: null argument");
  int c = 0;
  int32_t rc = kzg_check("kzg_fold_open", srs, n, batch, 1, &c); if (rc) return rc;
  if (batch == 0) return 0;
  const NttOps* fr = get_ntt_ops(srs->curve);
  const size_t fb = fr->fr_bytes;
  GB_DEVICE(ctx, srs->dev);
  rc = msm_join(ctx); if (rc) return rc;
  Staging st(ctx);
  const void* d_polys;
  void *d_proof, *d_f, *d_q, *d_value;
  CK(st.in(polys, batch * n * fb, polys_on_dev, &d_polys));
  CK(st.out(proof_jac_host, srs->ops->jac_bytes, false, &d_proof));
  CK(st.scratch(n * fb, &d_f));
  CK(st.scratch(n * fb, &d_q));
  CK(st.scratch(fb, &d_value));
  cudaError_t e = fr->poly_fold(ctx->stream, d_polys, n, batch, gamma_mont, d_f);
  if (e == cudaSuccess) e = fr->poly_div_linear_batch(ctx->stream, d_f, n, 1, z_mont, d_q, d_value);
  if (e == cudaSuccess) e = kzg_msm(ctx, st, srs, n ? n - 1 : 0, 1, n, c, d_q, d_proof);
  return st.finish("kzg_fold_open", e);
  GUARD_END
}

}  // extern "C"
