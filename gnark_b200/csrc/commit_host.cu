// Witness-side MSMs of the Groth16 prover (SURVEY.md 8a-a8, 8f-4):
//
//  * Pedersen / BSB22 commitments - backend/groth16/bn254/prove.go:72-129: inside the solver hint
//    `pk.CommitmentKeys[i].Commit(privateCommittedValues[i])` (:84), after the solver
//    `pk.CommitmentKeys[i].ProveKnowledge(...)` (:114) and `proof.CommitmentPok.Fold(poks, challenge, ...)` (:127);
//    GPU twin backend/accelerated/icicle/groth16/bn254/icicle.go:825-889,904-964.  Commit and ProveKnowledge are MSMs of
//    the SAME scalars over the key's two bases (Basis, BasisExpSigma), so one entry point uploads the scalars once and
//    runs both; Fold is a handful of host-side scalar multiplications.  Hashing the commitment to a field element (the
//    hint's output, :90-98) stays in Go.
//  * gather-index MSM - prove.go:147-168 copies the wire values whose base is not infinity into fresh slices
//    ("worst memory allocation offender", :232); here the table is the filtered bases and the scalars are gathered on
//    the device through an index list: sum_j scalars[idx[j]] * bases[off + j].
#include "capi_common.h"

using namespace gb200;

struct b200_pedersen_key_s {
  int dev = 0, curve = 0;
  size_t n = 0;
  b200_table_t basis = nullptr, basis_sigma = nullptr;
};

extern "C" {

int32_t b200_pedersen_key_free(b200_pedersen_key_t key) {
  GUARD_BEGIN
  if (!key) return 0;
  int32_t rc = b200_table_free(key->basis);
  int32_t rc2 = b200_table_free(key->basis_sigma);
  delete key;
  return rc ? rc : rc2;
  GUARD_END
}

int32_t b200_pedersen_key_load(int32_t dev, int32_t curve, const void* basis, const void* basis_exp_sigma, size_t n,
                               b200_pedersen_key_t* out) {
  GUARD_BEGIN
  if (!out || (n && (!basis || !basis_exp_sigma))) return set_error("pedersen_key_load: null argument");
  std::unique_ptr<b200_pedersen_key_s> key(new b200_pedersen_key_s());
  key->dev = dev; key->curve = curve; key->n = n;
  // committed-wire counts are small next to the circuit (usually << 2^16): plain tables unless the basis is large
  const int32_t flags = n >= ((size_t)1 << 14) ? B200_TABLE_PRECOMP : 0;
  int32_t rc = b200_table_upload(dev, curve, 1, basis, n, flags, &key->basis);
  if (!rc) rc = b200_table_upload(dev, curve, 1, basis_exp_sigma, n, flags, &key->basis_sigma);
  if (rc) {
    std::string m = b200_last_error();
    b200_pedersen_key_free(key.release());
    set_error(m);
    return rc;
  }
  *out = key.release();
  return 0;
  GUARD_END
}

int32_t b200_pedersen_commit(b200_pedersen_key_t key, const void* values, size_t n, int32_t values_on_device,
                             void* out_commitment, void* out_pok) {
  GUARD_BEGIN
  if (!key) return set_error("pedersen_commit: null key");
  if (n != key->n) return set_error("pedersen_commit: " + std::to_string(n) + " values for a basis of " + std::to_string(key->n) +
                                    " points (pedersen.ProvingKey.Commit requires equal lengths)");
  if (n && !values) return set_error("pedersen_commit: null values");
  if (!out_commitment && !out_pok) return 0;
  GB_DEVICE(ctx, key->dev);
  const MsmOps* ops = key->basis->ops;
  const HostGroupOps* h = get_host_group_ops(key->curve, 1);
  std::vector<uint8_t> host(2 * ops->jac_bytes);
  Staging st(ctx);
  void* d_res;
  const void* sc;
  CK(st.out(host.data(), host.size(), false, &d_res));
  CK(st.in(values, n * ops->fr_bytes, values_on_device, &sc));
  char* res = reinterpret_cast<char*>(d_res);
  int32_t rc = 0;
  if (out_commitment) rc = msm_on_stream(ctx, key->basis, 0, n, sc, res, nullptr, true);
  if (!rc && out_pok) rc = msm_on_stream(ctx, key->basis_sigma, 0, n, sc, res + ops->jac_bytes, nullptr, true);
  if (!rc) rc = msm_join(ctx);
  rc = st.finish("pedersen_commit", rc);
  if (rc) return rc;
  // affine on the host, after the sync
  if (out_commitment) h->to_affine(host.data(), out_commitment);
  if (out_pok) h->to_affine(host.data() + ops->jac_bytes, out_pok);
  return 0;
  GUARD_END
}

// pedersen.ProofOfKnowledge.Fold (prove.go:127): sum_i challenge^i * poks[i]; host CPU, `count` is the number of commitments
int32_t b200_pedersen_fold(int32_t curve, const void* poks_affine, size_t count, const void* challenge, void* out_affine) {
  GUARD_BEGIN
  const HostGroupOps* h = get_host_group_ops(curve, 1);
  const NttOps* fr = get_ntt_ops(curve);
  if (!h || !fr) return set_error("pedersen_fold: unsupported curve");
  if (!out_affine || (count && (!poks_affine || !challenge))) return set_error("pedersen_fold: null argument");
  const HostFrCtx* F = fr->host_fr();
  std::vector<uint8_t> acc(h->jac_bytes, 0), term(h->jac_bytes), kb(8 * HOSTFR_MAX_LIMBS);
  // infinity in gnark's Jacobian layout: Z = 0 (X = Y = 1 by convention; add_jac only looks at Z)
  const uint8_t* p = reinterpret_cast<const uint8_t*>(poks_affine);
  HostFr pw = F->one_();
  const HostFr c = count ? F->load(challenge) : F->one_();
  bool first = true;
  for (size_t i = 0; i < count; i++) {
    F->store(kb.data(), pw);
    h->scalar_mul_affine(p + i * h->affine_bytes, kb.data(), term.data());
    if (first) { acc = term; first = false; }
    else h->add_jac(acc.data(), term.data());
    pw = F->mul(pw, c);
  }
  if (first) { memset(out_affine, 0, h->affine_bytes); return 0; }     // no commitments: the point at infinity (0, 0)
  h->to_affine(acc.data(), out_affine);
  return 0;
  GUARD_END
}

// sum_j scalars[idx[j]] * bases[off + j], j < n_idx: scalars gathered on the device through an index list (wire
// filtering without host copies, prove.go:147-168,231-235)
int32_t b200_msm_gather(b200_table_t t, size_t off, const uint32_t* idx, size_t n_idx, int32_t idx_on_device,
                        const void* scalars, size_t n_scalars, int32_t scalars_on_device, void* out_jac_host) {
  GUARD_BEGIN
  if (!t) return set_error("msm_gather: null table");
  if (!out_jac_host || (n_idx && (!idx || !scalars))) return set_error("msm_gather: null argument");
  GB_DEVICE(ctx, t->dev);
  const NttOps* fr = get_ntt_ops(t->curve);
  if (!fr) return set_error("msm_gather: unsupported curve");
  if (!idx_on_device)
    for (size_t j = 0; j < n_idx; j++)
      if (idx[j] >= n_scalars) return set_error("msm_gather: index " + std::to_string(idx[j]) + " out of range at position " + std::to_string(j));
  const size_t fb = t->ops->fr_bytes;
  Staging st(ctx);
  void *d_out, *d_g;
  const void *sc, *ix;
  CK(st.out(out_jac_host, t->ops->jac_bytes, false, &d_out));
  CK(st.in(scalars, n_scalars * fb, scalars_on_device, &sc));
  CK(st.in(idx, n_idx * sizeof(uint32_t), idx_on_device, &ix));
  CK(st.scratch(n_idx * fb, &d_g));
  if (n_idx) CK(fr->gather(ctx->stream, d_g, sc, static_cast<const uint32_t*>(ix), n_idx));
  return st.finish("msm_gather", msm_on_stream(ctx, t, off, n_idx, d_g, d_out));
  GUARD_END
}

}  // extern "C"

// first_bad = the lowest position j < n with idx[j] >= count (stays 0xffffffff when every index is valid)
static __global__ void __launch_bounds__(256) k_msm_check_indices(const uint32_t* __restrict__ idx, uint32_t n,
                                                                  uint32_t count, uint32_t* __restrict__ first_bad) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n && !msm_index_ok(idx, j, count)) atomicMin(first_bad, j);
}

extern "C" {

// sum_j scalars[j] * bases[idx[j]], j < n: the bases are picked from the table through the index list (any order, repeats
// allowed) - a sparse vector committed against a whole table (the BSB22 hint's kzg.Commit over pk.KzgLagrange,
// backend/plonk/bn254/prove.go:280-315) at a cost that follows n, not the table size.  Every index is checked before any
// kernel reads a point through it: host indices here, device indices by k_msm_check_indices, whose verdict is downloaded
// (one synchronisation) before the MSM is enqueued.
int32_t b200_msm_indexed(b200_table_t t, const uint32_t* idx, size_t n, int32_t idx_on_device, const void* scalars,
                         int32_t scalars_on_device, void* out_jac_host) {
  GUARD_BEGIN
  if (!t) return set_error("msm_indexed: null table");
  if (!out_jac_host || (n && (!idx || !scalars))) return set_error("msm_indexed: null argument");
  if (n >= ((size_t)1 << 31)) return set_error("msm_indexed: n * windows exceeds 2^31 entries - split the call and add the results");
  GB_DEVICE(ctx, t->dev);
  if (!idx_on_device)
    for (size_t j = 0; j < n; j++)
      if (idx[j] >= t->n)
        return set_error("msm_indexed: index " + std::to_string(idx[j]) + " out of range at position " + std::to_string(j) +
                         " (table of " + std::to_string(t->n) + " points)");
  Staging st(ctx);
  void* d_out;
  const void *sc, *ix;
  CK(st.out(out_jac_host, t->ops->jac_bytes, false, &d_out));
  CK(st.in(idx, n * sizeof(uint32_t), idx_on_device, &ix));
  CK(st.in(scalars, n * t->ops->fr_bytes, scalars_on_device, &sc));
  if (idx_on_device && n) {
    void* d_bad;
    uint32_t bad = 0;
    CK(st.scratch(sizeof(uint32_t), &d_bad));
    CK(cudaMemsetAsync(d_bad, 0xff, sizeof(uint32_t), ctx->stream));
    k_msm_check_indices<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(static_cast<const uint32_t*>(ix), (uint32_t)n,
                                                                             (uint32_t)t->n, static_cast<uint32_t*>(d_bad));
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(&bad, d_bad, sizeof(bad), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (bad != 0xffffffffu)
      return st.finish("msm_indexed", set_error("msm_indexed: device index out of range at position " + std::to_string(bad) +
                                                " (table of " + std::to_string(t->n) + " points)"));
  }
  return st.finish("msm_indexed", msm_on_stream(ctx, t, 0, n, sc, d_out, nullptr, false, static_cast<const uint32_t*>(ix)));
  GUARD_END
}

}  // extern "C"
