// PLONK prover orchestration on the host, over the C ABI's own device entry points - the compiled twin of
// gnark_b200/plonk.py and, stage by stage, of the CPU prover backend/plonk/bn254/prove.go:
//
//   commitToLRO :404-489           canonical forms (iNTT), blinding :1211-1220, 3 MSMs on the canonical SRS
//   buildRatioCopyConstraint :635  b200_plonk_build_z, commit Z
//   computeQuotient :558-633       48 coset NTTs + fused constraint kernel x4 :841-1123, divideByZH :1287,
//                                  commitToQuotient :1263-1282
//   openZ :670-687, computeLinearizedPolynomial :724-794 (+ :1366-1487), batchOpening :796-837
//
// Every polynomial stays in HBM between the MSM / NTT stages; only blinding patches (<= 3 elements), opened
// values and digests cross to the host.  Challenges and blinding coefficients are INPUTS (the Fiat-Shamir
// transcript encoding is gnark-crypto's; a Go shim derives them exactly as prove.go:492-555 does).  BSB22 commitment
// gates (:867-884) are supported with the committed polynomials PI2_i supplied by the caller (the reference's solver
// hint :280-318 produces them), and so is StatisticalZK (:239-242,689-722,1476-1481: the two quotient-shard randomisers are
// inputs like the blinding coefficients).  Host-side scalar work uses host_fr.h.
#include <chrono>
#include <memory>
#include <vector>

#include "capi_common.h"

using namespace gb200;

namespace gb200_plonk {

// index of a key polynomial: the fixed ones, then the BSB22 selectors Qcp_j (trace.Qcp) at QCP0 + j
enum { QL = 0, QR, QM, QO, QK, S1, S2, S3, QCP0 };

// a key polynomial's canonical coefficients, in the two layouts the prover reads
struct KeyPoly {
  void* br = nullptr;                 // bit-reversed (input of the coset NTTs)
  void* canon = nullptr;              // regular
};

#define RC(x)                        \
  do {                               \
    int32_t rc__ = (x);              \
    if (rc__) return rc__;           \
  } while (0)

// stream-ordered device buffers, released on scope exit in the device stream's order (no host synchronisation)
struct Scratch {
  int dev;
  std::vector<void*> bufs;
  explicit Scratch(int d) : dev(d) {}
  ~Scratch() { for (void* p : bufs) if (p) scratch_free(dev, p); }
  int32_t alloc(size_t bytes, void** out) {
    RC(scratch_alloc(dev, bytes, out));
    bufs.push_back(*out);
    return 0;
  }
};

}  // namespace gb200_plonk
using namespace gb200_plonk;

struct b200_plonk_pk_s {
  int dev = 0, curve = 0;
  uint32_t logn = 0;
  size_t n = 0;
  size_t fb = 0;                      // sizeof(fr.Element)
  const HostFrCtx* fr = nullptr;
  HostFr g, w, w4;                    // FrMultiplicativeGen, domain0 generator, domain1 generator (Montgomery)
  b200_domain_t dom0[4] = {nullptr, nullptr, nullptr, nullptr};   // domain0 with coset generator g * w4^i
  b200_domain_t dom1 = nullptr;
  uint32_t n_qcp = 0;                 // BSB22 commitment gates
  std::vector<KeyPoly> key;           // QCP0 + n_qcp polynomials, by the index above
  int64_t* d_perm = nullptr;
  b200_table_t srs = nullptr;         // canonical SRS, n + 3 points
  // The key polynomials never change between proofs: their evaluations on the four cosets of the quotient domain
  // are computed once at key load and kept in HBM ((8 + n_qcp) x 4 x n elements: 4 GiB at n = 2^22 with 32-byte
  // elements), so a proof runs 16 coset NTTs (l, r, o, z) instead of 48.  key_cos[i][k]: coset i, key polynomial k;
  // empty when GB200_PLONK_COSET_CACHE=0.
  std::vector<std::vector<void*>> key_cos;
  // wall-clock ms of the five stages of the last b200_plonk_prove on this key (every stage ends in a b200_sync, so
  // these are device times + host orchestration): begin (L,R,O), commit_z, quotient, linearise, batch_open
  double last_stage_ms[5] = {0, 0, 0, 0, 0};
};

// one proof in flight: what the later Fiat-Shamir rounds need from the earlier ones
struct b200_plonk_session_s {
  b200_plonk_pk_s* pk;
  Scratch S;
  int stage = 0;
  size_t jb = 0;
  void *d_l = nullptr, *d_r = nullptr, *d_o = nullptr;
  void* cb[4] = {nullptr};        // l, r, o, z: canonical, bit-reversed (n)
  void* bl[4] = {nullptr};        // blinded canonical regular (n + 2, n + 2, n + 2, n + 3)
  std::vector<void*> pi2_br, pi2_canon;   // BSB22 committed polynomials, canonical (bit-reversed / regular)
  // per-proof Qk (b200_plonk_set_qk): the key's Qk with the public inputs and the BSB22 commitment values folded in
  // (completeQk, prove.go:349-373); canonical bit-reversed / regular, nullptr = the key's own Qk
  void *qk_br = nullptr, *qk_canon = nullptr;
  void* h = nullptr;              // quotient, canonical regular (4n)
  void* lin = nullptr;            // linearised polynomial (n + 3)
  // field elements kept as bytes; 16-byte aligned because callees may read them as limb structs
  alignas(16) uint8_t blind[4][3 * 8 * HOSTFR_MAX_LIMBS];   // bl, br, bo (2 each), bz (3)
  alignas(16) uint8_t beta[8 * HOSTFR_MAX_LIMBS], gamma[8 * HOSTFR_MAX_LIMBS], alpha[8 * HOSTFR_MAX_LIMBS], zeta[8 * HOSTFR_MAX_LIMBS];
  // StatisticalZK: quotientShardsRandomizers b1, b2 (b200_plonk_set_quotient_randomizers); szk = false: plain shards
  alignas(16) uint8_t hr[2][8 * HOSTFR_MAX_LIMBS];
  bool szk = false;
  explicit b200_plonk_session_s(b200_plonk_pk_s* p) : pk(p), S(p->dev) {}
};

namespace {

int32_t d2d(int dev, void* dst, const void* src, size_t bytes) {
  GB_DEVICE(ctx, dev);
  CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
  return 0;
}
int32_t dzero(int dev, void* dst, size_t bytes) {
  GB_DEVICE(ctx, dev);
  CK(cudaMemsetAsync(dst, 0, bytes, ctx->stream));
  return 0;
}

// Lagrange/regular values (n elements, on the host or the device) -> cb: canonical, bit-reversed ; reg: canonical,
// regular (its first n elements)
int32_t to_canonical(b200_plonk_pk_s* pk, const void* lagrange, bool on_host, void* cb, void* reg) {
  const size_t bytes = pk->n * pk->fb;
  RC(on_host ? b200_h2d(pk->dev, cb, lagrange, bytes) : d2d(pk->dev, cb, lagrange, bytes));
  RC(b200_ntt_async(pk->dom0[0], cb, 1, B200_DIF, 0));
  RC(d2d(pk->dev, reg, cb, bytes));
  return b200_vec_bit_reverse(pk->dev, pk->curve, reg, pk->logn);
}

// canonical, bit-reversed (n elements) -> dst: values on coset i of the quotient domain, regular
int32_t to_coset(b200_plonk_pk_s* pk, uint32_t i, const void* cb, void* dst) {
  RC(d2d(pk->dev, dst, cb, pk->n * pk->fb));
  return b200_ntt_async(pk->dom0[i], dst, 0, B200_DIT, 1);
}

// Lagrange/regular values (device, n elements) -> cb: canonical, bit-reversed (n) ; reg: canonical, regular,
// blinded p + b(X)(X^n - 1) with nb blinding coefficients (n + nb elements)     (getBlindedCoefficients :1211-1220)
int32_t canonical_blinded(b200_plonk_pk_s* pk, const void* d_lagrange, const uint8_t* b_mont, int nb, void* cb, void* reg) {
  const size_t n = pk->n, fb = pk->fb;
  RC(to_canonical(pk, d_lagrange, false, cb, reg));
  std::vector<uint8_t> low((size_t)nb * fb);
  RC(b200_d2h(pk->dev, low.data(), reg, (size_t)nb * fb));
  for (int i = 0; i < nb; i++) {       // low coefficients minus b_i (Montgomery form subtracts as is)
    const HostFr v = pk->fr->sub(pk->fr->load(low.data() + (size_t)i * fb), pk->fr->load(b_mont + (size_t)i * fb));
    pk->fr->store(low.data() + (size_t)i * fb, v);
  }
  RC(b200_h2d(pk->dev, reg, low.data(), (size_t)nb * fb));
  RC(b200_h2d(pk->dev, (uint8_t*)reg + n * fb, b_mont, (size_t)nb * fb));   // b on top
  return 0;
}

// element `idx` of a device vector += delta (one element crosses to the host and back, like the blinding patches)
int32_t add_to_element(b200_plonk_pk_s* pk, void* d_vec, size_t idx, const HostFr& delta) {
  alignas(16) uint8_t e[8 * HOSTFR_MAX_LIMBS];
  uint8_t* p = (uint8_t*)d_vec + idx * pk->fb;
  RC(b200_d2h(pk->dev, e, p, pk->fb));
  pk->fr->store(e, pk->fr->add(pk->fr->load(e), delta));
  return b200_h2d(pk->dev, p, e, pk->fb);
}

int32_t commit(b200_plonk_pk_s* pk, const void* d_coeffs, size_t count, void* out_jac) {
  return b200_msm_g1(pk->srs, 0, count, d_coeffs, 1, out_jac);
}

// Independent commitments of one round (L, R, O; H1, H2, H3) go through the pipelined MSM: results stay on the device,
// the reduction tail of one MSM and the upload / transforms of the next polynomial run under the next accumulate, and
// ONE join + download ends the round (the synchronous commit() pays a tail and a download per commitment).
int32_t commit_async(b200_plonk_pk_s* pk, const void* d_coeffs, size_t count, void* d_out_jac) {
  return b200_msm_pipelined(pk->srs, 0, count, d_coeffs, d_out_jac);
}
int32_t commit_join(b200_plonk_pk_s* pk, const void* d_res, size_t bytes, void* out_host) {
  RC(b200_msm_join(pk->dev));
  return b200_d2h(pk->dev, out_host, d_res, bytes);
}

int32_t eval_at(b200_plonk_pk_s* pk, const void* d_coeffs, size_t count, const HostFr& x, HostFr* out) {
  alignas(16) uint8_t xb[8 * HOSTFR_MAX_LIMBS], ob[8 * HOSTFR_MAX_LIMBS];
  pk->fr->store(xb, x);
  RC(b200_poly_eval(pk->dev, pk->curve, d_coeffs, count, xb, ob));
  *out = pk->fr->load(ob);
  return 0;
}
int32_t axpy(b200_plonk_pk_s* pk, void* d_y, const HostFr& a, const void* d_x, size_t count) {
  alignas(16) uint8_t ab[8 * HOSTFR_MAX_LIMBS];
  pk->fr->store(ab, a);
  return b200_vec_axpy(pk->dev, pk->curve, d_y, ab, d_x, count);
}

// the polynomials of the batch opening, in the order of BatchedProof.ClaimedValues (:796-807): linearised, l, r, o,
// s1, s2, then the Qcp_j
struct Opened { const void* p; size_t count; };
std::vector<Opened> opened(const b200_plonk_session_s* s) {
  const b200_plonk_pk_s* pk = s->pk;
  const size_t n = pk->n;
  std::vector<Opened> o = {{s->lin, n + 3}, {s->bl[0], n + 2}, {s->bl[1], n + 2}, {s->bl[2], n + 2},
                           {pk->key[S1].canon, n}, {pk->key[S2].canon, n}};
  for (uint32_t j = 0; j < pk->n_qcp; j++) o.push_back({pk->key[QCP0 + j].canon, n});
  return o;
}

}  // namespace

extern "C" {

int32_t b200_plonk_pk_free(b200_plonk_pk_t pk) {
  GUARD_BEGIN
  if (!pk) return 0;
  b200_sync(pk->dev);
  for (int i = 0; i < 4; i++) if (pk->dom0[i]) b200_ntt_domain_free(pk->dom0[i]);
  if (pk->dom1) b200_ntt_domain_free(pk->dom1);
  if (pk->d_perm) b200_free(pk->dev, pk->d_perm);
  for (size_t k = 0; k < pk->key.size(); k++) {
    std::vector<void*> bufs = {pk->key[k].br, pk->key[k].canon};
    for (auto& c : pk->key_cos) bufs.push_back(c[k]);
    for (void* q : bufs) if (q) b200_free(pk->dev, q);
  }
  if (pk->srs) b200_table_free(pk->srs);
  delete pk;
  return 0;
  GUARD_END
}

int32_t b200_plonk_pk_load(int32_t dev, int32_t curve, const b200_plonk_pk_desc* d, b200_plonk_pk_t* out) {
  GUARD_BEGIN
  if (!d || !out) return set_error("plonk_pk_load: null argument");
  if (!d->ql || !d->qr || !d->qm || !d->qo || !d->qk || !d->perm || !d->srs_canonical)
    return set_error("plonk_pk_load: null field in the descriptor");
  if (d->n_qcp > 16 || (d->n_qcp && !d->qcp)) return set_error("plonk_pk_load: invalid BSB22 selector list");
  for (uint32_t j = 0; j < d->n_qcp; j++)
    if (!d->qcp[j]) return set_error("plonk_pk_load: null BSB22 selector");
  const NttOps* ops = get_ntt_ops(curve);
  if (!ops) return set_error("plonk_pk_load: unsupported curve");
  if ((int)d->log2n + 2 > ops->two_adicity || d->log2n > 28) return set_error("plonk_pk_load: domain too large");
  // the quotient is read as three slices of n + 2 coefficients out of a 4n buffer (h1, h2, h3): 3 (n + 2) <= 4n needs
  // n >= 8 (the reference switches to an 8n quotient domain below 6 constraints, setup.go; not supported here)
  if (d->log2n < 3) return set_error("plonk_pk_load: domains below 2^3 are not supported");
  GB_DEVICE(ctx, dev);
  std::unique_ptr<b200_plonk_pk_s, int32_t (*)(b200_plonk_pk_t)> pk(new b200_plonk_pk_s(), &b200_plonk_pk_free);
  pk->dev = dev; pk->curve = curve; pk->logn = d->log2n; pk->n = (size_t)1 << d->log2n;
  pk->fb = ops->fr_bytes;
  const HostFrCtx* fr = pk->fr = ops->host_fr();
  const size_t n = pk->n, fb = pk->fb;
  pk->g = fr->mult_gen;
  pk->w = fr->domain_generator((int)d->log2n);
  pk->w4 = fr->domain_generator((int)d->log2n + 2);
  // domain0 handles for the four cosets g * w4^i (computeNumerator :943-948) and the big domain
  HostFr coset = pk->g;
  for (int i = 0; i < 4; i++) {
    alignas(16) uint8_t cb[8 * HOSTFR_MAX_LIMBS];
    fr->store(cb, coset);
    RC(b200_ntt_domain_new(dev, curve, d->log2n, nullptr, cb, &pk->dom0[i]));
    coset = fr->mul(coset, pk->w4);
  }
  RC(b200_ntt_domain_new(dev, curve, d->log2n + 2, nullptr, nullptr, &pk->dom1));
  RC(b200_alloc(dev, 3 * n * sizeof(int64_t), (void**)&pk->d_perm));
  RC(b200_h2d(dev, pk->d_perm, d->perm, 3 * n * sizeof(int64_t)));
  for (size_t i = 0; i < 3 * n; i++)
    if (d->perm[i] < 0 || (uint64_t)d->perm[i] >= 3 * n) return set_error("plonk_pk_load: permutation entry out of range");
  // sigma polynomials from the permutation: s_j[i] = supp[perm[j n + i]], supp = <w> || g<w> || g^2<w>
  // (setup.go:289-392); host side, once per key
  std::vector<uint8_t> wpow(n * fb), sj(n * fb);
  {
    HostFr acc = fr->one_();
    for (size_t i = 0; i < n; i++) { fr->store(wpow.data() + i * fb, acc); acc = fr->mul(acc, pk->w); }
  }
  const HostFr g2 = fr->mul(pk->g, pk->g);
  const void* lag[QCP0] = {d->ql, d->qr, d->qm, d->qo, d->qk, nullptr, nullptr, nullptr};
  pk->n_qcp = d->n_qcp;
  pk->key.resize(QCP0 + d->n_qcp);
  for (size_t k = 0; k < pk->key.size(); k++) {
    const void* src = k < QCP0 ? lag[k] : d->qcp[k - QCP0];
    if (k >= S1 && k <= S3) {
      const int j = k - S1;
      for (size_t i = 0; i < n; i++) {
        const uint64_t idx = (uint64_t)d->perm[(size_t)j * n + i];
        HostFr v = fr->load(wpow.data() + (idx % n) * fb);
        if (idx / n == 1) v = fr->mul(v, pk->g);
        else if (idx / n == 2) v = fr->mul(v, g2);
        fr->store(sj.data() + i * fb, v);
      }
      src = sj.data();
    }
    RC(b200_alloc(dev, n * fb, &pk->key[k].br));
    RC(b200_alloc(dev, n * fb, &pk->key[k].canon));
    RC(to_canonical(pk.get(), src, true, pk->key[k].br, pk->key[k].canon));
  }
  const char* e = getenv("GB200_PLONK_COSET_CACHE");
  if (!e || atoi(e) != 0) {
    pk->key_cos.assign(4, std::vector<void*>(pk->key.size(), nullptr));
    for (uint32_t i = 0; i < 4; i++)
      for (size_t k = 0; k < pk->key.size(); k++) {
        RC(b200_alloc(dev, n * fb, &pk->key_cos[i][k]));
        RC(to_coset(pk.get(), i, pk->key[k].br, pk->key_cos[i][k]));
      }
  }
  RC(b200_table_upload(dev, curve, 1, d->srs_canonical, n + 3, B200_TABLE_PRECOMP, &pk->srs));
  RC(b200_sync(dev));
  *out = pk.release();
  return 0;
  GUARD_END
}

// ---- staged prover: one entry point per Fiat-Shamir round (prove.go:492-555 derives gamma, beta from [L],[R],[O];
//      alpha from [Z]; zeta from [H]; the folding challenge v from the linearised digest and the opened values) ---
int32_t b200_plonk_end(b200_plonk_session_t s) {
  GUARD_BEGIN
  if (!s) return 0;
  b200_sync(s->pk->dev);
  delete s;       // Scratch frees the device buffers
  return 0;
  GUARD_END
}

int32_t b200_plonk_begin(b200_plonk_pk_t pk, const void* l, const void* r, const void* o, const void* bl,
                         const void* br, const void* bo, const void* const* pi2, void* out_bsb22,
                         b200_plonk_session_t* out, void* out_lro) {
  GUARD_BEGIN
  if (!pk || !l || !r || !o || !bl || !br || !bo || !out || !out_lro) return set_error("plonk_begin: null argument");
  if (pk->n_qcp && (!pi2 || !out_bsb22))
    return set_error("plonk_begin: the key has BSB22 commitment gates - one committed polynomial per gate is required");
  const int dev = pk->dev;
  const size_t n = pk->n, fb = pk->fb;
  std::unique_ptr<b200_plonk_session_s> s(new b200_plonk_session_s(pk));
  s->jb = get_msm_ops(pk->curve, 1)->jac_bytes;
  memcpy(s->blind[0], bl, 2 * fb); memcpy(s->blind[1], br, 2 * fb); memcpy(s->blind[2], bo, 2 * fb);
  // ---- commitToLRO :404-489
  RC(s->S.alloc(n * fb, &s->d_l)); RC(s->S.alloc(n * fb, &s->d_r)); RC(s->S.alloc(n * fb, &s->d_o));
  const int nbl[4] = {2, 2, 2, 3};
  for (int k = 0; k < 4; k++) { RC(s->S.alloc(n * fb, &s->cb[k])); RC(s->S.alloc((n + nbl[k]) * fb, &s->bl[k])); }
  void* lag[3] = {s->d_l, s->d_r, s->d_o};
  const void* host[3] = {l, r, o};
  void* d_lro;
  RC(s->S.alloc(3 * s->jb, &d_lro));
  for (int k = 0; k < 3; k++) {       // upload and transforms of wire k + 1 run under the MSM of wire k
    RC(b200_h2d(dev, lag[k], host[k], n * fb));
    RC(canonical_blinded(pk, lag[k], s->blind[k], 2, s->cb[k], s->bl[k]));
    RC(commit_async(pk, s->bl[k], n + 2, (uint8_t*)d_lro + (size_t)k * s->jb));
  }
  RC(commit_join(pk, d_lro, 3 * s->jb, out_lro));
  // BSB22: committed polynomials -> canonical, and their digests (Bsb22Commitments :300; canonical SRS here, the
  // same group element as the reference's Lagrange-SRS commitment)
  for (uint32_t j = 0; j < pk->n_qcp; j++) {
    if (!pi2[j]) return set_error("plonk_begin: null committed polynomial");
    void *b = nullptr, *c = nullptr;
    RC(s->S.alloc(n * fb, &b)); RC(s->S.alloc(n * fb, &c));
    s->pi2_br.push_back(b); s->pi2_canon.push_back(c);
    RC(to_canonical(pk, pi2[j], true, b, c));
    RC(commit(pk, c, n, (uint8_t*)out_bsb22 + j * s->jb));
  }
  s->stage = 1;
  *out = s.release();
  return 0;
  GUARD_END
}

// completeQk (prove.go:349-373): Qk of THIS proof = the trace's Qk with the public inputs written into its first rows and the
// BSB22 commitment values at their constraint rows; Lagrange / regular, n elements on the host.  Optional (keys whose Qk
// is already complete, circuits without public inputs); any time after plonk_begin and before plonk_quotient.
int32_t b200_plonk_set_qk(b200_plonk_session_t s, const void* qk_lagrange) {
  GUARD_BEGIN
  if (!s || !qk_lagrange) return set_error("plonk_set_qk: null argument");
  if (s->stage != 1 && s->stage != 2) return set_error("plonk_set_qk: call after plonk_begin and before plonk_quotient");
  b200_plonk_pk_s* pk = s->pk;
  const size_t n = pk->n, fb = pk->fb;
  if (!s->qk_br) { RC(s->S.alloc(n * fb, &s->qk_br)); RC(s->S.alloc(n * fb, &s->qk_canon)); }
  return to_canonical(pk, qk_lagrange, true, s->qk_br, s->qk_canon);
  GUARD_END
}

// buildRatioCopyConstraint :635-668 + commit Z
// optional, between begin and quotient: StatisticalZK (backend.WithStatisticalZeroKnowledge; newInstance samples the two
// quotientShardsRandomizers, prove.go:239-242)
int32_t b200_plonk_set_quotient_randomizers(b200_plonk_session_t s, const void* hr2) {
  GUARD_BEGIN
  if (!s || !hr2) return set_error("plonk_set_quotient_randomizers: null argument");
  if (s->stage < 1 || s->stage > 2) return set_error("plonk_set_quotient_randomizers: call after plonk_begin and before plonk_quotient");
  memcpy(s->hr[0], hr2, s->pk->fb);
  memcpy(s->hr[1], (const uint8_t*)hr2 + s->pk->fb, s->pk->fb);
  s->szk = true;
  return 0;
  GUARD_END
}

int32_t b200_plonk_commit_z(b200_plonk_session_t s, const void* beta, const void* gamma, const void* bz, void* out_z) {
  GUARD_BEGIN
  if (!s || !beta || !gamma || !bz || !out_z) return set_error("plonk_commit_z: null argument");
  if (s->stage != 1) return set_error("plonk_commit_z: call after plonk_begin");
  b200_plonk_pk_s* pk = s->pk;
  const size_t n = pk->n, fb = pk->fb;
  memcpy(s->beta, beta, fb); memcpy(s->gamma, gamma, fb); memcpy(s->blind[3], bz, 3 * fb);
  void* d_z;
  RC(s->S.alloc(n * fb, &d_z));
  RC(b200_plonk_build_z(pk->dom0[0], s->d_l, s->d_r, s->d_o, pk->d_perm, s->beta, s->gamma, d_z));
  RC(canonical_blinded(pk, d_z, s->blind[3], 3, s->cb[3], s->bl[3]));
  RC(commit(pk, s->bl[3], n + 3, out_z));
  s->stage = 2;
  return 0;
  GUARD_END
}

// computeQuotient :558-633: numerator on the 4 cosets, divide by Z_H, commit h1, h2, h3
int32_t b200_plonk_quotient(b200_plonk_session_t s, const void* alpha, void* out_h) {
  GUARD_BEGIN
  if (!s || !alpha || !out_h) return set_error("plonk_quotient: null argument");
  if (s->stage != 2) return set_error("plonk_quotient: call after plonk_commit_z");
  b200_plonk_pk_s* pk = s->pk;
  const HostFrCtx* fr = pk->fr;
  const int dev = pk->dev;
  const size_t n = pk->n, fb = pk->fb;
  memcpy(s->alpha, alpha, fb);
  RC(s->S.alloc(4 * n * fb, &s->h));
  RC(dzero(dev, s->h, 4 * n * fb));
  Scratch T(dev);     // the 12 polynomials on the current coset: released when this stage ends
  void* onc[12];
  for (int k = 0; k < 12; k++) RC(T.alloc(n * fb, &onc[k]));
  alignas(16) uint8_t gb[8 * HOSTFR_MAX_LIMBS], w4b[8 * HOSTFR_MAX_LIMBS];
  fr->store(gb, pk->g); fr->store(w4b, pk->w4);
  // argument order of b200_plonk_coset_args: l r o z, then the key polynomials s1 s2 s3 ql qr qm qo qk
  const int key_arg[8] = {S1, S2, S3, QL, QR, QM, QO, QK};
  const bool cached = !pk->key_cos.empty();
  for (uint32_t i = 0; i < 4; i++) {
    const void* on[12];
    for (int k = 0; k < 12; k++) {
      const int q = k < 4 ? -1 : key_arg[k - 4];
      if (cached && q >= 0 && !(q == QK && s->qk_br)) { on[k] = pk->key_cos[i][q]; continue; }
      const void* src = q < 0 ? s->cb[k] : q == QK && s->qk_br ? s->qk_br : pk->key[q].br;
      RC(to_coset(pk, i, src, onc[k]));
      on[k] = onc[k];
    }
    b200_plonk_coset_args a;
    memset(&a, 0, sizeof(a));
    a.l = on[0]; a.r = on[1]; a.o = on[2]; a.z = on[3]; a.s1 = on[4]; a.s2 = on[5]; a.s3 = on[6];
    a.ql = on[7]; a.qr = on[8]; a.qm = on[9]; a.qo = on[10]; a.qk = on[11];
    a.alpha = s->alpha; a.beta = s->beta; a.gamma = s->gamma;
    a.bl = s->blind[0]; a.br = s->blind[1]; a.bo = s->blind[2]; a.bz = s->blind[3];
    a.nbl = 2; a.nbr = 2; a.nbo = 2; a.nbz = 3;
    a.coset_index = i; a.rho = 4; a.out = s->h;
    RC(b200_plonk_constraints_coset(pk->dom0[i], gb, w4b, &a));
    for (uint32_t j = 0; j < pk->n_qcp; j++) {   // + Qcp_j * PI2_j on this coset (gateConstraint :881-884)
      const void* qc = cached ? pk->key_cos[i][QCP0 + j] : onc[0];
      if (!cached) RC(to_coset(pk, i, pk->key[QCP0 + j].br, onc[0]));
      RC(to_coset(pk, i, s->pi2_br[j], onc[1]));
      RC(b200_plonk_bsb22_coset(pk->dom0[i], qc, onc[1], i, 4, s->h));
    }
  }
  RC(b200_plonk_divide_by_zh(pk->dom1, pk->logn, s->h));      // -> h canonical regular (4n)
  void* d_hres;
  RC(T.alloc(3 * s->jb, &d_hres));
  if (!s->szk) {
    for (int k = 0; k < 3; k++)
      RC(commit_async(pk, (uint8_t*)s->h + (size_t)k * (n + 2) * fb, n + 2, (uint8_t*)d_hres + (size_t)k * s->jb));
  } else {
    // StatisticalZK (h1(), h2(), h3(), prove.go:689-722): h1 + b1 X^(n+2), h2 - b1 + b2 X^(n+2), h3 - b2.  The shards
    // are adjacent slices of s->h, so each randomised shard is committed from a copy; s->h keeps the plain quotient
    // and the linearised polynomial gets the matching correction (b200_plonk_linearise).
    const HostFr b1 = fr->load(s->hr[0]), b2 = fr->load(s->hr[1]);
    void* tmp;
    RC(T.alloc((n + 3) * fb, &tmp));
    for (int k = 0; k < 3; k++) {
      RC(dzero(dev, (uint8_t*)tmp + (n + 2) * fb, fb));
      RC(d2d(dev, tmp, (uint8_t*)s->h + (size_t)k * (n + 2) * fb, (n + 2) * fb));
      if (k > 0) RC(add_to_element(pk, tmp, 0, fr->neg(k == 1 ? b1 : b2)));
      if (k < 2) RC(b200_h2d(dev, (uint8_t*)tmp + (n + 2) * fb, s->hr[k], fb));
      // tmp is rewritten for the next shard in stream order, after this MSM's digit extraction has read it
      RC(commit_async(pk, tmp, k < 2 ? n + 3 : n + 2, (uint8_t*)d_hres + (size_t)k * s->jb));
    }
  }
  RC(commit_join(pk, d_hres, 3 * s->jb, out_h));
  RC(b200_sync(dev));   // T's buffers are in use until here
  s->stage = 3;
  return 0;
  GUARD_END
}

// openZ :670-687, evaluations at zeta, innerComputeLinearizedPoly :1366-1487 and its commitment :788
//   out_points: linearised digest, Z-shifted opening quotient (2 G1Jac)
//   out_values: p(zeta) of {linearised, l, r, o, s1, s2}, then Z(w zeta)   (7 fr.Elements)
int32_t b200_plonk_linearise(b200_plonk_session_t s, const void* zeta_, void* out_points, void* out_values) {
  GUARD_BEGIN
  if (!s || !zeta_ || !out_points || !out_values) return set_error("plonk_linearise: null argument");
  if (s->stage != 3) return set_error("plonk_linearise: call after plonk_quotient");
  b200_plonk_pk_s* pk = s->pk;
  const HostFrCtx* fr = pk->fr;
  const int dev = pk->dev, curve = pk->curve;
  const size_t n = pk->n, fb = pk->fb;
  uint8_t* vals = (uint8_t*)out_values;
  uint8_t* h = (uint8_t*)s->h;
  memcpy(s->zeta, zeta_, fb);
  const HostFr zeta = fr->load(s->zeta), alpha = fr->load(s->alpha), beta = fr->load(s->beta), gamma = fr->load(s->gamma);
  const HostFr wz = fr->mul(zeta, pk->w);
  HostFr zu, lz, rz, oz, s1z, s2z;
  RC(eval_at(pk, s->bl[3], n + 3, wz, &zu));
  RC(eval_at(pk, s->bl[0], n + 2, zeta, &lz));
  RC(eval_at(pk, s->bl[1], n + 2, zeta, &rz));
  RC(eval_at(pk, s->bl[2], n + 2, zeta, &oz));
  RC(eval_at(pk, pk->key[S1].canon, n, zeta, &s1z));
  RC(eval_at(pk, pk->key[S2].canon, n, zeta, &s2z));
  auto M = [&](const HostFr& a, const HostFr& b) { return fr->mul(a, b); };
  auto A = [&](const HostFr& a, const HostFr& b) { return fr->add(a, b); };
  const HostFr rl = M(rz, lz);
  // c1 = (lz + beta s1z + gamma)(rz + beta s2z + gamma) zu beta alpha
  const HostFr c1 = M(M(M(M(A(A(lz, M(beta, s1z)), gamma), A(A(rz, M(beta, s2z)), gamma)), zu), beta), alpha);
  const HostFr uz = M(zeta, pk->g), uuz = M(uz, pk->g);
  // c2 = -(lz + beta zeta + gamma)(rz + beta uz + gamma)(oz + beta uuz + gamma) alpha
  const HostFr c2 = fr->neg(M(M(M(A(A(lz, M(beta, zeta)), gamma), A(A(rz, M(beta, uz)), gamma)),
                                A(A(oz, M(beta, uuz)), gamma)), alpha));
  const HostFr zn = fr->pow2k(zeta, (int)pk->logn);
  const HostFr zn2 = M(M(zn, zeta), zeta);
  const HostFr zh = fr->sub(zn, fr->one_());
  const HostFr zm1 = fr->sub(zeta, fr->one_());
  if (fr->is_zero(zm1)) return set_error("plonk_linearise: zeta = 1");
  // alpha^2 L1(zeta) = alpha^2 (zeta^n - 1) / (n (zeta - 1))
  const HostFr a2l1 = M(M(M(zh, fr->inv(zm1)), M(alpha, alpha)), fr->inv(fr->from_u64((uint64_t)n)));
  RC(s->S.alloc((n + 3) * fb, &s->lin));
  void* lin = s->lin;
  RC(dzero(dev, lin, (n + 3) * fb));
  RC(axpy(pk, lin, A(c2, a2l1), s->bl[3], n + 3));
  RC(axpy(pk, lin, c1, pk->key[S3].canon, n));
  RC(axpy(pk, lin, rl, pk->key[QM].canon, n));
  RC(axpy(pk, lin, lz, pk->key[QL].canon, n));
  RC(axpy(pk, lin, rz, pk->key[QR].canon, n));
  RC(axpy(pk, lin, oz, pk->key[QO].canon, n));
  RC(axpy(pk, lin, fr->one_(), s->qk_canon ? s->qk_canon : pk->key[QK].canon, n));
  // + sum_j Qcp_j(zeta) PI2_j(X)   (:1457-1460); Qcp_j(zeta) are claimed values 6.. of the batch opening
  const std::vector<Opened> op = opened(s);
  for (uint32_t j = 0; j < pk->n_qcp; j++) {
    HostFr qz;
    RC(eval_at(pk, op[6 + j].p, op[6 + j].count, zeta, &qz));
    fr->store(vals + (7 + j) * fb, qz);
    RC(axpy(pk, lin, qz, s->pi2_canon[j], n));
  }
  HostFr hc = zh;     // zh, zh zn2, zh zn2^2
  for (int k = 0; k < 3; k++) {
    RC(axpy(pk, lin, fr->neg(hc), h + (size_t)k * (n + 2) * fb, n + 2));
    hc = M(hc, zn2);
  }
  if (s->szk) {
    // the randomised shards differ from the plain ones by (b1 + b2 zeta^(n+2)) (X^(n+2) - zeta^(n+2)) in
    // h1 + zeta^(n+2) h2 + zeta^(2(n+2)) h3   (prove.go:1466-1481: coefficient n + 2 exists in h1, h2 only)
    const HostFr d = M(zh, A(fr->load(s->hr[0]), M(fr->load(s->hr[1]), zn2)));
    RC(add_to_element(pk, lin, n + 2, fr->neg(d)));
    RC(add_to_element(pk, lin, 0, M(d, zn2)));
  }
  // the two commitments of this round go through the pipelined MSM: the evaluations and the division below run under the
  // accumulate of the linearised digest, one join + download at the end
  Scratch T(dev);
  void* d_two;
  RC(T.alloc(2 * s->jb, &d_two));
  RC(commit_async(pk, lin, n + 3, d_two));
  // claimed values of the batch opening (BatchedProof.ClaimedValues) - needed by the caller to derive v
  for (int k = 0; k < 6; k++) {
    HostFr e;
    RC(eval_at(pk, op[k].p, op[k].count, zeta, &e));
    fr->store(vals + (size_t)k * fb, e);
  }
  // Z-shifted opening: (Z(X) - Z(w zeta)) / (X - w zeta)
  alignas(16) uint8_t zb[8 * HOSTFR_MAX_LIMBS], rem[8 * HOSTFR_MAX_LIMBS];
  void* zq;
  RC(T.alloc((n + 3) * fb, &zq));
  RC(d2d(dev, zq, s->bl[3], (n + 3) * fb));
  fr->store(zb, wz);
  RC(b200_poly_div_by_linear(dev, curve, zq, n + 3, zb, rem));
  if (!fr->eq(fr->load(rem), zu)) return set_error("plonk_linearise: Z(w zeta) from the division differs from the evaluation");
  RC(commit_async(pk, zq, n + 2, (uint8_t*)d_two + s->jb));
  RC(commit_join(pk, d_two, 2 * s->jb, out_points));
  fr->store(vals + 6 * fb, zu);
  RC(b200_sync(dev));
  s->stage = 4;
  return 0;
  GUARD_END
}

// batchOpening :796-837: fold the opened polynomials with powers of v, divide by X - zeta, commit
int32_t b200_plonk_batch_open(b200_plonk_session_t s, const void* v_, void* out_point) {
  GUARD_BEGIN
  if (!s || !v_ || !out_point) return set_error("plonk_batch_open: null argument");
  if (s->stage != 4) return set_error("plonk_batch_open: call after plonk_linearise");
  b200_plonk_pk_s* pk = s->pk;
  const HostFrCtx* fr = pk->fr;
  const int dev = pk->dev, curve = pk->curve;
  const size_t n = pk->n, fb = pk->fb;
  const HostFr v = fr->load(v_);
  Scratch T(dev);
  void* fold;
  RC(T.alloc((n + 3) * fb, &fold));
  RC(dzero(dev, fold, (n + 3) * fb));
  HostFr vp = fr->one_();
  for (const Opened& p : opened(s)) {
    RC(axpy(pk, fold, vp, p.p, p.count));
    vp = fr->mul(vp, v);
  }
  alignas(16) uint8_t rem[8 * HOSTFR_MAX_LIMBS];
  RC(b200_poly_div_by_linear(dev, curve, fold, n + 3, s->zeta, rem));
  RC(commit(pk, fold, n + 2, out_point));
  RC(b200_sync(dev));
  s->stage = 5;
  return 0;
  GUARD_END
}

// the five stages behind one call, for callers that already hold every challenge
int32_t b200_plonk_prove(b200_plonk_pk_t pk, const void* l, const void* r, const void* o,
                         const b200_plonk_challenges* ch, void* out_points, void* out_values) {
  GUARD_BEGIN
  if (!pk || !l || !r || !o || !ch || !out_points || !out_values) return set_error("plonk_prove: null argument");
  if (!ch->gamma || !ch->beta || !ch->alpha || !ch->zeta || !ch->v || !ch->bl || !ch->br || !ch->bo || !ch->bz)
    return set_error("plonk_prove: null challenge / blinding pointer");
  const size_t jb = get_msm_ops(pk->curve, 1)->jac_bytes;
  uint8_t* pts = (uint8_t*)out_points;          // L, R, O, Z, H1, H2, H3, linearised, batch opening, Z opening
  b200_plonk_session_t s = nullptr;
  if (pk->n_qcp && (!ch->pi2 || !ch->out_bsb22))
    return set_error("plonk_prove: the key has BSB22 commitment gates - challenges.pi2 / out_bsb22 are required");
  using clk = std::chrono::steady_clock;
  auto ms_since = [](clk::time_point t0) { return std::chrono::duration<double, std::milli>(clk::now() - t0).count(); };
  double st_ms[5] = {0, 0, 0, 0, 0};
  clk::time_point t0 = clk::now();
  int32_t rc = b200_plonk_begin(pk, l, r, o, ch->bl, ch->br, ch->bo, ch->pi2, ch->out_bsb22, &s, pts);
  if (!rc && ch->qk) rc = b200_plonk_set_qk(s, ch->qk);
  if (!rc && ch->hr) rc = b200_plonk_set_quotient_randomizers(s, ch->hr);
  if (!rc) rc = b200_sync(pk->dev);
  st_ms[0] = ms_since(t0); t0 = clk::now();
  if (!rc) rc = b200_plonk_commit_z(s, ch->beta, ch->gamma, ch->bz, pts + 3 * jb);
  st_ms[1] = ms_since(t0); t0 = clk::now();
  if (!rc) rc = b200_plonk_quotient(s, ch->alpha, pts + 4 * jb);
  st_ms[2] = ms_since(t0); t0 = clk::now();
  uint8_t two[2 * 288];     // linearised digest, Z opening; 288 B = G1Jac of the largest curve (BW6-761: 3 x 96 B)
  if (jb > 288) { b200_plonk_end(s); return set_error("plonk_prove: unexpected point size"); }
  if (!rc) rc = b200_plonk_linearise(s, ch->zeta, two, out_values);
  st_ms[3] = ms_since(t0); t0 = clk::now();
  if (!rc) {
    memcpy(pts + 7 * jb, two, jb);
    memcpy(pts + 9 * jb, two + jb, jb);
    rc = b200_plonk_batch_open(s, ch->v, pts + 8 * jb);
  }
  st_ms[4] = ms_since(t0);
  std::string err = rc ? b200_last_error() : "";
  b200_plonk_end(s);
  if (rc) return set_error(err), rc;
  for (int k = 0; k < 5; k++) pk->last_stage_ms[k] = st_ms[k];
  return 0;
  GUARD_END
}

int32_t b200_plonk_last_stage_ms(b200_plonk_pk_t pk, double* out5) {
  GUARD_BEGIN
  if (!pk || !out5) return set_error("plonk_last_stage_ms: null argument");
  for (int k = 0; k < 5; k++) out5[k] = pk->last_stage_ms[k];
  return 0;
  GUARD_END
}

}  // extern "C"
