// Groth16 prover host layer: the GPU twin of
// backend/accelerated/icicle/groth16/bn254/icicle.go (setupDevicePointers :88-264,
// Prove :784-1360, computeH :1391-1488) and of the CPU prover
// backend/groth16/bn254/prove.go:52-315, from "solved witness" to "proof points".
// The R1CS solver (constraint/bn254/solver.go) stays in Go and is out of scope.
#include <atomic>
#include <thread>

#include "capi_common.h"

#include <chrono>
#include <future>
#include <cstdio>

using namespace gb200;

struct b200_pk_s {
  int dev = 0, curve = 0;
  int logn = 0;
  size_t n = 0;  // domain cardinality
  b200_domain_t dom = nullptr;
  b200_table_t A = nullptr, B1 = nullptr, Z = nullptr, K = nullptr, B2 = nullptr;
  std::vector<uint8_t> alpha, beta, delta, beta2, delta2;
  uint32_t* d_idx_a = nullptr;
  uint32_t* d_idx_b = nullptr;
  uint32_t* d_idx_k = nullptr;   // only for keys with BSB22 commitments: private wires minus the committed ones
  size_t n_a = 0, n_b = 0, nb_wires = 0, nb_public = 0;   // n_a/n_b: THIS shard's counts
  size_t off_z = 0, cnt_z = 0, off_k = 0, cnt_k = 0;       // this shard's slice of Z and K
  int shard_rank = 0, shard_world = 1;
  const HostGroupOps* h1 = nullptr;
  const HostGroupOps* h2 = nullptr;
  const NttOps* fr = nullptr;
  // no per-key lock: tables are read-only, every proof allocates its own stream-ordered buffers, and concurrent
  // callers on one device are ordered by the device context's lock + stream order (capi_common.h DeviceCtx::mu)
};

static std::vector<uint8_t> copy_bytes(const void* p, size_t n) {
  const uint8_t* b = reinterpret_cast<const uint8_t*>(p);
  return std::vector<uint8_t>(b, b + n);
}

extern "C" {

int32_t b200_point_add_jac(int32_t curve, int32_t group, void* acc, const void* q) {
  GUARD_BEGIN
  const HostGroupOps* h = get_host_group_ops(curve, group);
  if (!h) return set_error("point_add_jac: unsupported curve/group");
  h->add_jac(acc, q);
  return 0;
  GUARD_END
}
int32_t b200_point_to_affine(int32_t curve, int32_t group, const void* p, void* out) {
  GUARD_BEGIN
  const HostGroupOps* h = get_host_group_ops(curve, group);
  if (!h) return set_error("point_to_affine: unsupported curve/group");
  h->to_affine(p, out);
  return 0;
  GUARD_END
}

int32_t b200_groth16_pk_free(b200_pk_t pk);

int32_t b200_groth16_pk_load(int32_t dev, const b200_groth16_pk_desc* d, b200_pk_t* out) {
  GUARD_BEGIN
  if (!d || !out) return set_error("pk_load: null argument");
  GB_DEVICE(ctx, dev);
  const HostGroupOps* h1 = get_host_group_ops(d->curve, 1);
  const HostGroupOps* h2 = get_host_group_ops(d->curve, 2);
  const NttOps* fr = get_ntt_ops(d->curve);
  if (!h1 || !h2 || !fr) return set_error("pk_load: unsupported curve");
  if (d->domain_size == 0 || (d->domain_size & (d->domain_size - 1))) return set_error("pk_load: domain size must be a power of two");
  if (d->n_z + 1 != d->domain_size) return set_error("pk_load: len(G1.Z) must be domain size - 1");
  if (d->n_b2 != d->n_b) return set_error("pk_load: len(G2.B) != len(G1.B)");
  if (d->n_k_removed && !d->k_removed) return set_error("pk_load: null k_removed");
  if (d->nb_public > d->nb_wires || d->n_k + d->n_k_removed != d->nb_wires - d->nb_public)
    return set_error("pk_load: len(G1.K) must equal nb_wires - nb_public - (number of committed private wires)");
  std::unique_ptr<b200_pk_s> pk(new b200_pk_s());
  pk->dev = dev; pk->curve = d->curve; pk->n = d->domain_size;
  while ((1ull << pk->logn) < pk->n) pk->logn++;
  pk->h1 = h1; pk->h2 = h2; pk->fr = fr;
  pk->nb_wires = d->nb_wires; pk->nb_public = d->nb_public;
  pk->alpha = copy_bytes(d->g1_alpha, h1->affine_bytes);
  pk->beta = copy_bytes(d->g1_beta, h1->affine_bytes);
  pk->delta = copy_bytes(d->g1_delta, h1->affine_bytes);
  pk->beta2 = copy_bytes(d->g2_beta, h2->affine_bytes);
  pk->delta2 = copy_bytes(d->g2_delta, h2->affine_bytes);
  // wire filters (prove.go:147-168): indices of wires whose A / B base is not infinity
  std::vector<uint32_t> ia, ib;
  for (size_t i = 0; i < d->nb_wires; i++) {
    if (!d->infinity_a[i]) ia.push_back((uint32_t)i);
    if (!d->infinity_b[i]) ib.push_back((uint32_t)i);
  }
  if (ia.size() != d->n_a || ib.size() != d->n_b) return set_error("pk_load: infinity flags inconsistent with len(G1.A)/len(G1.B)");
  // point-range sharding (SURVEY.md §8e): contiguous, balanced slices of every table
  const int world = d->shard_world > 1 ? d->shard_world : 1;
  const int rank = world > 1 ? d->shard_rank : 0;
  if (rank < 0 || rank >= world) return set_error("pk_load: shard_rank out of range");
  pk->shard_rank = rank; pk->shard_world = world;
  auto shard = [&](size_t n, size_t* off, size_t* cnt) {
    const size_t base = n / world, rem = n % world;
    *cnt = base + ((size_t)rank < rem ? 1 : 0);
    *off = (size_t)rank * base + ((size_t)rank < rem ? (size_t)rank : rem);
  };
  size_t off_a, cnt_a, off_b, cnt_b;
  shard(d->n_a, &off_a, &cnt_a);
  shard(d->n_b, &off_b, &cnt_b);
  shard(d->n_z, &pk->off_z, &pk->cnt_z);
  shard(d->n_k, &pk->off_k, &pk->cnt_k);
  // Krs scalars: private wires minus the committed ones (filterHeap, prove.go:321-344); only built when needed,
  // otherwise the K MSM reads the contiguous tail of the wire vector
  std::vector<uint32_t> ik;
  if (d->n_k_removed) {
    size_t r_ = 0;
    for (size_t i = d->nb_public; i < d->nb_wires; i++) {
      while (r_ < d->n_k_removed && d->k_removed[r_] < i) r_++;
      if (r_ < d->n_k_removed && d->k_removed[r_] == i) continue;
      ik.push_back((uint32_t)i);
    }
    if (ik.size() != d->n_k) return set_error("pk_load: k_removed must be sorted, distinct private wire indices");
    ik = std::vector<uint32_t>(ik.begin() + pk->off_k, ik.begin() + pk->off_k + pk->cnt_k);
  }
  ia = std::vector<uint32_t>(ia.begin() + off_a, ia.begin() + off_a + cnt_a);
  ib = std::vector<uint32_t>(ib.begin() + off_b, ib.begin() + off_b + cnt_b);
  pk->n_a = cnt_a; pk->n_b = cnt_b;
  const size_t ab1 = h1->affine_bytes, ab2 = h2->affine_bytes;
  auto at = [](const void* p, size_t bytes) { return (const void*)((const char*)p + bytes); };
  b200_pk_t raw = pk.get();
#define PK_TRY(x) do { int32_t rc_ = (x); if (rc_) { std::string m = b200_last_error(); b200_groth16_pk_free(pk.release()); set_error(m); return rc_; } } while (0)
  PK_TRY(b200_ntt_domain_new(dev, d->curve, (uint32_t)pk->logn, d->domain_gen, d->coset_gen, &raw->dom));
  if (d->dump_path) {
    // tables (this shard's ranges) straight from the ProvingKey dump file, marshal.go:375-539
    PK_TRY(b200_table_upload_file(dev, d->curve, 1, d->dump_path, d->dump_off_a + off_a * ab1, cnt_a, d->flags, &raw->A));
    PK_TRY(b200_table_upload_file(dev, d->curve, 1, d->dump_path, d->dump_off_b + off_b * ab1, cnt_b, d->flags, &raw->B1));
    PK_TRY(b200_table_upload_file(dev, d->curve, 1, d->dump_path, d->dump_off_z + pk->off_z * ab1, pk->cnt_z, d->flags, &raw->Z));
    PK_TRY(b200_table_upload_file(dev, d->curve, 1, d->dump_path, d->dump_off_k + pk->off_k * ab1, pk->cnt_k, d->flags, &raw->K));
    PK_TRY(b200_table_upload_file(dev, d->curve, 2, d->dump_path, d->dump_off_b2 + off_b * ab2, cnt_b, d->flags, &raw->B2));
  } else {
    if (!d->g1_a || !d->g1_b || !d->g1_z || !d->g1_k || !d->g2_b) {
      if (cnt_a || cnt_b || pk->cnt_z || pk->cnt_k) PK_TRY(set_error("pk_load: null table pointer (and no dump_path)"));
    }
    PK_TRY(b200_table_upload(dev, d->curve, 1, at(d->g1_a, off_a * ab1), cnt_a, d->flags, &raw->A));
    PK_TRY(b200_table_upload(dev, d->curve, 1, at(d->g1_b, off_b * ab1), cnt_b, d->flags, &raw->B1));
    PK_TRY(b200_table_upload(dev, d->curve, 1, at(d->g1_z, pk->off_z * ab1), pk->cnt_z, d->flags, &raw->Z));
    PK_TRY(b200_table_upload(dev, d->curve, 1, at(d->g1_k, pk->off_k * ab1), pk->cnt_k, d->flags, &raw->K));
    PK_TRY(b200_table_upload(dev, d->curve, 2, at(d->g2_b, off_b * ab2), cnt_b, d->flags, &raw->B2));
  }
  auto up = [&](const std::vector<uint32_t>& v, uint32_t** dptr) -> int32_t {
    CK(cudaMalloc(dptr, (v.size() ? v.size() : 1) * sizeof(uint32_t)));
    if (!v.empty()) CK(cudaMemcpy(*dptr, v.data(), v.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    return 0;
  };
  PK_TRY(up(ia, &raw->d_idx_a));
  PK_TRY(up(ib, &raw->d_idx_b));
  if (d->n_k_removed) PK_TRY(up(ik, &raw->d_idx_k));
#undef PK_TRY
  *out = pk.release();
  return 0;
  GUARD_END
}

int32_t b200_groth16_pk_free(b200_pk_t pk) {
  GUARD_BEGIN
  if (!pk) return 0;
  GB_DEVICE(ctx, pk->dev);
  cudaStreamSynchronize(ctx->stream);
  b200_table_free(pk->A); b200_table_free(pk->B1); b200_table_free(pk->Z); b200_table_free(pk->K); b200_table_free(pk->B2);
  b200_ntt_domain_free(pk->dom);
  cudaFree(pk->d_idx_a); cudaFree(pk->d_idx_b); cudaFree(pk->d_idx_k);
  delete pk;
  return 0;
  GUARD_END
}

// Upload from PAGEABLE host memory (Go heap slices are pageable): cudaMemcpyAsync would stage it through the driver's
// single bounce buffer at host-memcpy speed of one thread.  With GB200_STAGE_THREADS=T (opt-in, 0 = off) the source is
// copied by T threads into two pinned 16 MiB slots and each slot is DMA'd while the other is being filled.
// Pinned / registered sources (b200_host_alloc) take the plain asynchronous copy.
static cudaError_t upload_async(cudaStream_t st, void* dst, const void* src, size_t bytes) {
  static const int T = [] { const char* e = getenv("GB200_STAGE_THREADS"); int v = e ? atoi(e) : 0; return v < 0 ? 0 : (v > 16 ? 16 : v); }();
  if (T == 0 || bytes < ((size_t)4 << 20)) return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st);
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, src) != cudaSuccess) { cudaGetLastError(); return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st); }
  if (attr.type != cudaMemoryTypeUnregistered) return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st);
  constexpr size_t SLOT = (size_t)16 << 20;
  struct Ring {
    void* slot[2] = {nullptr, nullptr};
    cudaEvent_t done[2] = {nullptr, nullptr};
    bool used[2] = {false, false};
    std::mutex mu;
  };
  static Ring rings[GB200_MAX_DEVICES];               // per device (pinned slots and events belong to its context)
  int dev_ = 0;
  if (cudaGetDevice(&dev_) != cudaSuccess || dev_ < 0 || dev_ >= GB200_MAX_DEVICES)
    return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st);
  Ring& ring = rings[dev_];
  std::lock_guard<std::mutex> lk(ring.mu);              // one upload at a time through the ring
  for (int k = 0; k < 2; k++)
    if (!ring.slot[k]) {
      cudaError_t e = cudaHostAlloc(&ring.slot[k], SLOT, cudaHostAllocDefault);
      if (e != cudaSuccess) return e;
      e = cudaEventCreateWithFlags(&ring.done[k], cudaEventDisableTiming);
      if (e != cudaSuccess) return e;
    }
  const char* s = static_cast<const char*>(src);
  char* d = static_cast<char*>(dst);
  int k = 0;
  for (size_t off = 0; off < bytes; off += SLOT, k ^= 1) {
    const size_t len = bytes - off < SLOT ? bytes - off : SLOT;
    if (ring.used[k]) { cudaError_t e = cudaEventSynchronize(ring.done[k]); if (e != cudaSuccess) return e; }
    std::vector<std::thread> th;
    const size_t part = (len + T - 1) / T;
    for (int t = 0; t < T; t++) {
      const size_t lo = (size_t)t * part;
      if (lo >= len) break;
      const size_t cnt = len - lo < part ? len - lo : part;
      char* slot = static_cast<char*>(ring.slot[k]);
      th.emplace_back([=] { memcpy(slot + lo, s + off + lo, cnt); });
    }
    for (auto& x : th) x.join();
    cudaError_t e = cudaMemcpyAsync(d + off, ring.slot[k], len, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return e;
    e = cudaEventRecord(ring.done[k], st);
    if (e != cudaSuccess) return e;
    ring.used[k] = true;
  }
  return cudaSuccess;
}

// Stream-ordered device buffers of one proof (or one batch of proofs).  Freed on every exit path, early error returns
// included: the pipelined MSM tails (tail stream) still read and write these buffers, so `st` must wait for them before
// the stream-ordered frees (and tail_pending must not leak to the next caller).
struct ProveBufs {
  DeviceCtx* ctx; cudaStream_t st; std::vector<void*> p;
  ~ProveBufs() { msm_join(ctx); for (void* q : p) cudaFreeAsync(q, st); }
  cudaError_t get(void** out, size_t bytes) { cudaError_t e = cudaMallocAsync(out, bytes ? bytes : 1, st); if (e == cudaSuccess) p.push_back(*out); return e; }
};

static double now_ms() {
  using namespace std::chrono;
  return duration<double, std::milli>(steady_clock::now().time_since_epoch()).count();
}

int32_t b200_groth16_msms(b200_pk_t pk, const void* wires, const void* a, const void* b, const void* c,
                          size_t n_constraints, void* msm_out) {
  GUARD_BEGIN
  if (!pk) return set_error("prove: null proving key");
  if (!wires || !a || !b || !c || !msm_out) return set_error("prove: null argument");
  if (n_constraints > pk->n) return set_error("prove: more constraints than the domain holds");
  GB_DEVICE(ctx, pk->dev);
  cudaStream_t st = ctx->stream;
  const size_t fb = pk->fr->fr_bytes;
  const size_t n = pk->n;
  const size_t j1 = pk->h1->jac_bytes, j2 = pk->h2->jac_bytes;
  // step profile, the twin of the reference's ICICLE_STEP_PROFILE (icicle.go:72-75): serialises the stages
  const bool profile = getenv("GB200_STEP_PROFILE") != nullptr;
  double t_prev = now_ms();
  auto lap = [&](const char* what) -> int32_t {
    if (!profile) return 0;
    int32_t r_ = msm_join(ctx); if (r_) return r_;
    CK(cudaStreamSynchronize(st));
    const double t = now_ms();
    fprintf(stderr, "[gb200 step] %-14s %8.3f ms\n", what, t - t_prev);
    t_prev = t;
    return 0;
  };

  ProveBufs bufs{ctx, st, {}};
  void *d_w, *d_a, *d_b, *d_c, *d_wa, *d_wb, *d_res;
  CK(bufs.get(&d_w, pk->nb_wires * fb));
  CK(bufs.get(&d_a, n * fb)); CK(bufs.get(&d_b, n * fb)); CK(bufs.get(&d_c, n * fb));
  CK(bufs.get(&d_wa, pk->n_a * fb)); CK(bufs.get(&d_wb, pk->n_b * fb));
  CK(bufs.get(&d_res, 4 * j1 + j2));

  // upload the solution (R1CSSolution{W,A,B,C}); pad A,B,C to the domain (prove.go:356-359)
  CK(upload_async(st, d_w, wires, pk->nb_wires * fb));
  // wire filtering (prove.go:147-168) and the three MSMs that do not need h start right after W lands
  CK(pk->fr->gather(st, d_wa, d_w, pk->d_idx_a, pk->n_a));
  CK(pk->fr->gather(st, d_wb, d_w, pk->d_idx_b, pk->n_b));
  int32_t rc = lap("h2d W+filter"); if (rc) return rc;
  char* res = reinterpret_cast<char*>(d_res);
  // prove.go:207 (Ar), :194 (Bs1), :237 (Krs), :283 (Bs2), :227 (Krs2 over h)
  rc = msm_on_stream(ctx, pk->A, 0, pk->n_a, d_wa, res + 0 * j1, nullptr, true); if (rc) return rc;
  rc = lap("msm A"); if (rc) return rc;
  rc = msm_on_stream(ctx, pk->B1, 0, pk->n_b, d_wb, res + 1 * j1, nullptr, true); if (rc) return rc;
  rc = lap("msm B1"); if (rc) return rc;
  const void* k_scalars = (char*)d_w + (pk->nb_public + pk->off_k) * fb;
  if (pk->d_idx_k) {       // committed wires filtered out (BSB22)
    void* d_wk;
    CK(bufs.get(&d_wk, pk->cnt_k * fb));
    CK(pk->fr->gather(st, d_wk, d_w, pk->d_idx_k, pk->cnt_k));
    k_scalars = d_wk;
  }
  rc = msm_on_stream(ctx, pk->K, 0, pk->cnt_k, k_scalars, res + 3 * j1, nullptr, true); if (rc) return rc;
  rc = lap("msm K"); if (rc) return rc;
  rc = msm_on_stream(ctx, pk->B2, 0, pk->n_b, d_wb, res + 4 * j1, nullptr, true); if (rc) return rc;
  rc = lap("msm B2 (G2)"); if (rc) return rc;
  // A, B, C go up on the copy stream while the four h-independent MSMs run (the copy engine is
  // idle otherwise); with pageable host memory the copies block this host thread, not the GPU
  cudaStream_t cs = profile ? st : ctx->copy_stream;
  if (!profile) {
    CK(cudaEventRecord(ctx->copy_ev, st));          // d_a/d_b/d_c were allocated in st's order
    CK(cudaStreamWaitEvent(cs, ctx->copy_ev, 0));
  }
  const void* src[3] = {a, b, c};
  void* dst[3] = {d_a, d_b, d_c};
  for (int k = 0; k < 3; k++) {
    if (n_constraints) CK(upload_async(cs, dst[k], src[k], n_constraints * fb));
    if (n_constraints < n) CK(cudaMemsetAsync((char*)dst[k] + n_constraints * fb, 0, (n - n_constraints) * fb, cs));
  }
  if (!profile) {
    CK(cudaEventRecord(ctx->copy_ev, cs));
    CK(cudaStreamWaitEvent(st, ctx->copy_ev, 0));
  }
  rc = lap("h2d A,B,C"); if (rc) return rc;
  // h (bit-reversed, Montgomery) - prove.go:134,346-389
  CK(pk->fr->compute_h(st, pk->dom->impl, d_a, d_b, d_c));
  rc = lap("computeH"); if (rc) return rc;
  rc = msm_on_stream(ctx, pk->Z, 0, pk->cnt_z, (char*)d_a + pk->off_z * fb, res + 2 * j1, nullptr, true); if (rc) return rc;
  rc = msm_join(ctx); if (rc) return rc;
  // sharded key on a device with a communicator of the same world size: gather + fold on the device (comm.cu), so that
  // msm_out holds the COMPLETE sums on every rank; without a communicator msm_out holds this shard's partial sums
  if (pk->shard_world > 1 && ctx->comm && ctx->comm_world == pk->shard_world) {
    rc = points_allreduce_on_stream(ctx, pk->A->ops, res, 4, res); if (rc) return rc;
    rc = points_allreduce_on_stream(ctx, pk->B2->ops, res + 4 * j1, 1, res + 4 * j1); if (rc) return rc;
  }
  CK(cudaMemcpyAsync(msm_out, d_res, 4 * j1 + j2, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  rc = lap("msm Z + d2h"); if (rc) return rc;
  return 0;
  GUARD_END
}

}  // extern "C"

namespace {
// deltas = [r, s, -rs] * delta in G1 and s * delta in G2 (prove.go:185): four scalar multiplications on the host that
// need nothing from the device, so b200_groth16_prove computes them on a second host thread while the MSMs run
struct Groth16Deltas {
  std::vector<uint8_t> rd, sd, krd, sd2;
};
Groth16Deltas groth16_deltas(b200_pk_t pk, const void* r, const void* s) {
  const HostGroupOps* h1 = pk->h1;
  const HostGroupOps* h2 = pk->h2;
  const size_t j1 = h1->jac_bytes, j2 = h2->jac_bytes;
  Groth16Deltas d{std::vector<uint8_t>(j1), std::vector<uint8_t>(j1), std::vector<uint8_t>(j1), std::vector<uint8_t>(j2)};
  std::vector<uint8_t> kr(pk->fr->fr_bytes);
  h1->fr_neg_mul(r, s, kr.data());
  h1->scalar_mul_affine(pk->delta.data(), r, d.rd.data());
  h1->scalar_mul_affine(pk->delta.data(), s, d.sd.data());
  h1->scalar_mul_affine(pk->delta.data(), kr.data(), d.krd.data());
  h2->scalar_mul_affine(pk->delta2.data(), s, d.sd2.data());
  return d;
}

void groth16_assemble_with(b200_pk_t pk, const void* msm5, const void* r, const void* s, const Groth16Deltas& d,
                           void* ar_out, void* bs_out, void* krs_out) {
  const HostGroupOps* h1 = pk->h1;
  const HostGroupOps* h2 = pk->h2;
  const size_t j1 = h1->jac_bytes, j2 = h2->jac_bytes;
  const uint8_t* m = reinterpret_cast<const uint8_t*>(msm5);
  const uint8_t* mA = m;
  const uint8_t* mB1 = m + j1;
  const uint8_t* mZ = m + 2 * j1;
  const uint8_t* mK = m + 3 * j1;
  const uint8_t* mB2 = m + 4 * j1;
  // ar = A + alpha + r*delta (prove.go:207-214)
  std::vector<uint8_t> ar(mA, mA + j1);
  h1->add_mixed(ar.data(), pk->alpha.data());
  h1->add_jac(ar.data(), d.rd.data());
  // bs1 = B + beta + s*delta (prove.go:194-200)
  std::vector<uint8_t> bs1(mB1, mB1 + j1);
  h1->add_mixed(bs1.data(), pk->beta.data());
  h1->add_jac(bs1.data(), d.sd.data());
  // krs = K + Z.h + (-rs)*delta + s*ar + r*bs1 (prove.go:227-269)
  std::vector<uint8_t> krs(mK, mK + j1), tmp(j1);
  h1->add_jac(krs.data(), d.krd.data());
  h1->add_jac(krs.data(), mZ);
  h1->scalar_mul_jac(ar.data(), s, tmp.data());
  h1->add_jac(krs.data(), tmp.data());
  h1->scalar_mul_jac(bs1.data(), r, tmp.data());
  h1->add_jac(krs.data(), tmp.data());
  // bs2 = B2 + s*delta2 + beta2 (prove.go:283-292)
  std::vector<uint8_t> bs2(mB2, mB2 + j2);
  h2->add_jac(bs2.data(), d.sd2.data());
  h2->add_mixed(bs2.data(), pk->beta2.data());
  h1->to_affine(ar.data(), ar_out);
  h1->to_affine(krs.data(), krs_out);
  h2->to_affine(bs2.data(), bs_out);
}
}  // namespace

extern "C" {

int32_t b200_groth16_assemble(b200_pk_t pk, const void* msm5, const void* r, const void* s, void* ar_out,
                              void* bs_out, void* krs_out) {
  GUARD_BEGIN
  if (!pk || !msm5 || !r || !s || !ar_out || !bs_out || !krs_out) return set_error("assemble: null argument");
  groth16_assemble_with(pk, msm5, r, s, groth16_deltas(pk, r, s), ar_out, bs_out, krs_out);
  return 0;
  GUARD_END
}

int32_t b200_groth16_prove(b200_pk_t pk, const void* wires, const void* a, const void* b, const void* c,
                           size_t n_constraints, const void* r, const void* s, void* ar_out, void* bs_out,
                           void* krs_out, void* msm_out) {
  GUARD_BEGIN
  if (!pk) return set_error("prove: null proving key");
  if (pk->shard_world > 1) {
    // a sharded key proves in one call only when the library's communicator combines the partial sums (comm.cu)
    GB_DEVICE(ctx, pk->dev);
    if (!ctx->comm || ctx->comm_world != pk->shard_world)
      return set_error("prove: sharded key without a matching communicator - b200_comm_init first, or use "
                       "b200_groth16_msms + your own gather + b200_groth16_assemble");
  }
  if (!r || !s || !ar_out || !bs_out || !krs_out) return set_error("prove: null argument");
  std::vector<uint8_t> msm(4 * pk->h1->jac_bytes + pk->h2->jac_bytes);
  const double t0 = now_ms();
  // the delta multiples (prove.go:185) on a second host thread, under the device work
  std::future<Groth16Deltas> deltas = std::async(std::launch::async, [&] { return groth16_deltas(pk, r, s); });
  int32_t rc = b200_groth16_msms(pk, wires, a, b, c, n_constraints, msm.data());
  const double t1 = now_ms();
  const Groth16Deltas d = deltas.get();      // joined on every path: the lambda reads pk, r, s
  if (rc) return rc;
  if (msm_out) memcpy(msm_out, msm.data(), msm.size());
  groth16_assemble_with(pk, msm.data(), r, s, d, ar_out, bs_out, krs_out);
  if (getenv("GB200_STEP_PROFILE")) fprintf(stderr, "[gb200 step] %-14s %8.3f ms (device part %.3f ms)\n", "host assembly", now_ms() - t1, t1 - t0);
  return 0;
  GUARD_END
}

}  // extern "C"

namespace {
// fn(k) for k < count on up to hardware_concurrency host threads; the first exception of a worker is rethrown here
template <class Fn>
void parallel_for(size_t count, Fn fn) {
  size_t threads = std::thread::hardware_concurrency();
  if (threads == 0) threads = 1;
  if (threads > count) threads = count;
  std::atomic<size_t> next{0};
  std::vector<std::future<void>> workers;
  for (size_t t = 0; t < threads; t++)
    workers.push_back(std::async(std::launch::async, [&] { for (size_t k; (k = next++) < count;) fn(k); }));
  for (auto& w : workers) w.get();
}

// Device part of b200_groth16_prove_batch: the launch sequence of b200_groth16_msms with every stage over the whole
// batch - the wires of all items go up and are filtered in one launch per filter, each table's MSM is one batched MSM
// (pipelined like the single proof's five), A, B, C of all items go up on the copy stream into one [3][batch][n]
// buffer whose computeH runs as batched NTTs.  msm_out: the five tables' results table-major, [A | B1 | Z | K][batch]
// G1 Jacobians, then [batch] G2 Jacobians of B2.
int32_t groth16_msms_batch(DeviceCtx* ctx, b200_pk_t pk, size_t batch, const void* const* wires, const void* const* a,
                           const void* const* b, const void* const* c, size_t n_constraints, void* msm_out) {
  cudaStream_t st = ctx->stream;
  const size_t fb = pk->fr->fr_bytes, n = pk->n, nw = pk->nb_wires;
  const size_t j1 = pk->h1->jac_bytes, j2 = pk->h2->jac_bytes;
  ProveBufs bufs{ctx, st, {}};
  void *d_w, *d_abc, *d_wa, *d_wb, *d_res;
  CK(bufs.get(&d_w, batch * nw * fb));
  CK(bufs.get(&d_abc, 3 * batch * n * fb));
  CK(bufs.get(&d_wa, batch * pk->n_a * fb));
  CK(bufs.get(&d_wb, batch * pk->n_b * fb));
  CK(bufs.get(&d_res, batch * (4 * j1 + j2)));
  char* w = static_cast<char*>(d_w);
  for (size_t k = 0; k < batch; k++) CK(upload_async(st, w + k * nw * fb, wires[k], nw * fb));
  CK(pk->fr->gather_batch(st, d_wa, d_w, pk->d_idx_a, pk->n_a, batch, nw, pk->n_a));
  CK(pk->fr->gather_batch(st, d_wb, d_w, pk->d_idx_b, pk->n_b, batch, nw, pk->n_b));
  char* res = static_cast<char*>(d_res);
  auto out = [&](int table) { return res + (size_t)table * batch * j1; };
  int32_t rc = msm_on_stream(ctx, pk->A, 0, pk->n_a, d_wa, out(0), nullptr, true, nullptr, batch, pk->n_a);
  if (rc) return rc;
  rc = msm_on_stream(ctx, pk->B1, 0, pk->n_b, d_wb, out(1), nullptr, true, nullptr, batch, pk->n_b);
  if (rc) return rc;
  const void* k_scalars = w + pk->nb_public * fb;     // the private tail of each wire vector (keys are not sharded here)
  size_t k_stride = nw;
  if (pk->d_idx_k) {
    void* d_wk;
    CK(bufs.get(&d_wk, batch * pk->cnt_k * fb));
    CK(pk->fr->gather_batch(st, d_wk, d_w, pk->d_idx_k, pk->cnt_k, batch, nw, pk->cnt_k));
    k_scalars = d_wk;
    k_stride = pk->cnt_k;
  }
  rc = msm_on_stream(ctx, pk->K, 0, pk->cnt_k, k_scalars, out(3), nullptr, true, nullptr, batch, k_stride);
  if (rc) return rc;
  rc = msm_on_stream(ctx, pk->B2, 0, pk->n_b, d_wb, out(4), nullptr, true, nullptr, batch, pk->n_b);
  if (rc) return rc;
  // A, B, C of every item on the copy stream while the four h-independent MSMs run
  cudaStream_t cs = ctx->copy_stream;
  CK(cudaEventRecord(ctx->copy_ev, st));            // d_abc was allocated in st's order
  CK(cudaStreamWaitEvent(cs, ctx->copy_ev, 0));
  const void* const* src[3] = {a, b, c};
  char* abc = static_cast<char*>(d_abc);
  for (int m = 0; m < 3; m++)
    for (size_t k = 0; k < batch; k++) {
      char* dst = abc + (m * batch + k) * n * fb;
      if (n_constraints) CK(upload_async(cs, dst, src[m][k], n_constraints * fb));
      if (n_constraints < n) CK(cudaMemsetAsync(dst + n_constraints * fb, 0, (n - n_constraints) * fb, cs));
    }
  CK(cudaEventRecord(ctx->copy_ev, cs));
  CK(cudaStreamWaitEvent(st, ctx->copy_ev, 0));
  CK(pk->fr->compute_h_batch(st, pk->dom->impl, d_abc, batch));
  // Z over the first n - 1 elements of each item's h
  rc = msm_on_stream(ctx, pk->Z, 0, pk->cnt_z, d_abc, out(2), nullptr, true, nullptr, batch, n);
  if (rc) return rc;
  rc = msm_join(ctx);
  if (rc) return rc;
  CK(cudaMemcpyAsync(msm_out, d_res, batch * (4 * j1 + j2), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return 0;
}
}  // namespace

extern "C" {

int32_t b200_groth16_prove_batch(b200_pk_t pk, size_t batch, const void* const* wires, const void* const* a,
                                 const void* const* b, const void* const* c, size_t n_constraints, const void* r,
                                 const void* s, void* ar_out, void* bs_out, void* krs_out, void* msm_out) {
  GUARD_BEGIN
  if (!pk) return set_error("prove_batch: null proving key");
  if (pk->shard_world > 1)
    return set_error("prove_batch: sharded keys are not supported - prove each proof with b200_groth16_prove");
  if (n_constraints > pk->n) return set_error("prove_batch: more constraints than the domain holds");
  if (batch == 0) return 0;
  if (!wires || !a || !b || !c || !r || !s || !ar_out || !bs_out || !krs_out) return set_error("prove_batch: null argument");
  // every index the batch needs fits its device counters: the five batched MSMs (2^31 entries, 2^31 - 1 bucket keys,
  // each at the window of the table's single MSM) and the 32-bit element indices of the pointwise and gather kernels
  const size_t n = pk->n, nw = pk->nb_wires;
  size_t fits = (((size_t)1 << 32) - 1) / (n > nw ? n : (nw ? nw : 1));
  const std::pair<b200_table_s*, size_t> tables[5] = {{pk->A, pk->n_a}, {pk->B1, pk->n_b}, {pk->Z, pk->cnt_z},
                                                      {pk->K, pk->cnt_k}, {pk->B2, pk->n_b}};
  for (const auto& t : tables) {
    const size_t m = msm_max_batch(t.first, t.second, t.first->c);
    if (m < fits) fits = m;
  }
  if (batch > fits)
    return set_error("prove_batch: a batch of " + std::to_string(batch) + " proofs exceeds the device indices (2^31 MSM "
                     "entries and bucket keys per table, 2^32 elements per batched vector) - the largest batch this key "
                     "takes is " + std::to_string(fits));
  for (size_t k = 0; k < batch; k++)
    if (!wires[k] || !a[k] || !b[k] || !c[k]) return set_error("prove_batch: null witness vector of item " + std::to_string(k));
  GB_DEVICE(ctx, pk->dev);
  const HostGroupOps* h1 = pk->h1;
  const HostGroupOps* h2 = pk->h2;
  const size_t fb = pk->fr->fr_bytes, j1 = h1->jac_bytes, j2 = h2->jac_bytes;
  auto item = [](const void* p, size_t k, size_t bytes) { return static_cast<const char*>(p) + k * bytes; };
  // the delta multiples of every item (prove.go:185) on host threads, under the device work
  std::vector<Groth16Deltas> deltas(batch);
  std::future<void> dfut = std::async(std::launch::async, [&] {
    parallel_for(batch, [&](size_t k) { deltas[k] = groth16_deltas(pk, item(r, k, fb), item(s, k, fb)); });
  });
  std::vector<uint8_t> msm(batch * (4 * j1 + j2));
  const int32_t rc = groth16_msms_batch(ctx, pk, batch, wires, a, b, c, n_constraints, msm.data());
  dfut.get();                                   // joined on every path: the workers read pk, r, s
  if (rc) return rc;
  parallel_for(batch, [&](size_t k) {
    // item k's five results in b200_groth16_prove's layout
    std::vector<uint8_t> m5(4 * j1 + j2);
    for (int t = 0; t < 4; t++) memcpy(m5.data() + t * j1, msm.data() + ((size_t)t * batch + k) * j1, j1);
    memcpy(m5.data() + 4 * j1, msm.data() + 4 * batch * j1 + k * j2, j2);
    if (msm_out) memcpy(static_cast<char*>(msm_out) + k * m5.size(), m5.data(), m5.size());
    groth16_assemble_with(pk, m5.data(), item(r, k, fb), item(s, k, fb), deltas[k],
                          static_cast<char*>(ar_out) + k * h1->affine_bytes, static_cast<char*>(bs_out) + k * h2->affine_bytes,
                          static_cast<char*>(krs_out) + k * h1->affine_bytes);
  });
  return 0;
  GUARD_END
}

}  // extern "C"
