// Per-curve instantiation of the kernel templates behind the type-erased tables of
// internal.h.  Included by inst_<curve>.cu only.
#pragma once
#include <vector>

#include "host_field.h"
#include "internal.h"
#include "fixed_base.cuh"
#include "msm_impl.cuh"
#include "ntt_impl.cuh"
#include "plonk.cuh"
#include "points_ntt.cuh"
#include "points_scale.cuh"
#include "../../include/gnark_b200.h"

namespace gb200 {

template <class Fr>
struct NttInst;   // below: MsmInst::points_scale builds its scalars with NttInst<Fr>::scale_powers

// ---------------------------------------------------------------------------
// MSM
// ---------------------------------------------------------------------------
template <class Fr, class F>
struct MsmInst {
  static MsmPlan plan(uint32_t n, uint32_t batch, uint32_t stride, uint32_t off, int c, int precomp, uint32_t task_len,
                      uint32_t chunk, uint32_t scalar_stride = 0) {
    // batch 1: msm_make_plan's
    return msm_make_batch_plan(batch, n, stride, off, Fr::Params::BITS, c, precomp, task_len, chunk, scalar_stride);
  }
  static cudaError_t ws_bytes(uint32_t n, uint32_t batch, uint32_t stride, int c, int precomp, uint32_t task_len, uint32_t chunk,
                              size_t* out) {
    MsmLayout<F> L;
    MsmPlan pl = plan(n, batch, stride, 0, c, precomp, task_len, chunk);
    GB_CUDA_TRY(msm_layout<F>(pl, L));
    *out = L.total;
    return cudaSuccess;
  }
  static cudaError_t run(cudaStream_t st, uint32_t n, uint32_t batch, uint32_t stride, uint32_t off, int c, int precomp,
                         uint32_t task_len, uint32_t chunk, const void* d_table, const void* d_scalars,
                         void* d_out_jac, void* ws, cudaEvent_t* ev, const MsmPipe* pipe, const uint32_t* d_idx,
                         uint32_t scalar_stride) {
    MsmPlan pl = plan(n, batch, stride, off, c, precomp, task_len, chunk, scalar_stride);
    MsmLayout<F> L;
    GB_CUDA_TRY(msm_layout<F>(pl, L));
    return msm_enqueue<Fr, F>(st, pl, reinterpret_cast<const Affine<F>*>(d_table),
                              reinterpret_cast<const Fr*>(d_scalars), reinterpret_cast<Jacobian<F>*>(d_out_jac), ws, L, ev, pipe, d_idx);
  }
  // d_table holds the n bases in slab 0 already; slabs 1.. are filled in place
  static cudaError_t precompute(cudaStream_t st, uint32_t n, int nwin, int c, void* d_table) {
    if (n == 0 || nwin <= 1) return cudaSuccess;
    Affine<F>* t = reinterpret_cast<Affine<F>*>(d_table);
    return msm_precompute_enqueue<F>(st, n, nwin, c, t, t);
  }
  static int acc_blocks_per_sm() {
    static const int cached = [] {
      int per_sm = 0;
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_msm_accumulate<F>, 128, 0) != cudaSuccess || per_sm < 1) {
        cudaGetLastError();
        per_sm = 1;
      }
      return per_sm;
    }();
    return cached;
  }
  static cudaError_t fixed_base(cudaStream_t st, const void* h_base, const void* d_scalars, size_t n, int c,
                                void* d_out_affine) {
    Affine<F> base;
    memcpy(&base, h_base, sizeof(base));
    return fixed_base_enqueue<Fr, F>(st, base, reinterpret_cast<const Fr*>(d_scalars), n, c,
                                     reinterpret_cast<Affine<F>*>(d_out_affine));
  }
  static cudaError_t fold(cudaStream_t st, const void* d_gathered, uint32_t world, uint32_t count, void* d_out_jac) {
    if (count == 0 || world == 0) return cudaSuccess;
    k_points_fold<F><<<(count + 63) / 64, 64, 0, st>>>(reinterpret_cast<const Jacobian<F>*>(d_gathered), world, count,
                                                       reinterpret_cast<Jacobian<F>*>(d_out_jac));
    return cudaGetLastError();
  }
  using FB = typename F::Base;
  static size_t encoded_bytes(int encoding) {
    if (encoding == POINTS_RAW) return sizeof(Affine<F>);
    if (encoding == POINTS_COMPRESSED) return sizeof(F);      // X only (G2: X.A1 || X.A0)
    return 0;
  }
  static cudaError_t decode(cudaStream_t st, const void* d_bytes, size_t n, int encoding, int curve, int group,
                            void* d_out_affine, uint32_t* d_status) {
    if (n == 0) return cudaSuccess;
    if (encoded_bytes(encoding) == 0) return cudaErrorNotSupported;
    const DecodeConsts<FB> k = decode_make_consts<F, FB>(curve, group);
    const size_t stride = encoded_bytes(encoding);
    k_points_decode<F, FB><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(reinterpret_cast<const uint8_t*>(d_bytes), n, stride,
                                                                       encoding == POINTS_COMPRESSED ? 1 : 0, k,
                                                                       reinterpret_cast<Affine<F>*>(d_out_affine), d_status);
    return cudaGetLastError();
  }
  // points_scale.cuh: d_points[i] <- (c * t^i) * d_points[i], i < n <= PS_MAX_POINTS; t null means t = 1
  static cudaError_t points_scale(cudaStream_t st, void* d_points, size_t n, const void* c_mont, const void* t_mont) {
    if (n == 0) return cudaSuccess;
    AsyncBuf kb;
    GB_CUDA_TRY(kb.alloc(n * sizeof(Fr), st));
    Fr* k = reinterpret_cast<Fr*>(kb.p);
    k_points_scale_ones<Fr><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(k, n);
    GB_CUDA_TRY(cudaGetLastError());
    const Fr one = Fr::one();
    GB_CUDA_TRY(NttInst<Fr>::scale_powers(st, k, n, c_mont, t_mont ? t_mont : &one));
    k_points_scale<Fr, F><<<(unsigned)((n + PS_THREADS - 1) / PS_THREADS), PS_THREADS, 0, st>>>(
        reinterpret_cast<Affine<F>*>(d_points), k, (uint32_t)n);
    GB_CUDA_TRY(cudaGetLastError());
    return kb.release_on(st);
  }
  static const MsmOps* ops() {
    static const MsmOps o = {Fr::Params::BITS, sizeof(Fr), sizeof(Affine<F>), sizeof(Jacobian<F>), &ws_bytes, &run,
                             &precompute, &acc_blocks_per_sm, &fixed_base, &fold, &encoded_bytes, &decode, nullptr,
                             &points_scale};
    return &o;
  }
  // G1 only: the group NTT is instantiated through ops_g1(), so G2 compiles none of its kernels
  static cudaError_t points_ntt(cudaStream_t st, void* dom, void* d_points, int inverse) {
    const NttDomainDev<Fr>& d = *reinterpret_cast<const NttDomainDev<Fr>*>(dom);
    return points_ntt_enqueue<Fr, F>(st, d.logn, inverse ? d.itw : d.tw, d.ninv, inverse != 0,
                                     reinterpret_cast<Affine<F>*>(d_points));
  }
  static const MsmOps* ops_g1() {
    static const MsmOps o = [] { MsmOps x = *ops(); x.points_ntt = &points_ntt; return x; }();
    return &o;
  }
};

// ---------------------------------------------------------------------------
// vector kernels
// ---------------------------------------------------------------------------
template <class Fr>
__global__ void __launch_bounds__(256) k_vec_op(int op, Fr* __restrict__ out, const Fr* __restrict__ a,
                                                const Fr* __restrict__ b, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Fr x = a[i], y = b[i];
  out[i] = op == 0 ? x * y : (op == 1 ? x + y : x - y);
}
template <class Fr>
__global__ void __launch_bounds__(256) k_bit_reverse(Fr* __restrict__ d, uint32_t logn) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (1u << logn)) return;
  const uint32_t j = ntt_bitrev(i, (int)logn);
  if (j > i) { Fr t = d[i]; d[i] = d[j]; d[j] = t; }
}
template <class Fr>
__global__ void __launch_bounds__(256) k_scale_powers(const Fr* __restrict__ pw, Fr s, size_t n, Fr* __restrict__ d) {
  const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  Fr acc = s;
  size_t e = k;
  for (int j = 0; e; j++, e >>= 1)
    if (e & 1) acc = acc * pw[j];
  d[k] = d[k] * acc;
}
template <class Fr>
__global__ void __launch_bounds__(256) k_axpy(Fr* __restrict__ y, Fr a, const Fr* __restrict__ x, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = y[i] + a * x[i];
}
template <class Fr>
__global__ void __launch_bounds__(256) k_gather(Fr* __restrict__ out, const Fr* __restrict__ src,
                                                const uint32_t* __restrict__ idx, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = src[idx[i]];
}
// the same filter over a batch of source vectors: blockIdx.y is the item, out[b * out_stride + j] = src[b * src_stride +
// idx[j]]; 32-bit element indices (the caller keeps batch * src_stride and batch * out_stride below 2^32)
template <class Fr>
__global__ void __launch_bounds__(256) k_gather_batch(Fr* __restrict__ out, const Fr* __restrict__ src,
                                                      const uint32_t* __restrict__ idx, uint32_t n, uint32_t src_stride,
                                                      uint32_t out_stride) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) out[blockIdx.y * out_stride + j] = src[blockIdx.y * src_stride + idx[j]];
}

// ---------------------------------------------------------------------------
// NTT
// ---------------------------------------------------------------------------
template <class Fr>
struct NttInst {
  using Dom = NttDomainDev<Fr>;
  static void* domain_new(cudaStream_t st, int logn, const void* gen, const void* coset, cudaError_t* err) {
    Dom* d = new Dom();
    *err = d->init(st, logn, reinterpret_cast<const Fr*>(gen), reinterpret_cast<const Fr*>(coset));
    if (*err != cudaSuccess) { d->destroy(); delete d; return nullptr; }
    return d;
  }
  static void domain_free(void* p) { Dom* d = reinterpret_cast<Dom*>(p); d->destroy(); delete d; }
  static size_t domain_bytes(void* p) { return reinterpret_cast<Dom*>(p)->table_bytes(); }
  static cudaError_t ntt(cudaStream_t st, void* dom, void* data, int inverse, int decimation, int on_coset) {
    return ntt_enqueue<Fr>(st, *reinterpret_cast<Dom*>(dom), reinterpret_cast<Fr*>(data), inverse != 0, decimation,
                           on_coset != 0);
  }
  static cudaError_t ntt_batch(cudaStream_t st, void* dom, void* data, size_t batch, int inverse, int decimation,
                               int on_coset) {
    return ntt_enqueue<Fr>(st, *reinterpret_cast<Dom*>(dom), reinterpret_cast<Fr*>(data), inverse != 0, decimation,
                           on_coset != 0, batch);
  }
  static cudaError_t compute_h_batch(cudaStream_t st, void* dom, void* abc, size_t batch) {
    return compute_h_batch_enqueue<Fr>(st, *reinterpret_cast<Dom*>(dom), reinterpret_cast<Fr*>(abc), batch);
  }
  static cudaError_t compute_h(cudaStream_t st, void* dom, void* a, void* b, void* c) {
    return compute_h_enqueue<Fr>(st, *reinterpret_cast<Dom*>(dom), reinterpret_cast<Fr*>(a), reinterpret_cast<Fr*>(b),
                                 reinterpret_cast<Fr*>(c));
  }
  static cudaError_t vec_op(cudaStream_t st, int op, void* out, const void* a, const void* b, size_t n) {
    if (!n) return cudaSuccess;
    k_vec_op<Fr><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(op, (Fr*)out, (const Fr*)a, (const Fr*)b, n);
    return cudaGetLastError();
  }
  static cudaError_t bit_reverse(cudaStream_t st, void* d, uint32_t logn) {
    k_bit_reverse<Fr><<<((1u << logn) + 255) / 256, 256, 0, st>>>((Fr*)d, logn);
    return cudaGetLastError();
  }
  static cudaError_t scale_powers(cudaStream_t st, void* d, size_t n, const void* s, const void* g) {
    if (!n) return cudaSuccess;
    Fr pw[64];
    Fr b = *reinterpret_cast<const Fr*>(g);
    for (int j = 0; j < 64; j++) { pw[j] = b; b = b.sqr(); }
    AsyncBuf pwb;
    GB_CUDA_TRY(pwb.alloc(sizeof(pw), st));
    Fr* d_pw = (Fr*)pwb.p;
    GB_CUDA_TRY(cudaMemcpyAsync(d_pw, pw, sizeof(pw), cudaMemcpyHostToDevice, st));
    k_scale_powers<Fr><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_pw, *reinterpret_cast<const Fr*>(s), n, (Fr*)d);
    GB_CUDA_TRY(cudaGetLastError());
    GB_CUDA_TRY(pwb.release_on(st));
    return cudaStreamSynchronize(st);
  }
  static cudaError_t batch_invert(cudaStream_t st, void* d, size_t n) {
    if (!n) return cudaSuccess;
    const size_t threads = (n + BI_CHUNK - 1) / BI_CHUNK;
    k_batch_invert<Fr><<<(unsigned)((threads + 127) / 128), 128, 0, st>>>((Fr*)d, n);
    return cudaGetLastError();
  }
  static cudaError_t plonk_coset(cudaStream_t st, void* dom0, const void* big_coset_gen, const void* big_gen,
                                 const void* args_) {
    Dom& d = *reinterpret_cast<Dom*>(dom0);
    const b200_plonk_coset_args& c = *reinterpret_cast<const b200_plonk_coset_args*>(args_);
    PlonkCosetArgs<Fr> a;
    a.l = (const Fr*)c.l; a.r = (const Fr*)c.r; a.o = (const Fr*)c.o; a.z = (const Fr*)c.z;
    a.s1 = (const Fr*)c.s1; a.s2 = (const Fr*)c.s2; a.s3 = (const Fr*)c.s3;
    a.ql = (const Fr*)c.ql; a.qr = (const Fr*)c.qr; a.qm = (const Fr*)c.qm; a.qo = (const Fr*)c.qo; a.qk = (const Fr*)c.qk;
    a.tw = d.tw; a.out = (Fr*)c.out;
    a.alpha = *(const Fr*)c.alpha; a.beta = *(const Fr*)c.beta; a.gamma = *(const Fr*)c.gamma;
    const Fr g = *(const Fr*)big_coset_gen, w4 = *(const Fr*)big_gen;
    Fr coset = g;
    for (uint32_t k = 0; k < c.coset_index; k++) coset = coset * w4;   // shifters (:943-948)
    a.coset = coset; a.cs = g; a.css = g.sqr();
    Fr cn = coset;
    for (int k = 0; k < d.logn; k++) cn = cn.sqr();
    a.coset_n_minus_one = cn - Fr::one();
    a.lone_scale = a.coset_n_minus_one * d.ninv;
    const void* bsrc[4] = {c.bl, c.br, c.bo, c.bz};
    const int bn[4] = {c.nbl, c.nbr, c.nbo, c.nbz};
    Fr* bdst[4] = {a.bl, a.br, a.bo, a.bz};
    for (int q = 0; q < 4; q++) {
      if (bn[q] < 0 || bn[q] > PLONK_MAX_BLIND) return cudaErrorInvalidValue;
      plonk_set_blinding<Fr>(a, bdst[q], (const Fr*)bsrc[q], bn[q]);
    }
    a.nbl = c.nbl; a.nbr = c.nbr; a.nbo = c.nbo; a.nbz = c.nbz;
    a.n = d.n; a.logn = (uint32_t)d.logn; a.rho = c.rho; a.coset_index = c.coset_index;
    a.log_rho = 0;
    while ((1u << a.log_rho) < c.rho) a.log_rho++;
    if ((1u << a.log_rho) != c.rho || c.coset_index >= c.rho) return cudaErrorInvalidValue;
    // denominators of L1 on this coset: cached in the domain handle (one handle per coset in the prover), else per call
    static const bool den_cache = [] { const char* e = getenv("GB200_PLONK_DEN_CACHE"); return !e || atoi(e) != 0; }();
    AsyncBuf denb;
    Fr* den;
    if (den_cache) {
      if (!d.den_inv) GB_CUDA_TRY(cudaMalloc(&d.den_inv, (size_t)d.n * sizeof(Fr)));
      den = d.den_inv;
    } else {
      GB_CUDA_TRY(denb.alloc((size_t)d.n * sizeof(Fr), st));
      den = (Fr*)denb.p;
    }
    if (!den_cache || !d.den_valid || !(d.den_coset == coset)) {
      k_plonk_denominators<Fr><<<(d.n + 255) / 256, 256, 0, st>>>(den, d.n, d.tw, coset);
      GB_CUDA_TRY(batch_invert(st, den, d.n));
      if (den_cache) { d.den_coset = coset; d.den_valid = true; }
    }
    a.den_inv = den;
    k_plonk_constraints<Fr><<<(d.n + 127) / 128, 128, 0, st>>>(a);
    GB_CUDA_TRY(cudaGetLastError());
    return denb.release_on(st);
  }
  static cudaError_t plonk_bsb22(cudaStream_t st, void* dom0, const void* qcp, const void* pi2, uint32_t coset_index,
                                 uint32_t rho, void* out) {
    const Dom& d = *reinterpret_cast<Dom*>(dom0);
    uint32_t log_rho = 0;
    while ((1u << log_rho) < rho) log_rho++;
    if ((1u << log_rho) != rho || coset_index >= rho) return cudaErrorInvalidValue;
    k_plonk_add_bsb22<Fr><<<(d.n + 255) / 256, 256, 0, st>>>((const Fr*)qcp, (const Fr*)pi2, (Fr*)out, d.n, coset_index, rho,
                                                           (uint32_t)d.logn, log_rho);
    return cudaGetLastError();
  }
  static cudaError_t plonk_divide_by_zh(cudaStream_t st, void* dom1, uint32_t log_n0, void* data) {
    const Dom& d = *reinterpret_cast<Dom*>(dom1);
    if ((int)log_n0 > d.logn || d.logn - (int)log_n0 > 6) return cudaErrorInvalidValue;
    const uint32_t rho = 1u << (d.logn - (int)log_n0);
    // evaluateXnMinusOneDomainBigCoset (:1327-1350): 1 / (g^n * (w^n)^i - 1), i < rho
    Fr tab[64];
    Fr gn = d.coset, wn = d.gen;
    for (uint32_t k = 0; k < log_n0; k++) { gn = gn.sqr(); wn = wn.sqr(); }
    Fr cur = gn;
    for (uint32_t i = 0; i < rho; i++) { tab[i] = (cur - Fr::one()).inverse(); cur = cur * wn; }
    AsyncBuf tabb;
    GB_CUDA_TRY(tabb.alloc(sizeof(tab), st));
    Fr* d_tab = (Fr*)tabb.p;
    GB_CUDA_TRY(cudaMemcpyAsync(d_tab, tab, sizeof(Fr) * rho, cudaMemcpyHostToDevice, st));
    k_plonk_zh_scale<Fr><<<(d.n + 255) / 256, 256, 0, st>>>((Fr*)data, (uint32_t)d.logn, rho, d_tab);
    GB_CUDA_TRY(cudaGetLastError());
    GB_CUDA_TRY(ntt_enqueue<Fr>(st, d, (Fr*)data, true, NTT_DIT, true));
    GB_CUDA_TRY(tabb.release_on(st));
    return cudaStreamSynchronize(st);  // tab is a stack buffer
  }
  static cudaError_t axpy(cudaStream_t st, void* y, const void* a, const void* x, size_t n) {
    if (!n) return cudaSuccess;
    k_axpy<Fr><<<(unsigned)((n + 255) / 256), 256, 0, st>>>((Fr*)y, *(const Fr*)a, (const Fr*)x, n);
    return cudaGetLastError();
  }
  static cudaError_t scan(cudaStream_t st, int op, void* d, size_t n, int exclusive) {
    return op == 0 ? scan_enqueue<Fr, 0>(st, (Fr*)d, n, exclusive != 0) : scan_enqueue<Fr, 1>(st, (Fr*)d, n, exclusive != 0);
  }
  // iop.BuildRatioCopyConstraint: Z[0] = 1, Z[i+1] = Z[i] * num_i / den_i  (Lagrange, regular layout)
  static cudaError_t plonk_build_z(cudaStream_t st, void* dom0, const void* l, const void* r, const void* o,
                                   const int64_t* perm, const void* beta, const void* gamma, void* z) {
    const Dom& d = *reinterpret_cast<Dom*>(dom0);
    AsyncBuf numb, denb;
    GB_CUDA_TRY(numb.alloc((size_t)d.n * sizeof(Fr), st));
    GB_CUDA_TRY(denb.alloc((size_t)d.n * sizeof(Fr), st));
    Fr *num = (Fr*)numb.p, *den = (Fr*)denb.p;
    k_plonk_ratio_terms<Fr><<<(d.n + 255) / 256, 256, 0, st>>>(d.n, (const Fr*)l, (const Fr*)r, (const Fr*)o, perm, d.tw,
                                                            *(const Fr*)beta, *(const Fr*)gamma, d.coset, num, den);
    GB_CUDA_TRY(cudaGetLastError());
    GB_CUDA_TRY(batch_invert(st, den, d.n));
    k_plonk_shift_ratio<Fr><<<(d.n + 255) / 256, 256, 0, st>>>(d.n, num, den, (Fr*)z);
    GB_CUDA_TRY(cudaGetLastError());
    GB_CUDA_TRY((scan_enqueue<Fr, 0>(st, (Fr*)z, d.n, false)));
    GB_CUDA_TRY(numb.release_on(st));
    return denb.release_on(st);
  }
  static cudaError_t upload_pow_table(cudaStream_t st, const Fr& x, AsyncBuf& d_pw) {
    Fr pw[64];
    Fr b = x;
    for (int j = 0; j < 64; j++) { pw[j] = b; b = b.sqr(); }
    GB_CUDA_TRY(d_pw.alloc(sizeof(pw), st));
    GB_CUDA_TRY(cudaMemcpyAsync(d_pw.p, pw, sizeof(pw), cudaMemcpyHostToDevice, st));
    return cudaStreamSynchronize(st);  // pw is a stack buffer
  }
  static cudaError_t poly_eval(cudaStream_t st, const void* c, size_t n, const void* x_, void* out_host) {
    const Fr x = *(const Fr*)x_;
    if (n == 0) { *(Fr*)out_host = Fr::zero(); return cudaSuccess; }
    AsyncBuf pwb, sumsb;
    GB_CUDA_TRY(upload_pow_table(st, x, pwb));
    Fr* d_pw = (Fr*)pwb.p;
    const size_t nblocks = (n + 256 * EVAL_E - 1) / (256 * EVAL_E);
    GB_CUDA_TRY(sumsb.alloc((nblocks + 1) * sizeof(Fr), st));
    Fr* sums = (Fr*)sumsb.p;
    k_poly_eval_partial<Fr><<<(unsigned)nblocks, 256, 0, st>>>((const Fr*)c, n, d_pw, x, sums);
    k_sum_reduce<Fr><<<1, 256, 0, st>>>(sums, nblocks, sums + nblocks);
    GB_CUDA_TRY(cudaGetLastError());
    GB_CUDA_TRY(cudaMemcpyAsync(out_host, sums + nblocks, sizeof(Fr), cudaMemcpyDeviceToHost, st));
    GB_CUDA_TRY(sumsb.release_on(st));
    GB_CUDA_TRY(pwb.release_on(st));
    return cudaStreamSynchronize(st);
  }
  // in place: coeffs[0..n-2] <- (p(X) - p(z)) / (X - z), coeffs[n-1] <- 0; remainder p(z) to the host
  static cudaError_t poly_div_linear(cudaStream_t st, void* c_, size_t n, const void* z_, void* rem_host) {
    Fr* c = (Fr*)c_;
    const Fr z = *(const Fr*)z_;
    if (n == 0) { *(Fr*)rem_host = Fr::zero(); return cudaSuccess; }
    if (z.is_zero()) {
      // q_i = c_{i+1}, remainder c_0
      GB_CUDA_TRY(cudaMemcpyAsync(rem_host, c, sizeof(Fr), cudaMemcpyDeviceToHost, st));
      AsyncBuf tmpb;
      GB_CUDA_TRY(tmpb.alloc(n * sizeof(Fr), st));
      Fr* tmp = (Fr*)tmpb.p;
      GB_CUDA_TRY(cudaMemcpyAsync(tmp, c, n * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
      if (n > 1) GB_CUDA_TRY(cudaMemcpyAsync(c, tmp + 1, (n - 1) * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
      GB_CUDA_TRY(cudaMemsetAsync(c + (n - 1), 0, sizeof(Fr), st));
      GB_CUDA_TRY(tmpb.release_on(st));
      return cudaStreamSynchronize(st);
    }
    const Fr zinv = z.inverse();
    AsyncBuf pwb, pwib, tb, remb;
    GB_CUDA_TRY(upload_pow_table(st, z, pwb));
    GB_CUDA_TRY(upload_pow_table(st, zinv, pwib));
    GB_CUDA_TRY(tb.alloc(n * sizeof(Fr), st));
    GB_CUDA_TRY(remb.alloc(sizeof(Fr), st));
    Fr *d_pw = (Fr*)pwb.p, *d_pwi = (Fr*)pwib.p, *t = (Fr*)tb.p, *d_rem = (Fr*)remb.p;
    const unsigned nb = (unsigned)((n + 256 * EVAL_E - 1) / (256 * EVAL_E));
    k_syndiv_pre<Fr><<<nb, 256, 0, st>>>(c, n, d_pwi, zinv, t);
    GB_CUDA_TRY((scan_enqueue<Fr, 1>(st, t, n, false)));
    k_syndiv_post<Fr><<<nb, 256, 0, st>>>(t, n, d_pw, z, c, d_rem);
    GB_CUDA_TRY(cudaGetLastError());
    GB_CUDA_TRY(cudaMemcpyAsync(rem_host, d_rem, sizeof(Fr), cudaMemcpyDeviceToHost, st));
    GB_CUDA_TRY(tb.release_on(st)); GB_CUDA_TRY(remb.release_on(st));
    GB_CUDA_TRY(pwb.release_on(st)); GB_CUDA_TRY(pwib.release_on(st));
    return cudaStreamSynchronize(st);
  }
  // ---- batches of polynomials (item-major rows of n coefficients), enqueued on `st` without a host synchronisation:
  // the point tables go up in one copy from a pageable host buffer, which cudaMemcpyAsync has consumed when it returns
  static cudaError_t upload_pow_tables(cudaStream_t st, const Fr* pts, size_t batch, uint32_t len, bool with_inv,
                                       AsyncBuf& d_pw) {
    std::vector<Fr> tab((with_inv ? 2 : 1) * batch * len);
    kzg_pow_tables<Fr>(pts, batch, len, with_inv, tab.data());
    GB_CUDA_TRY(d_pw.alloc(tab.size() * sizeof(Fr), st));
    return cudaMemcpyAsync(d_pw.p, tab.data(), tab.size() * sizeof(Fr), cudaMemcpyHostToDevice, st);
  }
  // d_values[b] = p_b(points[b]); points on the host
  static cudaError_t poly_eval_batch(cudaStream_t st, const void* polys, size_t n, size_t batch, const void* points_host,
                                     void* d_values) {
    if (!batch) return cudaSuccess;
    if (n == 0) return cudaMemsetAsync(d_values, 0, batch * sizeof(Fr), st);
    const uint32_t len = kzg_pow_len(n);
    AsyncBuf pwb, sumsb;
    GB_CUDA_TRY(upload_pow_tables(st, (const Fr*)points_host, batch, len, false, pwb));
    const size_t nblocks = (n + 256 * EVAL_E - 1) / (256 * EVAL_E);
    GB_CUDA_TRY(sumsb.alloc(batch * nblocks * sizeof(Fr), st));
    const Fr *c = (const Fr*)polys, *pw = (const Fr*)pwb.p;
    Fr *sums = (Fr*)sumsb.p, *vals = (Fr*)d_values;
    for (size_t b0 = 0; b0 < batch; b0 += NTT_MAX_GRID_Y) {
      const unsigned rows = (unsigned)(batch - b0 < NTT_MAX_GRID_Y ? batch - b0 : NTT_MAX_GRID_Y);
      k_poly_eval_partial<Fr, true><<<dim3((unsigned)nblocks, rows), 256, 0, st>>>(c + b0 * n, n, pw + b0 * len, Fr::zero(),
                                                                                 sums + b0 * nblocks, len);
      k_sum_reduce<Fr, true><<<dim3(1, rows), 256, 0, st>>>(sums + b0 * nblocks, nblocks, vals + b0);
      GB_CUDA_TRY(cudaGetLastError());
    }
    GB_CUDA_TRY(sumsb.release_on(st));
    return pwb.release_on(st);
  }
  // row b of d_q <- (p_b(X) - p_b(z_b)) / (X - z_b) (top coefficient zeroed), d_values[b] <- p_b(z_b); the polynomials
  // are only read.  Points on the host; a point of 0 divides by X.
  static cudaError_t poly_div_linear_batch(cudaStream_t st, const void* polys, size_t n, size_t batch,
                                           const void* points_host, void* d_q, void* d_values) {
    if (!batch) return cudaSuccess;
    if (n == 0) return cudaMemsetAsync(d_values, 0, batch * sizeof(Fr), st);
    const uint32_t len = kzg_pow_len(n);
    AsyncBuf pwb, tb;
    GB_CUDA_TRY(upload_pow_tables(st, (const Fr*)points_host, batch, len, true, pwb));
    GB_CUDA_TRY(tb.alloc(batch * n * sizeof(Fr), st));
    const Fr *c = (const Fr*)polys, *pw = (const Fr*)pwb.p, *pwi = pw + batch * len;
    Fr *t = (Fr*)tb.p, *q = (Fr*)d_q, *vals = (Fr*)d_values;
    const unsigned nb = (unsigned)((n + 256 * EVAL_E - 1) / (256 * EVAL_E));
    for (size_t b0 = 0; b0 < batch; b0 += NTT_MAX_GRID_Y) {
      const unsigned rows = (unsigned)(batch - b0 < NTT_MAX_GRID_Y ? batch - b0 : NTT_MAX_GRID_Y);
      const size_t off = b0 * n;
      k_syndiv_pre<Fr, true><<<dim3(nb, rows), 256, 0, st>>>(c + off, n, pwi + b0 * len, Fr::zero(), t + off, len);
      GB_CUDA_TRY(cudaGetLastError());
      GB_CUDA_TRY((scan_enqueue<Fr, 1, true>(st, t + off, n, false, rows)));
      k_syndiv_post<Fr, true><<<dim3(nb, rows), 256, 0, st>>>(t + off, n, pw + b0 * len, Fr::zero(), q + off, vals + b0, len,
                                                             c + off);
      GB_CUDA_TRY(cudaGetLastError());
    }
    GB_CUDA_TRY(tb.release_on(st));
    return pwb.release_on(st);
  }
  // d_out[j] = sum_b gamma^b p_b[j], j < n (batch >= 1)
  static cudaError_t poly_fold(cudaStream_t st, const void* polys, size_t n, size_t batch, const void* gamma, void* d_out) {
    if (!n || !batch) return cudaSuccess;
    k_poly_fold<Fr><<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const Fr*)polys, n, batch, *(const Fr*)gamma, (Fr*)d_out);
    return cudaGetLastError();
  }
  static cudaError_t gather(cudaStream_t st, void* out, const void* src, const uint32_t* idx, size_t n) {
    if (!n) return cudaSuccess;
    k_gather<Fr><<<(unsigned)((n + 255) / 256), 256, 0, st>>>((Fr*)out, (const Fr*)src, idx, n);
    return cudaGetLastError();
  }
  static cudaError_t gather_batch(cudaStream_t st, void* out, const void* src, const uint32_t* idx, size_t n, size_t batch,
                                  size_t src_stride, size_t out_stride) {
    if (!n || !batch) return cudaSuccess;
    for (size_t b0 = 0; b0 < batch; b0 += NTT_MAX_GRID_Y) {     // the y dimension's limit, as for the NTT
      const unsigned rows = (unsigned)(batch - b0 < NTT_MAX_GRID_Y ? batch - b0 : NTT_MAX_GRID_Y);
      k_gather_batch<Fr><<<dim3((unsigned)((n + 255) / 256), rows), 256, 0, st>>>(
          (Fr*)out + b0 * out_stride, (const Fr*)src + b0 * src_stride, idx, (uint32_t)n, (uint32_t)src_stride,
          (uint32_t)out_stride);
      GB_CUDA_TRY(cudaGetLastError());
    }
    return cudaSuccess;
  }
  static const HostFrCtx* host_fr() {
    static const HostFrCtx c = HostFrCtx::make<typename Fr::Params>();
    return &c;
  }
  static const NttOps* ops() {
    static const NttOps o = {sizeof(Fr), Fr::Params::TWO_ADICITY, &domain_new, &domain_free, &domain_bytes, &ntt,
                             &compute_h, &vec_op, &bit_reverse, &scale_powers, &batch_invert, &plonk_coset,
                             &plonk_divide_by_zh, &axpy, &scan, &plonk_build_z, &poly_eval, &poly_div_linear, &gather,
                             &host_fr, &plonk_bsb22, &ntt_batch, &compute_h_batch, &gather_batch,
                             &poly_eval_batch, &poly_div_linear_batch, &poly_fold};
    return &o;
  }
};

// ---------------------------------------------------------------------------
// host group arithmetic (proof assembly)
// ---------------------------------------------------------------------------
template <class HFr, class HF>
struct HostGroupInst {
  using A = Affine<HF>;
  using J = Jacobian<HF>;
  using X = XYZZ<HF>;
  static X mul(const X& p, const HFr& k_mont) {
    HFr k = k_mont.from_mont();
    X acc = X::inf();
    for (int i = HFr::M - 1; i >= 0; i--)
      for (int b = 63; b >= 0; b--) {
        acc.dbl();
        if ((k.l[i] >> b) & 1) acc.add(p);
      }
    return acc;
  }
  static void scalar_mul_affine(const void* p, const void* k, void* out) {
    *reinterpret_cast<J*>(out) = mul(X::from_affine(*reinterpret_cast<const A*>(p)), *reinterpret_cast<const HFr*>(k)).to_jacobian();
  }
  static void scalar_mul_jac(const void* p, const void* k, void* out) {
    *reinterpret_cast<J*>(out) = mul(X::from_jacobian(*reinterpret_cast<const J*>(p)), *reinterpret_cast<const HFr*>(k)).to_jacobian();
  }
  static void add_jac(void* acc, const void* q) {
    X a = X::from_jacobian(*reinterpret_cast<J*>(acc));
    a.add(X::from_jacobian(*reinterpret_cast<const J*>(q)));
    *reinterpret_cast<J*>(acc) = a.to_jacobian();
  }
  static void add_mixed(void* acc, const void* q) {
    X a = X::from_jacobian(*reinterpret_cast<J*>(acc));
    a.add_mixed(*reinterpret_cast<const A*>(q));
    *reinterpret_cast<J*>(acc) = a.to_jacobian();
  }
  static void to_affine(const void* p, void* out) {
    *reinterpret_cast<A*>(out) = X::from_jacobian(*reinterpret_cast<const J*>(p)).to_affine();
  }
  static void fr_neg_mul(const void* a, const void* b, void* out) {
    *reinterpret_cast<HFr*>(out) = ((*reinterpret_cast<const HFr*>(a)) * (*reinterpret_cast<const HFr*>(b))).neg();
  }
  static const HostGroupOps* ops() {
    static const HostGroupOps o = {sizeof(A), sizeof(J), sizeof(HFr), &scalar_mul_affine, &scalar_mul_jac, &add_jac,
                                   &add_mixed, &to_affine, &fr_neg_mul};
    return &o;
  }
};

#define GB200_REGISTER_MSM(TAG, ID, GROUP, FR, F)                                  \
  namespace {                                                                       \
  struct RegistrarMsm_##TAG {                                                       \
    RegistrarMsm_##TAG() { register_msm_ops(ID, GROUP, MsmInst<FR, F>::ops()); }    \
  } registrar_msm_##TAG;                                                            \
  }
#define GB200_REGISTER_MSM_G1(TAG, ID, FR, F)                                     \
  namespace {                                                                       \
  struct RegistrarMsm_##TAG {                                                       \
    RegistrarMsm_##TAG() { register_msm_ops(ID, 1, MsmInst<FR, F>::ops_g1()); }     \
  } registrar_msm_##TAG;                                                            \
  }
#define GB200_REGISTER_FR(TAG, ID, FR, HFR, HFP, HG2F)                             \
  namespace {                                                                       \
  struct RegistrarFr_##TAG {                                                        \
    RegistrarFr_##TAG() {                                                           \
      register_ntt_ops(ID, NttInst<FR>::ops());                                     \
      register_host_group_ops(ID, 1, HostGroupInst<HFR, HFP>::ops());               \
      register_host_group_ops(ID, 2, HostGroupInst<HFR, HG2F>::ops());              \
    }                                                                               \
  } registrar_fr_##TAG;                                                             \
  }

}  // namespace gb200
