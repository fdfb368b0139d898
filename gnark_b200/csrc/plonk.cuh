// PLONK quotient building blocks (SURVEY.md §8 rows a10/a11): the fused constraint
// evaluation of computeNumerator (backend/plonk/bn254/prove.go:841-1123, closures
// gateConstraint :871-889, orderingConstraint :907-931, localConstraint :933-941,
// allConstraints :961-988), the 1/(X^n - 1) scaling of divideByZH (:1287-1324) and a
// parallel batch inversion (batchInvert :1130-1143).  No BSB22 commitment gates yet.
#pragma once
#ifdef __CUDACC__
#include <cuda_runtime.h>
#endif

#include "ntt.cuh"

namespace gb200 {

constexpr int PLONK_MAX_BLIND = 4;  // blinding polynomials have degree <= 2 (order 1 or 2) in the reference

template <class Fr>
struct PlonkCosetArgs {
  // device vectors, n elements each, Lagrange basis ON THE CURRENT COSET, regular (natural) layout
  const Fr *l, *r, *o, *z, *s1, *s2, *s3, *ql, *qr, *qm, *qo, *qk;
  const Fr* tw;          // w^j, j < n/2 (domain0 twiddles)
  const Fr* den_inv;     // 1 / (coset*w^j - 1), j < n   (precomputedDenominators, :1002-1007)
  Fr* out;               // rho*n elements, LagrangeCoset on the big domain, BIT-REVERSED layout
  Fr alpha, beta, gamma;
  Fr coset;              // current coset shift  (g, g*w4, g*w4^2, ...)
  Fr cs, css;            // domain1.FrMultiplicativeGen and its square (:891-893)
  Fr coset_n_minus_one;  // coset^n - 1
  Fr lone_scale;         // (coset^n - 1) / n
  // blinding coefficients ALREADY multiplied by coset^n - 1 (plonk_set_blinding): on a coset X^n - 1 is that constant, so
  // p + (X^n - 1) b(X) costs deg(b) multiplications per point instead of deg(b) + 2 (the reference pre-scales too, :967-981)
  Fr bl[PLONK_MAX_BLIND], br[PLONK_MAX_BLIND], bo[PLONK_MAX_BLIND], bz[PLONK_MAX_BLIND];
  int nbl, nbr, nbo, nbz;  // number of blinding coefficients
  uint32_t n, logn, rho, log_rho, coset_index;
};

template <class Fr>
HD Fr plonk_horner(const Fr* c, int nc, const Fr& x) {
  if (nc <= 0) return Fr::zero();
  Fr acc = c[nc - 1];
  for (int k = nc - 2; k >= 0; k--) acc = acc * x + c[k];
  return acc;
}

// dst[k] = (coset^n - 1) * src[k] for k < nb, zero above; a.coset_n_minus_one must be set
template <class Fr>
HD void plonk_set_blinding(const PlonkCosetArgs<Fr>& a, Fr* dst, const Fr* src, int nb) {
  for (int k = 0; k < PLONK_MAX_BLIND; k++) dst[k] = k < nb ? a.coset_n_minus_one * src[k] : Fr::zero();
}

// One point of one coset.  wj = w^j, wj1 = w^(j+1 mod n).
template <class Fr>
HD Fr plonk_all_constraints(const PlonkCosetArgs<Fr>& a, uint32_t j, const Fr& wj, const Fr& wj1) {
  const uint32_t j1 = (j + 1 == a.n) ? 0 : j + 1;
  const Fr x = a.coset * wj;     // evaluation point
  const Fr x1 = a.coset * wj1;
  // blinded L, R, O, Z, ZS: p + (X^n - 1) b(X) on the coset (:967-981; the reference pre-scales b's
  // coefficients so that evaluating at w^j yields exactly this value)
  Fr L = a.l[j] + plonk_horner(a.bl, a.nbl, x);
  Fr R = a.r[j] + plonk_horner(a.br, a.nbr, x);
  Fr O = a.o[j] + plonk_horner(a.bo, a.nbo, x);
  Fr Z = a.z[j] + plonk_horner(a.bz, a.nbz, x);
  Fr ZS = a.z[j1] + plonk_horner(a.bz, a.nbz, x1);
  // gate (:871-889)
  Fr gate = a.ql[j] * L + a.qr[j] * R + a.qm[j] * L * R + a.qo[j] * O + a.qk[j];
  // ordering (:907-931)
  Fr id = x * a.beta;
  Fr t0 = a.gamma + L + id;
  Fr t1 = id * a.cs + R + a.gamma;
  Fr t2 = id * a.css + O + a.gamma;
  Fr rr = t0 * t1 * t2 * Z;
  t0 = a.s1[j] * a.beta + L + a.gamma;
  t1 = a.s2[j] * a.beta + R + a.gamma;
  t2 = a.s3[j] * a.beta + O + a.gamma;
  Fr ordering = t0 * t1 * t2 * ZS - rr;
  // local (:933-941): (Z - 1) * L1(x), L1(x) = (x^n - 1) / (n (x - 1))
  Fr local = (Z - Fr::one()) * (a.lone_scale * a.den_inv[j]);
  return (local * a.alpha + ordering) * a.alpha + gate;   // :985
}

// BSB22 commitment gate (gateConstraint :881-884): the term Qcp_i * PI2_i of one commitment at point j of one coset,
// added to the slot the fused kernel wrote (the gate enters allConstraints with coefficient 1, so the sum can be
// completed afterwards, one call per commitment and coset)
HD uint32_t plonk_scatter_index(uint32_t j, uint32_t coset_index, uint32_t rho, uint32_t logn, uint32_t log_rho) {
  return ntt_bitrev(rho * j + coset_index, (int)(logn + log_rho));
}
template <class Fr>
HD void plonk_add_bsb22_point(const Fr* qcp, const Fr* pi2, Fr* out, uint32_t j, uint32_t coset_index, uint32_t rho,
                              uint32_t logn, uint32_t log_rho) {
  const uint32_t k = plonk_scatter_index(j, coset_index, rho, logn, log_rho);
  out[k] = out[k] + qcp[j] * pi2[j];
}

#ifdef __CUDACC__
template <class Fr>
__global__ void __launch_bounds__(256) k_plonk_add_bsb22(const Fr* __restrict__ qcp, const Fr* __restrict__ pi2,
                                                         Fr* __restrict__ out, uint32_t n, uint32_t coset_index,
                                                         uint32_t rho, uint32_t logn, uint32_t log_rho) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) plonk_add_bsb22_point<Fr>(qcp, pi2, out, j, coset_index, rho, logn, log_rho);
}

// 128-thread blocks, 4 resident per SM asked of ptxas (<= 128 registers): left alone the kernel takes 136 registers and,
// with the 256-thread blocks of round 1, ran ONE block = 8 warps per SM - a chain of ~30 dependent field products per
// thread with nothing to overlap it (4.3 ms per coset at 2^22 against a 1.9 ms multiplier bound)
template <class Fr>
__global__ void __launch_bounds__(128, 4) k_plonk_constraints(PlonkCosetArgs<Fr> a) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.n) return;
  const uint32_t half = a.n >> 1;
  // w^j for j >= n/2 is -w^(j - n/2)
  auto w_at = [&](uint32_t k) -> Fr {
    if (a.n == 1) return Fr::one();
    return k < half ? a.tw[k] : a.tw[k - half].neg();
  };
  const uint32_t j1 = (j + 1 == a.n) ? 0 : j + 1;
  const Fr v = plonk_all_constraints<Fr>(a, j, w_at(j), w_at(j1));
  // cres[bitrev_{rho n}(rho*j + i)] (:1070-1076)
  const uint32_t m = a.rho * j + a.coset_index;
  a.out[ntt_bitrev(m, (int)(a.logn + a.log_rho))] = v;
}

// r[i] *= tab[bitrev(i) % rho]   (divideByZH :1312-1317)
template <class Fr>
__global__ void __launch_bounds__(256) k_plonk_zh_scale(Fr* __restrict__ r, uint32_t logm, uint32_t rho,
                                                        const Fr* __restrict__ tab) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (1u << logm)) return;
  r[i] = r[i] * tab[ntt_bitrev(i, (int)logm) % rho];
}

// in-place batch inversion, one thread per chunk of BI_CHUNK elements (Montgomery's trick);
// zeros are left as zeros.
constexpr int BI_CHUNK = 32;
template <class Fr>
__global__ void __launch_bounds__(128) k_batch_invert(Fr* __restrict__ v, size_t n) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t lo = t * BI_CHUNK;
  if (lo >= n) return;
  const size_t hi = lo + BI_CHUNK < n ? lo + BI_CHUNK : n;
  Fr pre[BI_CHUNK];
  Fr acc = Fr::one();
  for (size_t i = lo; i < hi; i++) {
    pre[i - lo] = acc;
    const Fr x = v[i];
    if (!x.is_zero()) acc = acc * x;
  }
  Fr inv = acc.inverse();
  for (size_t i = hi; i-- > lo;) {
    const Fr x = v[i];
    if (x.is_zero()) continue;
    v[i] = inv * pre[i - lo];
    inv = inv * x;
  }
}

// d[j] = coset * w^j - 1   (then batch-inverted: precomputedDenominators)
template <class Fr>
__global__ void __launch_bounds__(256) k_plonk_denominators(Fr* __restrict__ d, uint32_t n, const Fr* __restrict__ tw,
                                                            Fr coset) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t half = n >> 1;
  Fr w = n == 1 ? Fr::one() : (j < half ? tw[j] : tw[j - half].neg());
  d[j] = coset * w - Fr::one();
}
#endif

}  // namespace gb200

// ---------------------------------------------------------------------------------------------
// O(n) scans of the PLONK prover on device (SURVEY.md §8 row a11 / §8f-2): prefix scans over Fr,
// the permutation grand product Z (iop.BuildRatioCopyConstraint, plonk/bn254/prove.go:645-656),
// polynomial evaluation (Polynomial.Evaluate :742,1191,1382) and division by (X - z)
// (the quotient inside kzg.Open / BatchOpenSinglePoint :681,827).
// ---------------------------------------------------------------------------------------------
namespace gb200 {

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_E = 4;   // elements per thread

template <class Fr, int OP>   // OP 0: product, 1: sum
HD Fr scan_op(const Fr& a, const Fr& b) { return OP == 0 ? a * b : a + b; }
template <class Fr, int OP>
HD Fr scan_identity() { return OP == 0 ? Fr::one() : Fr::zero(); }

// x^k by square-and-multiply from pw[j] = x^(2^j)
template <class Fr>
HD Fr pow_from_table(const Fr* __restrict__ pw, size_t k) {
  Fr acc = Fr::one();
  for (int j = 0; k; j++, k >>= 1)
    if (k & 1) acc = acc * pw[j];
  return acc;
}

#ifdef __CUDACC__
// block-local scan of SCAN_THREADS*SCAN_E elements; block totals to block_sums (nullable).  kBatch: blockIdx.y selects
// the row (n elements at data + row * n) and the row's block totals go to block_sums + row * gridDim.x; blocks never
// span two rows.
template <class Fr, int OP, bool kBatch = false>
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_block(Fr* __restrict__ data, size_t n, Fr* __restrict__ block_sums,
                                                             int exclusive) {
  __shared__ Fr sm[SCAN_THREADS];
  if (kBatch) {
    data += (size_t)blockIdx.y * n;
    if (block_sums) block_sums += (size_t)blockIdx.y * gridDim.x;
  }
  const size_t base = ((size_t)blockIdx.x * SCAN_THREADS + threadIdx.x) * SCAN_E;
  Fr v[SCAN_E];
#pragma unroll
  for (int k = 0; k < SCAN_E; k++) v[k] = base + k < n ? data[base + k] : scan_identity<Fr, OP>();
#pragma unroll
  for (int k = 1; k < SCAN_E; k++) v[k] = scan_op<Fr, OP>(v[k - 1], v[k]);
  sm[threadIdx.x] = v[SCAN_E - 1];
  __syncthreads();
  for (int off = 1; off < SCAN_THREADS; off <<= 1) {
    Fr x = sm[threadIdx.x];
    if ((int)threadIdx.x >= off) x = scan_op<Fr, OP>(sm[threadIdx.x - off], x);
    __syncthreads();
    sm[threadIdx.x] = x;
    __syncthreads();
  }
  const Fr prefix = threadIdx.x == 0 ? scan_identity<Fr, OP>() : sm[threadIdx.x - 1];
  if (block_sums && threadIdx.x == SCAN_THREADS - 1) block_sums[blockIdx.x] = sm[SCAN_THREADS - 1];
#pragma unroll
  for (int k = 0; k < SCAN_E; k++) {
    if (base + k >= n) break;
    if (exclusive) data[base + k] = k == 0 ? prefix : scan_op<Fr, OP>(prefix, v[k - 1]);
    else data[base + k] = scan_op<Fr, OP>(prefix, v[k]);
  }
}
template <class Fr, int OP, bool kBatch = false>
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_fix(Fr* __restrict__ data, size_t n,
                                                           const Fr* __restrict__ block_prefix) {
  if (blockIdx.x == 0) return;
  if (kBatch) {
    data += (size_t)blockIdx.y * n;
    block_prefix += (size_t)blockIdx.y * gridDim.x;
  }
  const Fr p = block_prefix[blockIdx.x];
  const size_t base = ((size_t)blockIdx.x * SCAN_THREADS + threadIdx.x) * SCAN_E;
#pragma unroll
  for (int k = 0; k < SCAN_E; k++)
    if (base + k < n) data[base + k] = scan_op<Fr, OP>(p, data[base + k]);
}

// in-place scan of n elements on `st` (recursive over block totals).  kBatch: `rows` (<= 65 535, the grid's y limit)
// independent scans of n elements each, item-major, their block totals scanned per row.
template <class Fr, int OP, bool kBatch = false>
cudaError_t scan_enqueue(cudaStream_t st, Fr* data, size_t n, bool exclusive, unsigned rows = 1) {
  if (n == 0) return cudaSuccess;
  const size_t per_block = (size_t)SCAN_THREADS * SCAN_E;
  const size_t nblocks = (n + per_block - 1) / per_block;
  if (nblocks == 1) {
    k_scan_block<Fr, OP, kBatch><<<dim3(1, rows), SCAN_THREADS, 0, st>>>(data, n, nullptr, exclusive ? 1 : 0);
    return cudaGetLastError();
  }
  Fr* sums = nullptr;
  cudaError_t e = cudaMallocAsync(&sums, (size_t)rows * nblocks * sizeof(Fr), st);
  if (e != cudaSuccess) return e;
  k_scan_block<Fr, OP, kBatch><<<dim3((unsigned)nblocks, rows), SCAN_THREADS, 0, st>>>(data, n, sums, exclusive ? 1 : 0);
  e = scan_enqueue<Fr, OP, kBatch>(st, sums, nblocks, true, rows);
  if (e == cudaSuccess) {
    k_scan_fix<Fr, OP, kBatch><<<dim3((unsigned)nblocks, rows), SCAN_THREADS, 0, st>>>(data, n, sums);
    e = cudaGetLastError();
  }
  cudaError_t e2 = cudaFreeAsync(sums, st);
  return e != cudaSuccess ? e : e2;
}

// permutation ratios: num[i] = prod_j (f_j[i] + beta*id_j(i) + gamma), den[i] = prod_j (f_j[i] + beta*supp[S[j n+i]] + gamma)
// supp[k] = g^(k / n) * w^(k % n)   (getSupportPermutation, plonk/bn254/setup.go:377-392)
template <class Fr>
__global__ void __launch_bounds__(256) k_plonk_ratio_terms(uint32_t n, const Fr* __restrict__ l, const Fr* __restrict__ r,
                                                           const Fr* __restrict__ o, const int64_t* __restrict__ S,
                                                           const Fr* __restrict__ tw, Fr beta, Fr gamma, Fr g,
                                                           Fr* __restrict__ num, Fr* __restrict__ den) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t half = n >> 1;
  auto w_at = [&](uint32_t k) -> Fr { return n == 1 ? Fr::one() : (k < half ? tw[k] : tw[k - half].neg()); };
  const Fr g2 = g * g;
  auto supp = [&](int64_t k) -> Fr {
    const uint32_t blk = (uint32_t)(k / n), idx = (uint32_t)(k % n);
    const Fr w = w_at(idx);
    return blk == 0 ? w : (blk == 1 ? g * w : g2 * w);
  };
  const Fr f[3] = {l[i], r[i], o[i]};
  const Fr wi = w_at(i);
  const Fr id[3] = {wi, g * wi, g2 * wi};
  Fr a = Fr::one(), b = Fr::one();
#pragma unroll
  for (int j = 0; j < 3; j++) {
    a = a * (f[j] + beta * id[j] + gamma);
    b = b * (f[j] + beta * supp(S[(size_t)j * n + i]) + gamma);
  }
  num[i] = a;
  den[i] = b;
}
// z[0] = 1, z[i+1] = ratio[i] for i < n-1 (then an inclusive product scan yields Z)
template <class Fr>
__global__ void __launch_bounds__(256) k_plonk_shift_ratio(uint32_t n, const Fr* __restrict__ num,
                                                           const Fr* __restrict__ den_inv, Fr* __restrict__ z) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  z[i] = i == 0 ? Fr::one() : num[i - 1] * den_inv[i - 1];
}

#endif

// ---- per-thread steps of evaluation and division (shared by the kernels below and their host emulation) ----
// Thread t of block blk handles the EVAL_E coefficients from base = (blk * 256 + t) * EVAL_E of its polynomial.
constexpr int EVAL_E = 8;

// the thread's share of p(x): sum_{k < EVAL_E} c[base + k] x^(base + k)  (zero past the end)
template <class Fr>
HD Fr poly_eval_chunk(const Fr* __restrict__ c, size_t n, const Fr* __restrict__ pw, const Fr& x, size_t base) {
  Fr acc = Fr::zero();
  if (base < n) {
#pragma unroll
    for (int k = EVAL_E - 1; k >= 0; k--) acc = acc * x + (base + k < n ? c[base + k] : Fr::zero());
    acc = acc * pow_from_table<Fr>(pw, base);
  }
  return acc;
}

// synthetic division by (X - z), z != 0:  t_k = c_{n-1-k} z^-k ; s = inclusive sum scan(t) ;
// q_{n-2-k} = s_k z^k (k <= n-2) ; remainder = s_{n-1} z^(n-1) = p(z)
template <class Fr>
HD void syndiv_pre_chunk(const Fr* __restrict__ c, size_t n, const Fr* __restrict__ pw_inv, const Fr& zinv,
                         Fr* __restrict__ t, size_t base) {
  if (base >= n) return;
  Fr p = pow_from_table<Fr>(pw_inv, base);
#pragma unroll
  for (int k = 0; k < EVAL_E; k++) {
    if (base + k >= n) break;
    t[base + k] = c[n - 1 - (base + k)] * p;
    p = p * zinv;
  }
}
template <class Fr>
HD void syndiv_post_chunk(const Fr* __restrict__ s, size_t n, const Fr* __restrict__ pw, const Fr& z, Fr* __restrict__ q,
                          Fr* __restrict__ rem, size_t base) {
  if (base >= n) return;
  Fr p = pow_from_table<Fr>(pw, base);
#pragma unroll
  for (int k = 0; k < EVAL_E; k++) {
    const size_t kk = base + k;
    if (kk >= n) break;
    const Fr v = s[kk] * p;
    if (kk == n - 1) { *rem = v; q[n - 1] = Fr::zero(); }
    else q[n - 2 - kk] = v;
    p = p * z;
  }
}
// division by X: q_i = c_{i+1}, q_{n-1} = 0, remainder c_0 (a batch item whose point is 0)
template <class Fr>
HD void syndiv_zero_chunk(const Fr* __restrict__ c, size_t n, Fr* __restrict__ q, Fr* __restrict__ rem, size_t base) {
  for (int k = 0; k < EVAL_E; k++) {
    const size_t kk = base + k;
    if (kk >= n) break;
    q[kk] = kk + 1 < n ? c[kk + 1] : Fr::zero();
    if (kk == 0) *rem = c[0];
  }
}
// out[j] = sum_b gamma^b p_b[j] over `batch` item-major polynomials of n coefficients (Horner in gamma, gamma^0 = 1)
template <class Fr>
HD Fr poly_fold_coeff(const Fr* __restrict__ polys, size_t n, size_t batch, const Fr& gamma, size_t j) {
  Fr acc = polys[(batch - 1) * n + j];
  for (size_t b = batch - 1; b-- > 0;) acc = acc * gamma + polys[b * n + j];
  return acc;
}

// Power tables of a batch of points: entries j <= ceil(log2 n) of x^(2^j), which is every entry pow_from_table reads for
// an exponent below n (and entry 0 is the point itself)
HD uint32_t kzg_pow_len(size_t n) {
  uint32_t l = 0;
  while (l < 63 && ((size_t)1 << l) < n) l++;
  return l + 1;
}
// out[b * len + j] = x_b^(2^j); with_inv: then out[(batch + b) * len + j] = x_b^(-2^j), the batch's inverses from ONE
// inversion (Montgomery's trick; a zero point gets a zero table)
template <class Fr>
void kzg_pow_tables(const Fr* pts, size_t batch, uint32_t len, bool with_inv, Fr* out) {
  for (int half = 0; half < (with_inv ? 2 : 1); half++) {
    Fr* o = out + (size_t)half * batch * len;
    if (half == 1) {
      // prefix products of the non-zero points, one inversion, then back to front
      Fr acc = Fr::one();
      for (size_t b = 0; b < batch; b++) {
        o[b * len] = acc;
        if (!pts[b].is_zero()) acc = acc * pts[b];
      }
      Fr inv = acc.inverse();
      for (size_t b = batch; b-- > 0;) {
        if (pts[b].is_zero()) { o[b * len] = Fr::zero(); continue; }
        o[b * len] = inv * o[b * len];
        inv = inv * pts[b];
      }
    } else {
      for (size_t b = 0; b < batch; b++) o[b * len] = pts[b];
    }
    for (size_t b = 0; b < batch; b++)
      for (uint32_t j = 1; j < len; j++) o[b * len + j] = o[b * len + j - 1].sqr();
  }
}

#ifdef __CUDACC__
// polynomial evaluation: block partial sums of c_i x^i.  kBatch: blockIdx.y selects the polynomial (n coefficients at
// c + row * n), whose point is pw[row * pw_len] (its table's entry 0) and whose block sums go to row `row` of
// block_sums (gridDim.x each)
template <class Fr, bool kBatch = false>
__global__ void __launch_bounds__(256) k_poly_eval_partial(const Fr* __restrict__ c, size_t n, const Fr* __restrict__ pw,
                                                           Fr x, Fr* __restrict__ block_sums, uint32_t pw_len = 0) {
  __shared__ Fr sm[256];
  if (kBatch) {
    c += (size_t)blockIdx.y * n;
    pw += (size_t)blockIdx.y * pw_len;
    x = pw[0];
    block_sums += (size_t)blockIdx.y * gridDim.x;
  }
  const size_t base = ((size_t)blockIdx.x * 256 + threadIdx.x) * EVAL_E;
  sm[threadIdx.x] = poly_eval_chunk<Fr>(c, n, pw, x, base);
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) sm[threadIdx.x] = sm[threadIdx.x] + sm[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) block_sums[blockIdx.x] = sm[0];
}
// kBatch: blockIdx.y selects the row of n values at v + row * n, whose sum goes to out[row]
template <class Fr, bool kBatch = false>
__global__ void __launch_bounds__(256) k_sum_reduce(const Fr* __restrict__ v, size_t n, Fr* __restrict__ out) {
  __shared__ Fr sm[256];
  if (kBatch) {
    v += (size_t)blockIdx.y * n;
    out += blockIdx.y;
  }
  Fr acc = Fr::zero();
  for (size_t i = threadIdx.x; i < n; i += 256) acc = acc + v[i];
  sm[threadIdx.x] = acc;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) sm[threadIdx.x] = sm[threadIdx.x] + sm[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = sm[0];
}

// kBatch (both passes): blockIdx.y selects the polynomial, rows of n at c, t, s and q; its tables start at
// pw_inv / pw + row * pw_len and its point is their entry 0; the remainder goes to rem[row]
template <class Fr, bool kBatch = false>
__global__ void __launch_bounds__(256) k_syndiv_pre(const Fr* __restrict__ c, size_t n, const Fr* __restrict__ pw_inv,
                                                    Fr zinv, Fr* __restrict__ t, uint32_t pw_len = 0) {
  if (kBatch) {
    c += (size_t)blockIdx.y * n;
    t += (size_t)blockIdx.y * n;
    pw_inv += (size_t)blockIdx.y * pw_len;
    zinv = pw_inv[0];
  }
  syndiv_pre_chunk<Fr>(c, n, pw_inv, zinv, t, ((size_t)blockIdx.x * 256 + threadIdx.x) * EVAL_E);
}
// kBatch: an item whose point is 0 takes its quotient from its coefficients c instead (syndiv_zero_chunk)
template <class Fr, bool kBatch = false>
__global__ void __launch_bounds__(256) k_syndiv_post(const Fr* __restrict__ s, size_t n, const Fr* __restrict__ pw, Fr z,
                                                     Fr* __restrict__ q, Fr* __restrict__ rem, uint32_t pw_len = 0,
                                                     const Fr* __restrict__ c = nullptr) {
  const size_t base = ((size_t)blockIdx.x * 256 + threadIdx.x) * EVAL_E;
  if (kBatch) {
    const size_t off = (size_t)blockIdx.y * n;
    s += off;
    q += off;
    pw += (size_t)blockIdx.y * pw_len;
    rem += blockIdx.y;
    z = pw[0];
    if (z.is_zero()) {
      syndiv_zero_chunk<Fr>(c + off, n, q, rem, base);
      return;
    }
  }
  syndiv_post_chunk<Fr>(s, n, pw, z, q, rem, base);
}

template <class Fr>
__global__ void __launch_bounds__(256) k_poly_fold(const Fr* __restrict__ polys, size_t n, size_t batch, Fr gamma,
                                                   Fr* __restrict__ out) {
  const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) out[j] = poly_fold_coeff<Fr>(polys, n, batch, gamma, j);
}
#endif

}  // namespace gb200
