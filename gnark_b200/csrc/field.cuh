// Prime-field arithmetic in Montgomery form, 32-bit limbs, for sm_90a.
//
// Memory layout is gnark-crypto's fp.Element / fr.Element bit for bit
// ([Limbs]uint64 little-endian, value x*R mod q, R = 2^(64*Limbs); SURVEY.md
// Appendix A, evidence backend/accelerated/icicle/groth16/bn254/icicle.go:119-130),
// so proving-key tables and witness vectors are used as uploaded: the
// reference's FromMontgomery / AffineFromMontgomery passes (icicle.go:121,322,350,
// 1008,1028,1452,1480) have no counterpart here.
//
// Multiplication: operand-scanning Montgomery product with TWO interleaved
// accumulators so that every 32x32 partial product (lo word, hi word) lands in a
// carry chain that visits each accumulator word exactly once:
//   row i adds a*b[i] and m_i*p;  products whose start position i+j is even go to
//   accumulator E, odd to O; both are indexed by ABSOLUTE word position, and the
//   word at position i of the "other" accumulator is folded in before m_i is
//   computed.  4N^2+N multiplier ops, no carry ripple, result < 2p, one
//   conditional subtraction.  (No tensor cores: integer path.)
#pragma once
#include "ptx.cuh"
#include "params_gen.cuh"

namespace gb200 {

// ---------------------------------------------------------------------------
// raw limb routines
// ---------------------------------------------------------------------------

// acc[base + j], acc[base + j + 1] += lo/hi(s[j] * m) for j = J0, J0+2, ... < N, one carry
// chain; the carry out of the chain is added to the next (fresh or carry-only) word.
template <int N, int J0, bool CARRY_IN>
HD void mad_chain(uint32_t* acc, int base, const uint32_t* s, uint32_t m) {
#pragma unroll
  for (int j = J0; j < N; j += 2) {
    if (j == J0 && !CARRY_IN)
      acc[base + j] = ptx::mad_lo_cc(s[j], m, acc[base + j]);
    else
      acc[base + j] = ptx::madc_lo_cc(s[j], m, acc[base + j]);
    acc[base + j + 1] = ptx::madc_hi_cc(s[j], m, acc[base + j + 1]);
  }
  constexpr int JL = J0 + 2 * ((N - 1 - J0) / 2);  // last j visited
  acc[base + JL + 2] = ptx::addc(acc[base + JL + 2], 0);
}

// r = a * b * R^-1 mod p, inputs < p (or < 2p with p having >= 2 spare bits), output < p
template <class P>
HD void mont_mul_raw(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  constexpr int N = P::N;
  static_assert(N % 2 == 0, "even limb count expected");
  uint32_t acc[2][2 * N + 3];
  uint32_t p[N];
#pragma unroll
  for (int k = 0; k < N; k++) p[k] = P::mod(k);
#pragma unroll
  for (int k = 0; k < 2 * N + 3; k++) { acc[0][k] = 0; acc[1][k] = 0; }

#pragma unroll
  for (int i = 0; i < N; i++) {
    uint32_t* X = acc[i & 1];        // chain starting at absolute position i
    uint32_t* Y = acc[(i & 1) ^ 1];  // chain starting at absolute position i+1
    const uint32_t bi = b[i];
    if (i > 0) {
      X[i] = ptx::add_cc(X[i], Y[i]);             // fold; carry goes into the Y chain
      mad_chain<N, 1, true>(Y, i, a, bi);         // odd limbs of a: positions i+1 .. i+N
    } else {
      mad_chain<N, 1, false>(Y, i, a, bi);
    }
    mad_chain<N, 0, false>(X, i, a, bi);          // even limbs of a: positions i .. i+N-1
    const uint32_t m = X[i] * P::INV;
    mad_chain<N, 0, false>(X, i, p, m);           // X[i] becomes 0
    mad_chain<N, 1, false>(Y, i, p, m);
  }
  // result words are positions N .. 2N-1 of E + O (value < 2p < 2^(32N): higher words cancel)
  uint32_t s[N];
  s[0] = ptx::add_cc(acc[0][N], acc[1][N]);
#pragma unroll
  for (int k = 1; k < N; k++) s[k] = ptx::addc_cc(acc[0][N + k], acc[1][N + k]);
  // conditional subtract
  uint32_t d[N];
  d[0] = ptx::sub_cc(s[0], p[0]);
#pragma unroll
  for (int k = 1; k < N; k++) d[k] = ptx::subc_cc(s[k], p[k]);
  const uint32_t borrow = ptx::subc(0, 0);  // 0xffffffff if s < p
#pragma unroll
  for (int k = 0; k < N; k++) r[k] = borrow ? s[k] : d[k];
}

// ---------------------------------------------------------------------------
// Wide (unreduced) products and a separate Montgomery reduction: the building blocks of the lazily reduced Fp2 product
// (Fp2::mul_lazy: 3 wide products + 2 reductions instead of 3 + 3).  Bit-exact against the fused product
// (tests/test_emulation.py::test_wide_arithmetic).
// ---------------------------------------------------------------------------

// t[0..2N) = a * b for ANY N-limb a, b (no reduction).  Same even/odd carry chains as mont_mul_raw without the m*p rows.
template <int N>
HD void wide_mul_raw(uint32_t* t, const uint32_t* a, const uint32_t* b) {
  uint32_t acc[2][2 * N + 3];
#pragma unroll
  for (int k = 0; k < 2 * N + 3; k++) { acc[0][k] = 0; acc[1][k] = 0; }
#pragma unroll
  for (int i = 0; i < N; i++) {
    mad_chain<N, 0, false>(acc[i & 1], i, a, b[i]);          // products starting at even+i positions
    mad_chain<N, 1, false>(acc[(i & 1) ^ 1], i, a, b[i]);
  }
  t[0] = ptx::add_cc(acc[0][0], acc[1][0]);
#pragma unroll
  for (int k = 1; k < 2 * N; k++) t[k] = ptx::addc_cc(acc[0][k], acc[1][k]);
  (void)ptx::addc(0, 0);
}

// r = T * R^-1 mod p for a 2N-limb T < p * R; output < p.  The m*p rows of mont_mul_raw on their own.
// Only the LOW half of T goes through the accumulators: T / R = T_hi + (T_lo + sum_i m_i p 2^(32 i)) / R, and T_hi is
// added after the rows.  mad_chain adds the carry out of a chain to the next word WITHOUT propagating further, which
// is sound only if that word holds nothing but earlier carries; with all of T preloaded (round 2's first version) the
// word was T[i + N] and a carry was lost whenever it was 0xffffffff - once in ~2^33 reductions, found by the verified
// 2^20 Groth16 proof (one G2 table point in 10^6; regression vectors in tests/test_emulation.py).
template <class P>
HD void mont_reduce_wide(uint32_t* r, const uint32_t* T) {
  constexpr int N = P::N;
  uint32_t acc[2][2 * N + 3];
  uint32_t p[N];
#pragma unroll
  for (int k = 0; k < N; k++) p[k] = P::mod(k);
#pragma unroll
  for (int k = 0; k < 2 * N + 3; k++) { acc[0][k] = k < N ? T[k] : 0; acc[1][k] = 0; }
#pragma unroll
  for (int i = 0; i < N; i++) {
    uint32_t* X = acc[i & 1];
    uint32_t* Y = acc[(i & 1) ^ 1];
    // m from the folded low word, computed before the fold so that no carry is live across plain code
    const uint32_t m = (X[i] + Y[i]) * P::INV;
    if (i > 0) {
      X[i] = ptx::add_cc(X[i], Y[i]);             // fold; the carry goes into the Y chain
      mad_chain<N, 1, true>(Y, i, p, m);
    } else {
      mad_chain<N, 1, false>(Y, i, p, m);
    }
    mad_chain<N, 0, false>(X, i, p, m);           // X[i] becomes 0
  }
  // (T_lo + sum m_i p 2^(32 i)) / R <= p, then + T_hi < p: the sum stays below 2p + 1 < 2^(32 N), no carry out
  uint32_t s[N];
  s[0] = ptx::add_cc(acc[0][N], acc[1][N]);
#pragma unroll
  for (int k = 1; k < N; k++) s[k] = ptx::addc_cc(acc[0][N + k], acc[1][N + k]);
  (void)ptx::addc(0, 0);
  s[0] = ptx::add_cc(s[0], T[N]);
#pragma unroll
  for (int k = 1; k < N; k++) s[k] = ptx::addc_cc(s[k], T[N + k]);
  (void)ptx::addc(0, 0);
  uint32_t d[N];
  d[0] = ptx::sub_cc(s[0], p[0]);
#pragma unroll
  for (int k = 1; k < N; k++) d[k] = ptx::subc_cc(s[k], p[k]);
  const uint32_t borrow = ptx::subc(0, 0);
#pragma unroll
  for (int k = 0; k < N; k++) r[k] = borrow ? s[k] : d[k];
}

// multi-limb helpers without reduction (K limbs)
template <int K>
HD void limbs_add(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  r[0] = ptx::add_cc(a[0], b[0]);
#pragma unroll
  for (int k = 1; k < K; k++) r[k] = ptx::addc_cc(a[k], b[k]);
  (void)ptx::addc(0, 0);
}
template <int K>
HD void limbs_sub(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  r[0] = ptx::sub_cc(a[0], b[0]);
#pragma unroll
  for (int k = 1; k < K; k++) r[k] = ptx::subc_cc(a[k], b[k]);
  (void)ptx::subc(0, 0);
}

template <class P>
HD void mod_add_raw(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  constexpr int N = P::N;
  uint32_t s[N], d[N];
  s[0] = ptx::add_cc(a[0], b[0]);
#pragma unroll
  for (int k = 1; k < N; k++) s[k] = ptx::addc_cc(a[k], b[k]);
  d[0] = ptx::sub_cc(s[0], P::mod(0));
#pragma unroll
  for (int k = 1; k < N; k++) d[k] = ptx::subc_cc(s[k], P::mod(k));
  const uint32_t borrow = ptx::subc(0, 0);
#pragma unroll
  for (int k = 0; k < N; k++) r[k] = borrow ? s[k] : d[k];
}

template <class P>
HD void mod_sub_raw(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  constexpr int N = P::N;
  uint32_t d[N];
  d[0] = ptx::sub_cc(a[0], b[0]);
#pragma unroll
  for (int k = 1; k < N; k++) d[k] = ptx::subc_cc(a[k], b[k]);
  const uint32_t borrow = ptx::subc(0, 0);  // all ones if a < b
  r[0] = ptx::add_cc(d[0], P::mod(0) & borrow);
#pragma unroll
  for (int k = 1; k < N; k++) r[k] = ptx::addc_cc(d[k], P::mod(k) & borrow);
}

// ---------------------------------------------------------------------------
// Fp<P>: value type
// ---------------------------------------------------------------------------
template <class P>
struct alignas(16) Fp {
  static constexpr int N = P::N;
  static constexpr int DEGREE = 1;
  using Params = P;
  using Base = Fp<P>;
  uint32_t l[N];

  HD static Fp zero() { Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.l[i] = 0; return r; }
  HD static Fp one() { Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.l[i] = P::r1(i); return r; }
  HD static Fp r2() { Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.l[i] = P::r2(i); return r; }

  HD bool is_zero() const { uint32_t t = 0;
#pragma unroll
    for (int i = 0; i < N; i++) t |= l[i]; return t == 0; }
  HD bool operator==(const Fp& o) const { uint32_t t = 0;
#pragma unroll
    for (int i = 0; i < N; i++) t |= (l[i] ^ o.l[i]); return t == 0; }
  HD bool operator!=(const Fp& o) const { return !(*this == o); }

  HD friend Fp operator+(const Fp& a, const Fp& b) { Fp r; mod_add_raw<P>(r.l, a.l, b.l); return r; }
  HD friend Fp operator-(const Fp& a, const Fp& b) { Fp r; mod_sub_raw<P>(r.l, a.l, b.l); return r; }
  // Fields of up to 8 limbs get the product inlined at every use; larger ones keep ONE copy of the unrolled product per
  // kernel (I-cache, compile time), called with operands and result in REGISTERS: a reference parameter makes the
  // caller spill both operands to its stack frame and the callee load them back.
  static constexpr int INLINE_LIMBS = 8;
#if defined(__CUDA_ARCH__)
  static __device__ __noinline__ Fp mul_ni(Fp a, Fp b) { Fp r; mont_mul_raw<P>(r.l, a.l, b.l); return r; }
  HD friend Fp operator*(const Fp& a, const Fp& b) {
    if (N > INLINE_LIMBS) return mul_ni(a, b);
    Fp r; mont_mul_raw<P>(r.l, a.l, b.l); return r;
  }
#else
  HD friend Fp operator*(const Fp& a, const Fp& b) { Fp r; mont_mul_raw<P>(r.l, a.l, b.l); return r; }
#endif
  HD Fp sqr() const { return (*this) * (*this); }
  HD Fp neg() const { return is_zero() ? *this : (zero() - *this); }
  HD Fp dbl() const { return *this + *this; }
  // Montgomery -> canonical (multiply by 1) and back
  HD Fp from_mont() const { Fp o = zero(); o.l[0] = 1; return (*this) * o; }
  HD Fp to_mont() const { return (*this) * r2(); }

  // a^(p-2) (only used a handful of times per MSM / for batch inversion seeds)
  HD Fp inverse() const {
    Fp result = one();
    Fp base = *this;
    for (int w = 0; w < N; w++) {
      uint32_t e = P::pm2(w);
      // constant-time-ish square and multiply, LSB first
      for (int bit = 0; bit < 32; bit++) {
        if ((e >> bit) & 1) result = result * base;
        base = base.sqr();
      }
    }
    return result;
  }
  // multiply by a small unsigned constant via additions
  HD Fp mul_small(unsigned k) const {
    Fp acc = zero();
    Fp cur = *this;
    while (k) {
      if (k & 1) acc = acc + cur;
      cur = cur.dbl();
      k >>= 1;
    }
    return acc;
  }
};

// runtime-index pm2 lookup needs a real array on device; provide via switch-free table
// (P::pm2(w) with runtime w compiles to a local constant array; fine for the rare inverse)

// ---------------------------------------------------------------------------
// Fp2<F, BETA>: F[u]/(u^2 + BETA), i.e. u^2 = -BETA  (BETA = 1: BN254, BLS12-381; 5: BLS12-377)
// rule restated from std/algebra/emulated/fields_bn254/e2.go:203-213 and
// std/algebra/native/fields_bls12377/e2.go:134.  Memory = gnark E2{A0, A1}.
// ---------------------------------------------------------------------------
// Fp2 product / square: out of line (one copy of the 3-multiplication body per kernel), operands by value on the device
template <class T> struct is_device_fp { static constexpr bool value = false; };
template <class P> struct is_device_fp<Fp<P>> { static constexpr bool value = true; };

template <class F, unsigned BETA>
struct alignas(16) Fp2 {
  static constexpr int DEGREE = 2;
  static constexpr unsigned BETA_VALUE = BETA;
  using Base = F;
  F a0, a1;
  HD static Fp2 zero() { Fp2 r; r.a0 = F::zero(); r.a1 = F::zero(); return r; }
  HD static Fp2 one() { Fp2 r; r.a0 = F::one(); r.a1 = F::zero(); return r; }
  HD bool is_zero() const { return a0.is_zero() && a1.is_zero(); }
  HD bool operator==(const Fp2& o) const { return a0 == o.a0 && a1 == o.a1; }
  HD bool operator!=(const Fp2& o) const { return !(*this == o); }
  HD friend Fp2 operator+(const Fp2& x, const Fp2& y) { Fp2 r; r.a0 = x.a0 + y.a0; r.a1 = x.a1 + y.a1; return r; }
  HD friend Fp2 operator-(const Fp2& x, const Fp2& y) { Fp2 r; r.a0 = x.a0 - y.a0; r.a1 = x.a1 - y.a1; return r; }
  HD static F mul_beta(const F& t) { return BETA == 1 ? t : t.mul_small(BETA); }
  // not inlined on device: one copy of the 3-multiplication body per kernel
  // Karatsuba on UNREDUCED double-width products: 3 wide products and 2 Montgomery reductions instead of 3 of each.
  //   c1 = (a0+a1)(b0+b1) - a0b0 - a1b1   (>= 0, < 2p^2)
  //   c0 = a0b0 + BETA (p^2 - a1b1)       (>= 0, < (1+BETA) p^2 < pR for every modulus here)
  template <class FF = F>
  HD static Fp2 mul_lazy(const Fp2& x, const Fp2& y) {
    constexpr int N = FF::N;
    using P = typename FF::Params;
    uint32_t t0[2 * N], t1[2 * N], t2[2 * N], sa[N], sb[N];
    wide_mul_raw<N>(t0, x.a0.l, y.a0.l);
    wide_mul_raw<N>(t1, x.a1.l, y.a1.l);
    limbs_add<N>(sa, x.a0.l, x.a1.l);           // < 2p: fits N limbs (top bit of p clear)
    limbs_add<N>(sb, y.a0.l, y.a1.l);
    wide_mul_raw<N>(t2, sa, sb);
    limbs_sub<2 * N>(t2, t2, t0);
    limbs_sub<2 * N>(t2, t2, t1);
    uint32_t q[2 * N];
#pragma unroll
    for (int k = 0; k < 2 * N; k++) q[k] = P::psq(k);
    limbs_sub<2 * N>(q, q, t1);                 // p^2 - a1 b1
#pragma unroll
    for (unsigned k = 0; k < BETA; k++) limbs_add<2 * N>(t0, t0, q);
    Fp2 r;
    mont_reduce_wide<P>(r.a0.l, t0);
    mont_reduce_wide<P>(r.a1.l, t2);
    return r;
  }
  HDNI static Fp2 mul(Fp2 x, Fp2 y) {        // by value: operands travel in registers (see Fp::mul_ni)
    if constexpr (is_device_fp<F>::value) return mul_lazy<F>(x, y);
    // generic base field (host-side 64-bit limbs): Karatsuba, 3 base multiplications
    F v0 = x.a0 * y.a0;
    F v1 = x.a1 * y.a1;
    F s = (x.a0 + x.a1) * (y.a0 + y.a1);
    Fp2 r;
    r.a0 = v0 - mul_beta(v1);
    r.a1 = s - v0 - v1;
    return r;
  }
  HD friend Fp2 operator*(const Fp2& x, const Fp2& y) { return mul(x, y); }
  HDNI static Fp2 sqr_ni(Fp2 x) {
    if (BETA == 1) {  // (a0+a1)(a0-a1), 2 a0 a1
      Fp2 r;
      F t = x.a0 * x.a1;
      r.a0 = (x.a0 + x.a1) * (x.a0 - x.a1);
      r.a1 = t + t;
      return r;
    }
    return mul(x, x);
  }
  HD Fp2 sqr() const { return sqr_ni(*this); }
  HD Fp2 neg() const { Fp2 r; r.a0 = a0.neg(); r.a1 = a1.neg(); return r; }
  HD Fp2 dbl() const { Fp2 r; r.a0 = a0.dbl(); r.a1 = a1.dbl(); return r; }
  HD Fp2 inverse() const {
    F n = a0.sqr() + mul_beta(a1.sqr());
    F ni = n.inverse();
    Fp2 r; r.a0 = a0 * ni; r.a1 = (a1 * ni).neg();
    return r;
  }
};

// concrete fields
using bn254_fp = Fp<bn254_fp_params>;
using bn254_fr = Fp<bn254_fr_params>;
using bls12_381_fp = Fp<bls12_381_fp_params>;
using bls12_381_fr = Fp<bls12_381_fr_params>;
using bls12_377_fp = Fp<bls12_377_fp_params>;
using bls12_377_fr = Fp<bls12_377_fr_params>;
using bw6_761_fp = Fp<bw6_761_fp_params>;
using bw6_761_fr = Fp<bw6_761_fr_params>;
using bn254_fp2 = Fp2<bn254_fp, 1>;
using bls12_381_fp2 = Fp2<bls12_381_fp, 1>;
using bls12_377_fp2 = Fp2<bls12_377_fp, 5>;

}  // namespace gb200
