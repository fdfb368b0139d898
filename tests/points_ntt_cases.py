"""Inputs and independent answers for the group-element NTT tests (test_points_ntt_emulation.py on the CPU,
test_gpu_points_ntt.py on the device).

Known discrete logs: the points P_k = d_k * B go in, and the answer is (iNTT(d))_i * B for the inverse transform,
NTT(d)_k * B for the forward one, with the Fr transform of the C++ oracle (corelib.ntt, itself pinned by
tests/test_golden_kzg.py); the points come from the big-int oracle or, on the device, from b200_fixed_base_batch.

The Ethereum ceremony (tests/golden/eth_kzg_srs_v1.bin, tau unknown, both bases computed by somebody else): for
m = 2^s <= 4096 the inverse m-point transform of monomial[(4096/m) k], k < m, is [L_j^(m)(tau^(4096/m))] G =
sum_{t < 4096/m} lagrange[j + m t], and the forward transform maps those sums back."""
import random

import numpy as np

from oracle import corelib, ec, ff, kzg_srs, ntt
from oracle.params import BLS12_381

FAMILIES = ("random", "constant", "zero", "single", "ramp", "r_minus_1")


def dlogs(curve, family, n, seed):
    """discrete logs d_k, k < n, of one input family"""
    rng = random.Random(f"pntt/{curve.name}/{family}/{n}/{seed}")
    r = curve.r
    if family == "random":
        return [rng.randrange(r) for _ in range(n)]
    if family == "constant":          # every output but one is infinity: P + (-P) in the additions
        return [rng.randrange(1, r)] * n
    if family == "zero":              # every input is the point at infinity
        return [0] * n
    if family == "single":
        d = [0] * n
        d[rng.randrange(n)] = rng.randrange(1, r)
        return d
    if family == "ramp":              # d_k = k
        return list(range(n))
    if family == "r_minus_1":         # -B at every even k, random at odd k
        return [r - 1 if k % 2 == 0 else rng.randrange(r) for k in range(n)]
    raise ValueError(family)


def bitrev_perm(logn):
    return np.array([ntt.bitrev(i, logn) for i in range(1 << logn)], dtype=np.int64)


def fr_transform(curve, K, logn, inverse):
    """natural-order NTT (inverse: with 1/n) of the Montgomery limb array K, as a new array: the C++ oracle's DIF,
    whose output position j holds element bitrev(j)"""
    A = np.ascontiguousarray(K, dtype=np.uint64).copy()
    if logn == 0:
        return A
    corelib.ntt(curve, A, logn, inverse, ntt.DIF, False)
    return np.ascontiguousarray(A[bitrev_perm(logn)])


def scalar_mul_points(curve, base, K):
    """[k_i * base] as packed affine points by the big-int oracle (small n); K: Montgomery limb array"""
    F = ff.base_field(curve, 1)
    return ec.pack_points(curve, 1, [ec.scalar_mul(F, k, base) for k in ff.unpack_elements(K, curve.r, curve.fr_limbs)])


def known_dlog_cases(curve, base, family, logn, points, seed=0):
    """(input points, {inverse: expected output}) of both transforms of one input, all packed affine"""
    K = ff.pack_elements(dlogs(curve, family, 1 << logn, seed), curve.r, curve.fr_limbs)
    return points(curve, base, K), {inv: points(curve, base, fr_transform(curve, K, logn, inv)) for inv in (True, False)}


def ceremony():
    """(monomial, lagrange sums by m): sums[m][j] = sum_{t < 4096/m} lagrange[j + m t], as affine points, m = 1..4096"""
    mono, lag, _ = kzg_srs.load()
    F = ff.Fp(BLS12_381.p)
    sums = {kzg_srs.N: list(lag)}
    m = kzg_srs.N
    while m > 1:
        prev = sums[m]
        m //= 2
        sums[m] = [ec.affine_add(F, prev[j], prev[j + m]) for j in range(m)]
    return mono, sums


def ceremony_case(mono, sums, m):
    """packed (monomial[(4096/m) k], k < m) and packed Lagrange sums of the m-point transform"""
    step = kzg_srs.N // m
    return (ec.pack_points(BLS12_381, 1, [mono[step * k] for k in range(m)]),
            ec.pack_points(BLS12_381, 1, sums[m]))
