"""The PLONK device entry points on all four curves, at the block, grid and recursion edges of their kernels,
element by element and limb for limb against the big-int oracle (oracle/plonk.py, oracle/ntt.py); then the whole
prover (b200_plonk_prove and gnark_b200/plonk.py) on BLS12-377 and BW6-761 against the oracle prover.

Edges (gnark_b200/csrc/plonk.cuh, inst.cuh):
  * k_plonk_constraints: 128-thread blocks; the L1 denominators are cached in the domain handle per coset
  * k_plonk_zh_scale, k_plonk_add_bsb22, k_vec_op, k_axpy, k_scale_powers, k_bit_reverse: 256-thread blocks
  * k_batch_invert: 32-element chunks, 128 chunks (4096 elements) per block
  * k_scan_block / k_scan_fix: 1024 elements per block, recursive over the block totals (a second level past 2^20)
  * k_poly_eval_partial: 2048 coefficients per block; k_sum_reduce strides over the partial sums 256 at a time

Every result is compared with the packed reference, so a value left unreduced (>= r) fails as well as a wrong one.
BW6-761 has no recalled G1 generator (CURVES["bw6-761"].g1 is None): the prover tests take their SRS base from
util.pick_base and assert it is a real point, else every digest would be the point at infinity."""
import itertools
import random

import numpy as np
import pytest
import torch

from oracle import corelib, ec, ff, ntt, plonk
from oracle import plonk_prover as pp
from oracle.params import CURVES
from util import jac_to_affine, pick_base

pytestmark = pytest.mark.gpu
ALL = list(CURVES.values())
BIG = [CURVES["bn254"], CURVES["bw6-761"]]
NAME = lambda c: c.name


def pe(c, v):
    return ff.pack_elements(v, c.r, c.fr_limbs)


def dev(arr):
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.int64)).cuda()


def fetch(gpu, c, t):
    gpu.sync(0)
    return t.cpu().numpy().view(np.uint64).reshape(-1, c.fr_limbs)


def assert_elements(c, got, want, what):
    exp = pe(c, want)
    got = np.asarray(got, dtype=np.uint64).reshape(-1, c.fr_limbs)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    bad = np.nonzero((got != exp).any(axis=1))[0]
    if bad.size:
        i = int(bad[0])
        raise AssertionError(f"{c.name} {what}: {bad.size} of {len(want)} elements differ, first at {i}: "
                             f"got limbs {[hex(x) for x in got[i]]}, want {want[i]:#x}")


def edge_vector(rng, r, n, lo=0):
    """random elements of [lo, r), with 0 (if lo == 0), 1 and r - 1 at both ends and around 256"""
    v = [rng.randrange(lo, r) for _ in range(n)]
    edges = [x for x in (0, 1, r - 1) if x >= lo]
    for k, i in enumerate(sorted({0, 1, 2, 254, 255, 256, 257, n - 3, n - 2, n - 1} & set(range(n)))):
        v[i] = edges[(k + rng.randrange(3)) % len(edges)]
    return v


# ---- the quotient: constraints per coset, divideByZH, BSB22 gates ----------------------------------------------

def coset_values(c, dom0, lagrange, coset):
    """values on coset * <w> (natural order) of the polynomial given in Lagrange form on <w>, through the oracle's
    NTT (plonk.coset_values evaluates point by point, O(n^2))"""
    coeffs = ntt.bit_reverse(dom0.fft_inverse(lagrange, ntt.DIF))
    return ntt.bit_reverse(ntt.Domain(c, dom0.n, coset_gen=coset).fft(coeffs, ntt.DIF, on_coset=True))


def numerator_from_values(c, n, rho, vals, alpha, beta, gamma, blind):
    """plonk.numerator with the coset values given (vals[i][name], coset i): plonk.all_constraints per point"""
    r = c.r
    dom0, dom1 = ntt.Domain(c, n), ntt.Domain(c, rho * n)
    g, w4, w = dom1.coset_gen, dom1.generator, dom0.generator
    logm = (rho * n).bit_length() - 1
    cres = [0] * (rho * n)
    for i, u in enumerate(vals):
        coset = g * pow(w4, i, r) % r
        xn1 = (pow(coset, n, r) - 1) % r
        xs = [coset]
        for _ in range(n - 1):
            xs.append(xs[-1] * w % r)
        for j in range(n):
            pt = {k: u[k][j] for k in plonk.POLYS}
            pt["zs"] = u["z"][(j + 1) % n]
            cres[ntt.bitrev(rho * j + i, logm)] = plonk.all_constraints(
                r, n, dom0.cardinality_inv, pt, xs[j], xs[(j + 1) % n], alpha, beta, gamma, g, blind, xn1)
    return cres


# blinding coefficients of L, R, O, Z per size: 0 to 3 each, Z unblinded at log n = 7
BLIND_COUNTS = {6: (2, 2, 2, 3), 7: (0, 1, 3, 0), 8: (3, 0, 1, 2), 10: (1, 3, 2, 1)}


@pytest.mark.parametrize("logn", sorted(BLIND_COUNTS))     # below one 128-thread block, one, two, eight
@pytest.mark.parametrize("c", ALL, ids=NAME)
def test_constraints_then_divide_by_zh(gpu, c, logn):
    """plonk_constraints_coset on the four cosets against plonk.numerator, once with a fresh domain handle per coset
    and once through one handle whose cached L1 denominators must follow the coset; then plonk_divide_by_zh against
    plonk.divide_by_zh"""
    r, L, n, rho = c.r, c.fr_limbs, 1 << logn, 4
    rng = random.Random(7000 + 10 * logn + c.curve_id)
    dom0, dom1 = ntt.Domain(c, n), ntt.Domain(c, rho * n)
    g, w4 = dom1.coset_gen, dom1.generator
    polys = {k: [rng.randrange(r) for _ in range(n)] for k in plonk.POLYS}
    alpha, beta, gamma = (rng.randrange(r) for _ in range(3))
    blind = {k: [rng.randrange(r) for _ in range(m)] for k, m in zip("lroz", BLIND_COUNTS[logn])}
    vals = [{k: coset_values(c, dom0, polys[k], g * pow(w4, i, r) % r) for k in plonk.POLYS} for i in range(rho)]
    want = numerator_from_values(c, n, rho, vals, alpha, beta, gamma, blind)
    if logn <= 8:
        assert want == plonk.numerator(c, n, rho, polys, alpha, beta, gamma, blind)

    d_vals = [{k: dev(pe(c, u[k])) for k in plonk.POLYS} for u in vals]
    h_blind = {k: pe(c, v) for k, v in blind.items()}
    consts = [pe(c, [x]) for x in (g, w4, alpha, beta, gamma)]

    def constraints(d0, i, out):
        gpu.plonk_constraints_coset(d0, consts[0], consts[1], d_vals[i], consts[2], consts[3], consts[4], h_blind,
                                    i, rho, out)

    fresh = torch.zeros(rho * n * L, dtype=torch.int64, device="cuda")
    for i in range(rho):
        d0 = gpu.Domain(c.curve_id, logn)
        constraints(d0, i, fresh)
        gpu.sync(0)
        d0.free()
    assert_elements(c, fetch(gpu, c, fresh), want, f"constraints, log n {logn}, a fresh handle per coset")
    reused = torch.zeros_like(fresh)
    d0 = gpu.Domain(c.curve_id, logn)
    for i in range(rho):
        constraints(d0, i, reused)
    assert np.array_equal(fetch(gpu, c, reused), fetch(gpu, c, fresh)), "one handle for all cosets"
    d0.free()

    d1 = gpu.Domain(c.curve_id, logn + 2)
    gpu.plonk_divide_by_zh(d1, logn, reused)
    assert_elements(c, fetch(gpu, c, reused), plonk.divide_by_zh(c, n, rho, want), f"divide_by_zh, log n {logn}")
    d1.free()


@pytest.mark.parametrize("log_rho", (1, 2, 3))
@pytest.mark.parametrize("c", ALL, ids=NAME)
def test_divide_by_zh_ratios(gpu, c, log_rho):
    """plonk_divide_by_zh at rho = 2, 4, 8 over rho * 256 points (two to eight 256-thread blocks)"""
    logn, rho = 8, 1 << log_rho
    n = 1 << logn
    rng = random.Random(7100 + log_rho)
    cres = edge_vector(rng, c.r, rho * n)
    d = dev(pe(c, cres))
    d1 = gpu.Domain(c.curve_id, logn + log_rho)
    gpu.plonk_divide_by_zh(d1, logn, d)
    assert_elements(c, fetch(gpu, c, d), plonk.divide_by_zh(c, n, rho, cres), f"divide_by_zh, rho {rho}")
    d1.free()


@pytest.mark.parametrize("logn", (6, 9))
@pytest.mark.parametrize("c", ALL, ids=NAME)
def test_bsb22_coset(gpu, c, logn):
    """plonk_bsb22_coset: out[bitrev_{rho n}(rho j + i)] += qcp[j] * pi2[j] on coset i, on top of a prefilled out"""
    r, n, rho = c.r, 1 << logn, 4
    logm = logn + 2
    rng = random.Random(7200 + logn)
    want = edge_vector(rng, r, rho * n)
    out = dev(pe(c, want))
    d0 = gpu.Domain(c.curve_id, logn)
    for i in range(rho):
        qcp = [rng.randrange(r) if rng.random() < 0.5 else rng.choice((0, 1, r - 1)) for _ in range(n)]
        pi2 = edge_vector(rng, r, n)
        gpu.plonk_bsb22_coset(d0, dev(pe(c, qcp)), dev(pe(c, pi2)), i, rho, out)
        for j in range(n):
            k = ntt.bitrev(rho * j + i, logm)
            want[k] = (want[k] + qcp[j] * pi2[j]) % r
        assert_elements(c, fetch(gpu, c, out), want, f"bsb22, log n {logn}, coset {i}")
    d0.free()


# ---- element-wise vector kernels ------------------------------------------------------------------------------

VEC_SIZES = (1, 255, 256, 257, 5000)


@pytest.mark.parametrize("c", ALL, ids=NAME)
def test_vec_axpy(gpu, c):
    r = c.r
    rng = random.Random(7300)
    for n in VEC_SIZES:
        x, y = edge_vector(rng, r, n), edge_vector(rng, r, n)
        dx = dev(pe(c, x))
        for a in (0, 1, r - 1, rng.randrange(r)):
            dy = dev(pe(c, y))
            gpu.vec_axpy(0, c.curve_id, dy, pe(c, [a]), dx, n)
            assert_elements(c, fetch(gpu, c, dy), [(v + a * u) % r for u, v in zip(x, y)], f"axpy n {n} a {a:#x}")


@pytest.mark.parametrize("c", ALL, ids=NAME)
def test_vec_op(gpu, c):
    """mul / add / sub into a separate vector and into a (out aliasing a); every pair of 0, 1, r - 1 is among the
    operands at the front, at the 256-thread block edge and at the back"""
    r = c.r
    rng = random.Random(7400)
    pairs = list(itertools.product((r - 1, 1, 0), repeat=2))
    ops = ((gpu.VEC_MUL, lambda x, y: x * y % r), (gpu.VEC_ADD, lambda x, y: (x + y) % r),
           (gpu.VEC_SUB, lambda x, y: (x - y) % r))
    for n in VEC_SIZES:
        a, b = [rng.randrange(r) for _ in range(n)], [rng.randrange(r) for _ in range(n)]
        for k, i in enumerate(sorted(set(range(9)) | set(range(250, 263)) | set(range(n - 9, n)))):
            if 0 <= i < n:
                a[i], b[i] = pairs[k % 9]
        db = dev(pe(c, b))
        for op, f in ops:
            want = [f(x, y) for x, y in zip(a, b)]
            da, out = dev(pe(c, a)), torch.zeros(n * c.fr_limbs, dtype=torch.int64, device="cuda")
            gpu.vec_op(0, c.curve_id, op, out, da, db, n)
            assert_elements(c, fetch(gpu, c, out), want, f"vec_op {op} n {n}")
            gpu.vec_op(0, c.curve_id, op, da, da, db, n)
            assert_elements(c, fetch(gpu, c, da), want, f"vec_op {op} n {n}, out aliasing a")


@pytest.mark.parametrize("n", (1, 31, 32, 33, 4095, 4096, 4097, 10000))
@pytest.mark.parametrize("c", ALL, ids=NAME)
def test_vec_batch_invert(gpu, c, n):
    """32-element chunks, 128 chunks per block; zeros stay zero, at chunk starts (32, 4096), chunk ends (31, 4095)
    and over the whole chunk 64..95.  The self-inverse 1 and r - 1 sit inside a chunk, never at its end."""
    r = c.r
    rng = random.Random(7500 + n)
    v = [rng.randrange(2, r - 1) for _ in range(n)]
    for i, x in ((5, 1), (6, r - 1), (31, 0), (32, 0), (4095, 0), (4096, 0)) + tuple((i, 0) for i in range(64, 96)):
        if i < n:
            v[i] = x
    d = dev(pe(c, v))
    gpu.vec_batch_invert(0, c.curve_id, d, n)
    assert_elements(c, fetch(gpu, c, d), [pow(x, -1, r) if x else 0 for x in v], f"batch_invert n {n}")


@pytest.mark.parametrize("c", ALL, ids=NAME)
def test_vec_bit_reverse_and_scale_powers(gpu, c):
    r = c.r
    rng = random.Random(7600)
    for logn in (1, 8, 13):
        v = [rng.randrange(r) for _ in range(1 << logn)]
        d = dev(pe(c, v))
        gpu.vec_bit_reverse(0, c.curve_id, d, logn)
        assert_elements(c, fetch(gpu, c, d), ntt.bit_reverse(v), f"bit_reverse log n {logn}")
    for n in (1, 255, 256, 257, 1000):
        v = edge_vector(rng, r, n)
        s, g = rng.randrange(r), rng.randrange(r)
        d = dev(pe(c, v))
        gpu.vec_scale_powers(0, c.curve_id, d, n, pe(c, [s]), pe(c, [g]))
        assert_elements(c, fetch(gpu, c, d), [x * s % r * pow(g, i, r) % r for i, x in enumerate(v)],
                        f"scale_powers n {n}")


# ---- the permutation grand product, scans, evaluation and division by (X - z) ---------------------------------

@pytest.mark.parametrize("logn", (7, 10, 11, 12))          # one, one, two and four 1024-element scan blocks
@pytest.mark.parametrize("c", ALL, ids=NAME)
def test_build_z(gpu, c, logn):
    """plonk_build_z against plonk.build_ratio_copy_constraint on a satisfied trace, whose last ratio brings the
    product back to one"""
    r, n = c.r, 1 << logn
    rng = random.Random(7700 + logn)
    circ, l, rr, o = pp.random_satisfied_instance(c, n, seed=7700 + logn)
    beta, gamma = rng.randrange(r), rng.randrange(r)
    dom0 = ntt.Domain(c, n)
    want = plonk.build_ratio_copy_constraint(c, dom0, l, rr, o, circ.perm, beta, gamma)
    d0 = gpu.Domain(c.curve_id, logn)
    dz = torch.zeros(n * c.fr_limbs, dtype=torch.int64, device="cuda")
    gpu.plonk_build_z(d0, dev(pe(c, l)), dev(pe(c, rr)), dev(pe(c, o)), torch.tensor(circ.perm, dtype=torch.int64,
                      device="cuda"), pe(c, [beta]), pe(c, [gamma]), dz)
    got = fetch(gpu, c, dz)
    d0.free()
    assert_elements(c, got, want, f"build_z log n {logn}")
    supp = plonk.support_permutation(c, dom0)
    num = den = 1
    for j, f in enumerate((l, rr, o)):
        num = num * ((f[n - 1] + beta * supp[j * n + n - 1] + gamma) % r) % r
        den = den * ((f[n - 1] + beta * supp[circ.perm[j * n + n - 1]] + gamma) % r) % r
    assert want[n - 1] * num % r * pow(den, -1, r) % r == 1


def scan_ref(r, v, op, exclusive):
    f = (lambda a, b: a * b % r) if op == "product" else (lambda a, b: (a + b) % r)
    acc, out = 1 if op == "product" else 0, []
    for x in v:
        if exclusive:
            out.append(acc)
        acc = f(acc, x)
        if not exclusive:
            out.append(acc)
    return out


def check_scan(gpu, c, v, op, exclusive):
    d = dev(pe(c, v))
    gpu.vec_scan(0, c.curve_id, gpu.SCAN_PRODUCT if op == "product" else gpu.SCAN_SUM, d, len(v), exclusive=exclusive)
    assert_elements(c, fetch(gpu, c, d), scan_ref(c.r, v, op, exclusive),
                    f"{'exclusive' if exclusive else 'inclusive'} {op} scan, n {len(v)}")


@pytest.mark.parametrize("n", (1023, 1024, 1025, 2047, 2048, 2049))
@pytest.mark.parametrize("c", ALL, ids=NAME)
def test_scans_eval_division(gpu, c, n):
    """1024 elements per scan block, 2048 coefficients per evaluation block; z = 0, 1, a 2048-th root of unity and a
    random point"""
    r = c.r
    rng = random.Random(7800 + n)
    for op in ("product", "sum"):
        v = edge_vector(rng, r, n, lo=1 if op == "product" else 0)
        for exclusive in (False, True):
            check_scan(gpu, c, v, op, exclusive)
    coeffs = edge_vector(rng, r, n)
    for z in (0, 1, ntt.Domain(c, 2048).generator, rng.randrange(r)):
        got = gpu.poly_eval(0, c.curve_id, dev(pe(c, coeffs)), n, pe(c, [z]))
        assert_elements(c, got, [ntt.poly_eval(r, coeffs, z)], f"poly_eval n {n} z {z:#x}")
        d = dev(pe(c, coeffs))
        rem = gpu.poly_div_by_linear(0, c.curve_id, d, n, pe(c, [z]))
        q, want_rem = plonk.div_by_linear(r, coeffs, z)
        assert_elements(c, rem, [want_rem], f"poly_div_by_linear remainder n {n} z {z:#x}")
        assert_elements(c, fetch(gpu, c, d), q + [0], f"poly_div_by_linear quotient n {n} z {z:#x}")


@pytest.mark.parametrize("c", BIG, ids=NAME)
def test_large_scans_and_eval(gpu, c):
    """a sum and a product scan of 2^20 + 5 elements (1025 block totals: a second recursion level) and an evaluation
    of 2^19 + 3 coefficients (257 partial sums: k_sum_reduce takes a second stride)"""
    r = c.r
    rng = random.Random(7900)
    n = (1 << 20) + 5
    check_scan(gpu, c, [rng.randrange(r) for _ in range(n)], "sum", False)
    check_scan(gpu, c, [rng.randrange(1, r) for _ in range(n)], "product", True)
    m = (1 << 19) + 3
    coeffs = [rng.randrange(r) for _ in range(m)]
    x = rng.randrange(r)
    got = gpu.poly_eval(0, c.curve_id, dev(pe(c, coeffs)), m, pe(c, [x]))
    assert_elements(c, got, [ntt.poly_eval(r, coeffs, x)], f"poly_eval n {m}")


# ---- the prover on BLS12-377 and BW6-761 ----------------------------------------------------------------------

@pytest.mark.parametrize("logn,n_commit", [(4, 0), (6, 0), (5, 1)])
@pytest.mark.parametrize("c", [CURVES["bls12-377"], CURVES["bw6-761"]], ids=NAME)
def test_prover_vs_oracle(gpu, c, logn, n_commit):
    """b200_plonk_prove (gpu.PlonkKey) and the Python orchestrator (gnark_b200/plonk.py) against the big-int oracle
    prover with the same injected challenges and blinding: the ten digests (and [PI2] of a BSB22 gate) as
    dlog * base over a trapdoor SRS, and the opened values.  The oracle proof passes the verifier's equations in the
    exponent (no pairing on these curves in the oracle)."""
    from gnark_b200 import plonk as b200_plonk
    r, n = c.r, 1 << logn
    F, base = pick_base(c, 1)
    assert base is not None and ec.scalar_mul(F, c.r, base) is None
    rng = random.Random(8000 + 10 * logn + n_commit)
    inst = pp.random_satisfied_instance(c, n, seed=8000 + logn, n_commit=n_commit)
    circ, l, rr, o = inst[:4]
    pi2 = inst[4] if n_commit else []
    rnd = lambda: rng.randrange(r)
    ch = pp.Challenges(gamma=rnd(), beta=rnd(), alpha=rnd(), zeta=rnd(), v=rnd(), bl=[rnd(), rnd()], br=[rnd(), rnd()],
                       bo=[rnd(), rnd()], bz=[rnd(), rnd(), rnd()])
    tau = rnd()
    want = pp.prove(c, circ, l, rr, o, ch, tau, pi2=pi2)
    assert pp.verify(c, circ, want, ch, tau)
    P = lambda v: pe(c, v)
    srs = corelib.fixed_base(c, 1, ec.pack_points(c, 1, [base]), P([pow(tau, i, r) for i in range(n + 3)]))
    want_pts = [want.L, want.R, want.O, want.Z, *want.H, want.lin, want.batch_opening, want.z_opening] + want.bsb22
    names = ["L", "R", "O", "Z", "H1", "H2", "H3", "lin", "batch", "zopen"] + [f"bsb22_{j}" for j in range(n_commit)]
    assert all(d != 0 for d in want_pts)

    def check(path, pts, claimed, zu):
        for name, p_, d in zip(names, pts, want_pts):
            assert jac_to_affine(c, 1, p_) == ec.scalar_mul(F, d, base), (path, name)
        assert claimed == want.claimed and zu == want.zu, path

    key = gpu.PlonkKey(c.curve_id, logn, P(circ.ql), P(circ.qr), P(circ.qm), P(circ.qo), P(circ.qk),
                       np.array(circ.perm, dtype=np.int64), srs, qcp=[P(v) for v in circ.qcp])
    res = key.prove(P(l), P(rr), P(o), P([ch.gamma]), P([ch.beta]), P([ch.alpha]), P([ch.zeta]), P([ch.v]),
                    P(ch.bl), P(ch.br), P(ch.bo), P(ch.bz), pi2=[P(v) for v in pi2])
    key.free()
    vals = ff.unpack_elements(res[1], r, c.fr_limbs)
    check("b200_plonk_prove", list(res[0]) + (list(res[2]) if n_commit else []), vals[:6] + vals[7:], vals[6])

    pk = b200_plonk.ProvingKey.from_trace(c.curve_id, logn, P(circ.ql), P(circ.qr), P(circ.qm), P(circ.qo),
                                         P(circ.qk), np.array(circ.perm, dtype=np.int64), srs,
                                         qcp=[P(v) for v in circ.qcp])
    got = b200_plonk.Prove(pk, P(l), P(rr), P(o),
                           b200_plonk.Challenges(gamma=ch.gamma, beta=ch.beta, alpha=ch.alpha, zeta=ch.zeta, v=ch.v,
                                                 bl=ch.bl, br=ch.br, bo=ch.bo, bz=ch.bz), pi2=[P(v) for v in pi2])
    pk.free()
    check("gnark_b200.plonk", [*got.LRO, got.Z, *got.H, got.LinearizedDigest, got.BatchedProofH, got.ZShiftedOpeningH,
                               *got.Bsb22Commitments[:n_commit]], got.BatchedClaimedValues, got.ZShiftedClaimedValue)
