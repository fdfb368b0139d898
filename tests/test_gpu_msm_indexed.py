"""b200_msm_indexed on the device: sum_j s_j * bases[idx[j]], the bases picked from a table by index.

Known discrete logs (bases P_i = k_i B from the fixed-base batch, a sample checked against the big-int oracle by
test_gpu_msm_plans.build_bases): the expected sum is (sum_j k_{idx[j]} s_j mod r) B, on every curve and group, plain and
precomputed tables, for index lists with repeats, with both ends of the table, with one index only and for a full
permutation, and at index counts on both sides of every size where the window of a plain table changes.  Also: the
BSB22 hint's shape (a handful of indices into a 2^20-point table), equality with b200_msm over the dense vector, every
host/device placement, the Ethereum ceremony's Lagrange basis as a commitment key, plonk.bsb22_commitment against the
oracle prover and against the device prover's [PI2_j], and the argument errors."""
import ctypes
import random

import numpy as np
import pytest

from msm_families import pack, seeded
from oracle import corelib, ec, ff, kzg_srs, ntt
from oracle.params import BLS12_381, BN254
from points_ntt_cases import fr_transform
from test_gpu_msm_plans import BY_NAME, PAIR_IDS, default_window, expected, make_table
from util import jac_to_affine

pytestmark = pytest.mark.gpu
N_TABLE = 3000


def to_dev(a, dtype=np.int64):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a).view(dtype).copy()).cuda()
    torch.cuda.synchronize()
    return t


def index_sets(T, rng):
    return {
        "random_repeats": np.array([rng.randrange(T) for _ in range(1500)], dtype=np.uint32),
        "ends": np.array([T - 1, 0] + [rng.randrange(T) for _ in range(300)] + [0, T - 1], dtype=np.uint32),
        "one_index": np.full(700, rng.randrange(T), dtype=np.uint32),
        "permutation": np.array(rng.sample(range(T), T), dtype=np.uint32),
    }


def check_indexed(t, curve, group, ks, idx, sc, what):
    got = jac_to_affine(curve, group, t.msm_indexed(idx, sc))
    assert got == expected(curve, group, np.ascontiguousarray(ks[idx]), sc), what
    return got


def canonical_affine(gpu, curve, group, jac):
    return gpu.point_to_affine(curve.curve_id, group, np.ascontiguousarray(jac, dtype=np.uint64)).tobytes()


# ---- 1. known discrete logs ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precomp", (False, True), ids=("plain", "precomp"))
@pytest.mark.parametrize("pair", PAIR_IDS)
def test_index_sets(gpu, monkeypatch, pair, precomp):
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    t, ks = make_table(gpu, curve, group, N_TABLE, precomp)
    rng = seeded("indexed", pair, precomp)
    for name, idx in index_sets(N_TABLE, rng).items():
        c = default_window(curve, idx.size)
        for fam in ("mixed", "uniform"):
            check_indexed(t, curve, group, ks, idx, pack(curve, c, fam, idx.size, rng),
                          f"{pair} precomp={precomp} index set {name} family={fam}")
    t.free()


WINDOW_EDGES = sorted({(1 << k) + d for k in range(9, 21) for d in (-1, 0)})


@pytest.mark.parametrize("k", WINDOW_EDGES)
@pytest.mark.parametrize("pair", ["bn254-g1", "bls12-381-g2", "bw6-761-g1"])
def test_window_edges(gpu, monkeypatch, pair, k):
    """index counts on both sides of every size where msm_window_for changes, into a plain table of N_TABLE points
    (the window follows k, not the table); up to 2^20 indices, so every base is used many times"""
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    t, ks = make_table(gpu, curve, group, N_TABLE, False)
    g = np.random.default_rng(seeded("edges", pair, k).randrange(1 << 63))
    idx = g.integers(0, N_TABLE, size=k, dtype=np.uint32)
    sc = pack(curve, default_window(curve, k), "mixed", k, seeded("edges-sc", pair, k))
    check_indexed(t, curve, group, ks, idx, sc, f"{pair} k={k}")
    t.free()


# ---- 2. the BSB22 shape --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve", [BN254, BLS12_381], ids=["bn254", "bls12-381"])
def test_bsb22_shape(gpu, monkeypatch, curve):
    """1, 2, 3 and 100 indices into a plain 2^20-point table: the last point, the first, and random ones"""
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    n = 1 << 20
    t, ks = make_table(gpu, curve, 1, n, False)
    rng = seeded("bsb22-shape", curve.name)
    for k in (1, 2, 3, 100):
        idx = np.array(([n - 1, 0] + [rng.randrange(n) for _ in range(k)])[:k], dtype=np.uint32)
        check_indexed(t, curve, 1, ks, idx, pack(curve, 4, "uniform", k, rng), f"{curve.name} k={k}")
    t.free()


# ---- 3. equal to b200_msm over the dense vector ------------------------------------------------------------------------
@pytest.mark.parametrize("precomp", (False, True), ids=("plain", "precomp"))
@pytest.mark.parametrize("pair", ["bn254-g1", "bn254-g2", "bls12-381-g1", "bls12-377-g2", "bw6-761-g1"])
def test_equals_dense_msm(gpu, monkeypatch, pair, precomp):
    """canonical affine bytes of the indexed MSM = those of b200_msm over the n-vector that scatters and sums the same
    (index, scalar) entries"""
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    t, ks = make_table(gpu, curve, group, N_TABLE, precomp)
    rng = seeded("dense", pair, precomp)
    idx = np.array([rng.randrange(N_TABLE) for _ in range(800)], dtype=np.uint32)
    sc = pack(curve, 9, "mixed", idx.size, rng)
    dense = [0] * N_TABLE
    for i, s in zip(idx.tolist(), ff.unpack_elements(sc, curve.r, curve.fr_limbs)):
        dense[i] = (dense[i] + s) % curve.r
    got = t.msm_indexed(idx, sc)
    want = t.msm(ff.pack_elements(dense, curve.r, curve.fr_limbs))
    assert canonical_affine(gpu, curve, group, got) == canonical_affine(gpu, curve, group, want)
    assert jac_to_affine(curve, group, got) == expected(curve, group, np.ascontiguousarray(ks[idx]), sc)
    t.free()


# ---- 4. placements -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precomp", (False, True), ids=("plain", "precomp"))
@pytest.mark.parametrize("pair", ["bn254-g1", "bn254-g2", "bls12-381-g1", "bls12-381-g2"])
def test_placements(gpu, monkeypatch, pair, precomp):
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    t, ks = make_table(gpu, curve, group, N_TABLE, precomp)
    rng = seeded("placement", pair, precomp)
    idx = np.array([rng.randrange(N_TABLE) for _ in range(1234)], dtype=np.uint32)
    sc = pack(curve, 6, "uniform", idx.size, rng)
    check_indexed(t, curve, group, ks, idx, sc, f"{pair} all host")
    want = canonical_affine(gpu, curve, group, t.msm_indexed(idx, sc))
    for idx_dev in (False, True):
        for sc_dev in (False, True):
            i_ = to_dev(idx, np.int32) if idx_dev else idx
            s_ = to_dev(sc) if sc_dev else sc
            got = canonical_affine(gpu, curve, group, t.msm_indexed(i_, s_))
            assert got == want, f"{pair} idx on device={idx_dev} scalars on device={sc_dev}"
    t.free()


# ---- 5. the Ethereum ceremony ----------------------------------------------------------------------------------------------
def test_ethereum_ceremony_lagrange_commitment(gpu):
    """the fixture's 4096 Lagrange points as a table (natural order, as test_gpu_points_ntt.py): the indexed commitment
    of a sparse Lagrange-form vector v equals the MSM of the monomial points with the oracle's inverse NTT of v (its
    coefficients) - tau is unknown, both bases come from the ceremony"""
    mono, lag, _ = kzg_srs.load()
    C, logn = BLS12_381, 12
    F = ff.Fp(C.p)
    t = gpu.Table(C.curve_id, 1, ec.pack_points(C, 1, lag), precomp=False)
    rng = random.Random(4096)
    for k in (1, 3, 40):
        pos = rng.sample(range(kzg_srs.N), k - 1) + [kzg_srs.N - 1]
        vals = [rng.randrange(1, C.r) for _ in range(k)]
        v = [0] * kzg_srs.N
        for p_, x in zip(pos, vals):
            v[p_] = x
        coeffs = fr_transform(C, ff.pack_elements(v, C.r, C.fr_limbs), logn, True)
        want = ec.from_jac(F, ec.unpack_points(C, 1, corelib.msm(C, 1, ec.pack_points(C, 1, mono), coeffs), ncoords=3)[0])
        got = jac_to_affine(C, 1, t.msm_indexed(np.array(pos, dtype=np.uint32), ff.pack_elements(vals, C.r, C.fr_limbs)))
        assert got == want, f"k={k}"
    t.free()


# ---- 6. PLONK: the hint's commitment ---------------------------------------------------------------------------------------
def lagrange_dlogs(curve, n, tau):
    """L_i(tau) = (w^i / n) (tau^n - 1) / (tau - w^i) on the domain of size n"""
    r = curve.r
    w = ntt.Domain(curve, n).generator
    zh = (pow(tau, n, r) - 1) % r
    ninv = pow(n, -1, r)
    return [pow(w, i, r) * ninv % r * zh % r * pow((tau - pow(w, i, r)) % r, -1, r) % r for i in range(n)]


@pytest.mark.parametrize("n_commit", (1, 2))
@pytest.mark.parametrize("curve", [BN254, BLS12_381], ids=["bn254", "bls12-381"])
def test_plonk_bsb22_commitment(gpu, curve, n_commit):
    """plonk.bsb22_commitment over the Lagrange SRS [L_i(tau)]G = the oracle prover's [PI2_j] = the device prover's
    [PI2_j] (canonical form on the monomial SRS) for the same committed polynomial, laid out as the hint lays it out"""
    from gnark_b200 import plonk as b200_plonk
    from oracle import plonk_prover as pp
    r, L = curve.r, curve.fr_limbs
    logn = 5
    n = 1 << logn
    rng = random.Random(9000 + 10 * n_commit + curve.curve_id)
    circ, l, rr, o, pi2_rand = pp.random_satisfied_instance(curve, n, seed=81 + n_commit, n_commit=n_commit)
    tau = rng.randrange(r)
    pe = lambda v: ff.pack_elements(v, r, L)
    lag = gpu.Table(curve.curve_id, 1, gpu.fixed_base_batch(curve.curve_id, 1, ec.pack_points(curve, 1, [curve.g1])[0],
                                                            pe(lagrange_dlogs(curve, n, tau))), precomp=False)
    nb_public, nb_constraints = 3, n - 3
    digests, pi2 = [], []
    for j in range(n_commit):
        free = rng.sample(range(nb_constraints - 1), 6)
        committed, commitment_index = free[:5], free[5]
        values = pe([rng.randrange(r) for _ in committed])
        blind2 = [(commitment_index, pe([rng.randrange(r)])[0]), (nb_constraints - 1, pe([rng.randrange(r)])[0])]
        d, dense = b200_plonk.bsb22_commitment(lag, nb_public, committed, values, blind2)
        assert dense.shape == (n, L) and np.count_nonzero(dense.any(axis=1)) == 7
        digests.append(d)
        pi2.append(ff.unpack_elements(dense, r, L))
    lag.free()
    # keep the gate equation satisfied with the hint's vectors: qk absorbs the difference (o and the copy constraints
    # stay as the instance built them)
    for i in range(n):
        circ.qk[i] = (circ.qk[i] + sum(circ.qcp[j][i] * (pi2_rand[j][i] - pi2[j][i]) for j in range(n_commit))) % r
    rnd = lambda: rng.randrange(r)
    ch = pp.Challenges(gamma=rnd(), beta=rnd(), alpha=rnd(), zeta=rnd(), v=rnd(), bl=[rnd(), rnd()], br=[rnd(), rnd()],
                       bo=[rnd(), rnd()], bz=[rnd(), rnd(), rnd()])
    want = pp.prove(curve, circ, l, rr, o, ch, tau, pi2=pi2)
    assert pp.verify(curve, circ, want, ch, tau)
    F = ff.Fp(curve.p)
    for j in range(n_commit):
        assert jac_to_affine(curve, 1, digests[j]) == ec.scalar_mul(F, want.bsb22[j], curve.g1), f"oracle [PI2_{j}]"
    srs = corelib.fixed_base(curve, 1, ec.pack_points(curve, 1, [curve.g1]), pe([pow(tau, i, r) for i in range(n + 3)]))
    key = gpu.PlonkKey(curve.curve_id, logn, pe(circ.ql), pe(circ.qr), pe(circ.qm), pe(circ.qo), pe(circ.qk),
                       np.array(circ.perm, dtype=np.int64), srs, qcp=[pe(v) for v in circ.qcp])
    _, _, bsb = key.prove(pe(l), pe(rr), pe(o), pe([ch.gamma]), pe([ch.beta]), pe([ch.alpha]), pe([ch.zeta]), pe([ch.v]),
                          pe(ch.bl), pe(ch.br), pe(ch.bo), pe(ch.bz), pi2=[pe(v) for v in pi2])
    key.free()
    for j in range(n_commit):
        assert jac_to_affine(curve, 1, bsb[j]) == jac_to_affine(curve, 1, digests[j]), f"device [PI2_{j}]"


# ---- 7. errors -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precomp", (False, True), ids=("plain", "precomp"))
def test_errors(gpu, precomp):
    import torch
    c = BN254
    L = gpu.load()
    null = ctypes.c_void_p(0)
    n = 64
    t, ks = make_table(gpu, c, 1, n, precomp)
    rng = seeded("errors", precomp)
    sc = pack(c, 4, "uniform", 10, rng)
    idx = np.array([rng.randrange(n) for _ in range(10)], dtype=np.uint32)
    want = check_indexed(t, c, 1, ks, idx, sc, "valid call")
    out = np.full(3 * c.fp_limbs, 7, dtype=np.uint64)

    def fails(match, rc):
        assert rc != 0
        assert match in L.b200_last_error().decode(), L.b200_last_error()
        assert (out == 7).all(), "the output was written"

    fails("msm_indexed: null table", L.b200_msm_indexed(null, gpu.ptr(idx), 10, 0, gpu.ptr(sc), 0, gpu.ptr(out)))
    fails("msm_indexed: null argument", L.b200_msm_indexed(t.handle, null, 10, 0, gpu.ptr(sc), 0, gpu.ptr(out)))
    fails("msm_indexed: null argument", L.b200_msm_indexed(t.handle, gpu.ptr(idx), 10, 0, null, 0, gpu.ptr(out)))
    with pytest.raises(gpu.B200Error, match="null argument"):
        gpu.check(L.b200_msm_indexed(t.handle, gpu.ptr(idx), 10, 0, gpu.ptr(sc), 0, null))
    # n = 0: null buffers are accepted, the result is the point at infinity
    for on_dev in (0, 1):
        gpu.check(L.b200_msm_indexed(t.handle, null, 0, on_dev, null, on_dev, gpu.ptr(out)))
        assert jac_to_affine(c, 1, out) is ec.INF
        out[:] = 7
    # a host index out of range: the message names it and its position
    bad = idx.copy()
    bad[7] = n
    fails(f"msm_indexed: index {n} out of range at position 7",
          L.b200_msm_indexed(t.handle, gpu.ptr(bad), 10, 0, gpu.ptr(sc), 0, gpu.ptr(out)))
    assert jac_to_affine(c, 1, t.msm_indexed(idx, sc)) == want
    # device indices out of range: the check kernel finds the lowest bad position before the MSM is enqueued
    bad[3] = 0xFFFFFFFF
    d_bad, d_sc = to_dev(bad, np.int32), to_dev(sc)
    fails("msm_indexed: device index out of range at position 3",
          L.b200_msm_indexed(t.handle, gpu.ptr(d_bad), 10, 1, gpu.ptr(d_sc), 1, gpu.ptr(out)))
    torch.cuda.synchronize()
    assert jac_to_affine(c, 1, t.msm_indexed(to_dev(idx, np.int32), d_sc)) == want
    t.free()
