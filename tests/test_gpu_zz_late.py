"""GPU tests of the entry points added late in round 1 (all of them run unguarded on an H100).

  * test_cuda_reproduces_golden   - the CUDA path on the committed known-answer vectors (tests/golden)
  * test_cuda_reproduces_eth_kzg_srs - the CUDA path on the reference's external fixture (Ethereum KZG ceremony SRS)
  * test_cuda_reproduces_intree_known_answers - the CUDA path on the curve constants the reference spells out (GLV
                                    endomorphism on G1, [2^k] G2), all curves
  * test_full_prover_vs_oracle    - the device PLONK prover (gnark_b200/plonk.py) against the big-int oracle
                                    prover, same injected challenges
"""
import json
import os
import random

import numpy as np
import pytest

from oracle import ec, ff, groth16 as g16
from oracle.params import CURVES
from util import jac_to_affine

pytestmark = pytest.mark.gpu
KAT = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_v1.json")))
ALL = list(CURVES.values())
H = lambda s: int(s, 16)


def pt(F, v):
    if v is None:
        return None
    conv = (lambda x: (H(x[0]), H(x[1]))) if F.degree == 2 else H
    return (conv(v[0]), conv(v[1]))


@pytest.mark.parametrize("c", ALL, ids=lambda c: c.name)
def test_cuda_reproduces_golden(gpu, c):
    e = KAT["curves"][c.name]
    for group in (1, 2):
        F = ff.base_field(c, group)
        m = e[f"msm_g{group}"]
        pts = [pt(F, p) for p in m["points"]]
        sc = [H(s) for s in m["scalars"]]
        for precomp in (False, True):
            t = gpu.Table(c.curve_id, group, ec.pack_points(c, group, pts), precomp=precomp)
            got = t.msm(ff.pack_elements(sc, c.r, c.fr_limbs))
            assert ec.from_jac(F, ec.unpack_points(c, group, got, ncoords=3)[0]) == pt(F, m["result"])
            t.free()
    n8 = e["ntt8"]
    a = [H(x) for x in n8["input"]]
    d = gpu.Domain(c.curve_id, 3)
    for key, out in n8["out"].items():
        inv, dec, cos = int(key[3]), int(key[8]), int(key[-1])
        A = d.ntt(ff.pack_elements(a, c.r, c.fr_limbs), inverse=bool(inv), decimation=dec, on_coset=bool(cos))
        assert ff.unpack_elements(A, c.r, c.fr_limbs) == [H(x) for x in out]
    # computeH of the cubic circuit
    gc = e["groth16_cubic"]
    cs, W = g16.cubic_r1cs(), g16.cubic_witness(c.r)
    A_, B_, C_ = g16.solve_abc(cs, W, c.r)
    d2 = gpu.Domain(c.curve_id, 2)
    got = d2.compute_h(*(ff.pack_elements(v, c.r, c.fr_limbs) for v in (A_, B_, C_)))
    assert ff.unpack_elements(got, c.r, c.fr_limbs) == [H(v) for v in gc["h_bitreversed"]]
    d.free(); d2.free()


def test_cuda_reproduces_eth_kzg_srs(gpu):
    """EXTERNAL known-answer vectors (tests/test_golden_kzg.py): the Ethereum KZG ceremony SRS the reference ships
    (std/evmprecompiles/kzg_trusted_setup.json).  CUDA BLS12-381 G1 MSM of 4096 externally produced points against
    externally produced answers, and the CUDA NTT pinned through MSM(monomial, c) = MSM(lagrange, NTT(c))."""
    import random as _r
    from oracle import kzg_srs, ntt
    from oracle.params import BLS12_381 as C
    from test_golden_kzg import kat_cases
    mono, lag, _ = kzg_srs.load()
    pts = {"mono": mono, "lag": lag}
    F = ff.Fp(C.p)
    N, LOGN = kzg_srs.N, kzg_srs.LOGN
    aff = lambda out: ec.from_jac(F, ec.unpack_points(C, 1, out, ncoords=3)[0])
    for precomp in (False, True):
        T = {"MONO": gpu.Table(C.curve_id, 1, ec.pack_points(C, 1, mono), precomp=precomp),
             "LAG": gpu.Table(C.curve_id, 1, ec.pack_points(C, 1, lag), precomp=precomp)}
        for base, sc, (other, j) in kat_cases(_r.Random(1)):
            assert aff(T[base].msm(ff.pack_elements(sc, C.r, C.fr_limbs))) == pts[other][j], (precomp, base, other, j)
        rng = _r.Random(2)
        c = [rng.randrange(C.r) for _ in range(N)]
        commit = aff(T["MONO"].msm(ff.pack_elements(c, C.r, C.fr_limbs)))
        d = gpu.Domain(C.curve_id, LOGN)
        e_br = d.ntt(ff.pack_elements(c, C.r, C.fr_limbs), inverse=False, decimation=ntt.DIF)
        e = d.ntt(ff.pack_elements(ntt.bit_reverse(list(c)), C.r, C.fr_limbs), inverse=False, decimation=ntt.DIT)
        assert ntt.bit_reverse(ff.unpack_elements(e_br, C.r, C.fr_limbs)) == ff.unpack_elements(e, C.r, C.fr_limbs)
        assert aff(T["LAG"].msm(e)) == commit
        back = d.ntt(e.copy(), inverse=True, decimation=ntt.DIF)
        assert ntt.bit_reverse(ff.unpack_elements(back, C.r, C.fr_limbs)) == c
        d.free()
        for t in T.values():
            t.free()
    # G2: CUDA MSM over the fixture's 65 G2 points, tied to the (known-answer-pinned) G1 side through the pairing
    from oracle import pairing_bls12_381 as pr
    from test_golden_kzg import g2_case
    g2pts = kzg_srs.load()[2]
    F2 = ff.base_field(C, 2)
    c2, SC2, A = g2_case({"mono": mono})
    for precomp in (False, True):
        t2 = gpu.Table(C.curve_id, 2, ec.pack_points(C, 2, g2pts), precomp=precomp)
        B = ec.from_jac(F2, ec.unpack_points(C, 2, t2.msm(SC2), ncoords=3)[0])
        t2.free()
        assert B == ec.msm_naive(F2, g2pts, c2)
    assert pr.pairing_product_is_one([(A, C.g2), (ec.affine_neg(F, C.g1), B)])


@pytest.mark.parametrize("cname,group", [(n, g) for n in ("bn254", "bls12-381", "bls12-377", "bw6-761") for g in (1, 2)
                                         if not (n == "bls12-377" and g == 2)])
def test_cuda_reproduces_intree_known_answers(gpu, cname, group):
    """EXTERNAL known answers (tests/test_golden_intree.py): [lambda] P = (omega x, y) on G1 of all four curves and
    [2^65] G2 / [2^96] G2 from the constants the reference spells out in its sources - as a one-point MSM and folded
    into a 200-point MSM, plain and precomputed tables."""
    from test_golden_intree import folded_msm, known_answer
    c = CURVES[cname]
    F, base, k, expected = known_answer(c, group)
    aff = lambda out: ec.from_jac(F, ec.unpack_points(c, group, out, ncoords=3)[0])
    F, pts, sc, want = folded_msm(c, group, 200, 13)
    assert want == expected
    for precomp in (False, True):
        t1 = gpu.Table(c.curve_id, group, ec.pack_points(c, group, [base]), precomp=precomp)
        assert aff(t1.msm(ff.pack_elements([k], c.r, c.fr_limbs))) == expected
        t1.free()
        t = gpu.Table(c.curve_id, group, ec.pack_points(c, group, pts), precomp=precomp)
        assert aff(t.msm(ff.pack_elements(sc, c.r, c.fr_limbs))) == expected
        t.free()


@pytest.mark.parametrize("c", [CURVES["bn254"], CURVES["bls12-381"]], ids=lambda c: c.name)
@pytest.mark.parametrize("logn", (4, 6))
def test_full_prover_vs_oracle(gpu, c, logn):
    """The device PLONK prover (gnark_b200/plonk.py, twin of backend/plonk/bn254/prove.go) against the
    big-int oracle prover with the same injected challenges / blinding: every digest (as dlog * G with a
    trapdoor SRS), every opened value; the oracle proof itself passes the verifier's equations."""
    from gnark_b200 import plonk as b200_plonk
    from oracle import corelib, plonk_prover as pp
    rng = random.Random(1000 + logn)
    r, L = c.r, c.fr_limbs
    n = 1 << logn
    circ, l, rr, o = pp.random_satisfied_instance(c, n, seed=logn)
    rnd = lambda: rng.randrange(r)
    ch = pp.Challenges(gamma=rnd(), beta=rnd(), alpha=rnd(), zeta=rnd(), v=rnd(), bl=[rnd(), rnd()], br=[rnd(), rnd()],
                       bo=[rnd(), rnd()], bz=[rnd(), rnd(), rnd()])
    tau = rnd()
    want = pp.prove(c, circ, l, rr, o, ch, tau)
    assert pp.verify(c, circ, want, ch, tau)
    # trapdoor SRS: [tau^i] G, i < n + 3  (test/unsafekzg/kzgsrs.go:142-172)
    pe = lambda v: ff.pack_elements(v, r, L)
    srs = corelib.fixed_base(c, 1, ec.pack_points(c, 1, [c.g1]), pe([pow(tau, i, r) for i in range(n + 3)]))
    pk = b200_plonk.ProvingKey.from_trace(c.curve_id, logn, pe(circ.ql), pe(circ.qr), pe(circ.qm), pe(circ.qo),
                                         pe(circ.qk), np.array(circ.perm, dtype=np.int64), srs)
    got = b200_plonk.Prove(pk, pe(l), pe(rr), pe(o),
                           b200_plonk.Challenges(gamma=ch.gamma, beta=ch.beta, alpha=ch.alpha, zeta=ch.zeta, v=ch.v,
                                                 bl=ch.bl, br=ch.br, bo=ch.bo, bz=ch.bz))
    F = ff.Fp(c.p)
    pt = lambda dlog: ec.scalar_mul(F, dlog, c.g1)
    for name, g_, w_ in (("L", got.LRO[0], want.L), ("R", got.LRO[1], want.R), ("O", got.LRO[2], want.O),
                         ("Z", got.Z, want.Z), ("H1", got.H[0], want.H[0]), ("H2", got.H[1], want.H[1]),
                         ("H3", got.H[2], want.H[2]), ("lin", got.LinearizedDigest, want.lin),
                         ("batch", got.BatchedProofH, want.batch_opening), ("zopen", got.ZShiftedOpeningH, want.z_opening)):
        assert jac_to_affine(c, 1, g_) == pt(w_), name
    assert got.BatchedClaimedValues == want.claimed
    assert got.ZShiftedClaimedValue == want.zu
    pk.free()


@pytest.mark.parametrize("c", [CURVES["bn254"], CURVES["bls12-381"]], ids=lambda c: c.name)
@pytest.mark.parametrize("logn", (4, 6))
def test_plonk_prove_c_abi_vs_oracle(gpu, c, logn):
    """b200_plonk_pk_load / b200_plonk_prove (one C call per proof) against the big-int oracle prover with the same
    injected challenges / blinding: all ten digests (trapdoor SRS: digest = dlog * G) and the seven opened values"""
    from oracle import corelib, plonk_prover as pp
    rng = random.Random(2000 + logn)
    r, L = c.r, c.fr_limbs
    n = 1 << logn
    circ, l, rr, o = pp.random_satisfied_instance(c, n, seed=logn + 50)
    rnd = lambda: rng.randrange(r)
    ch = pp.Challenges(gamma=rnd(), beta=rnd(), alpha=rnd(), zeta=rnd(), v=rnd(), bl=[rnd(), rnd()], br=[rnd(), rnd()],
                       bo=[rnd(), rnd()], bz=[rnd(), rnd(), rnd()])
    tau = rnd()
    want = pp.prove(c, circ, l, rr, o, ch, tau)
    assert pp.verify(c, circ, want, ch, tau)
    pe = lambda v: ff.pack_elements(v, r, L)
    srs = corelib.fixed_base(c, 1, ec.pack_points(c, 1, [c.g1]), pe([pow(tau, i, r) for i in range(n + 3)]))
    key = gpu.PlonkKey(c.curve_id, logn, pe(circ.ql), pe(circ.qr), pe(circ.qm), pe(circ.qo), pe(circ.qk),
                       np.array(circ.perm, dtype=np.int64), srs)
    pts, vals = key.prove(pe(l), pe(rr), pe(o), pe([ch.gamma]), pe([ch.beta]), pe([ch.alpha]), pe([ch.zeta]), pe([ch.v]),
                          pe(ch.bl), pe(ch.br), pe(ch.bo), pe(ch.bz))
    F = ff.Fp(c.p)
    dl = [want.L, want.R, want.O, want.Z, want.H[0], want.H[1], want.H[2], want.lin, want.batch_opening, want.z_opening]
    for k, name in enumerate(("L", "R", "O", "Z", "H1", "H2", "H3", "lin", "batch", "zopen")):
        assert jac_to_affine(c, 1, pts[k]) == ec.scalar_mul(F, dl[k], c.g1), name
    got_vals = ff.unpack_elements(vals, r, L)
    assert got_vals[:6] == want.claimed and got_vals[6] == want.zu
    # prove -> Verify: the verifier's equations on the CUDA prover's points, real pairings
    assert pp.verify_pairing(c, circ, [jac_to_affine(c, 1, pts[k]) for k in range(10)], got_vals, ch, tau)
    key.free()


def test_plonk_proof_over_the_ethereum_srs_verifies(gpu):
    """No trapdoor anywhere: b200_plonk_prove commits with the Ethereum KZG ceremony SRS the reference ships (tau unknown,
    2051 of its 4096 G1 points, n = 2^11) and the proof is checked by the verifier's pairing equations with the fixture's
    own [tau]_2 (CPU twin with the mocked kernels: tests/test_plonk_host_cpu.py)."""
    from oracle import corelib, kzg_srs, plonk_prover as pp
    c = CURVES["bls12-381"]
    logn = 11
    n = 1 << logn
    r, L = c.r, c.fr_limbs
    rng = random.Random(78)
    mono, _, g2 = kzg_srs.load()
    circ, l, rr, o = pp.random_satisfied_instance(c, n, seed=124)
    rnd = lambda: rng.randrange(r)
    ch = pp.Challenges(gamma=rnd(), beta=rnd(), alpha=rnd(), zeta=rnd(), v=rnd(), bl=[rnd(), rnd()], br=[rnd(), rnd()],
                       bo=[rnd(), rnd()], bz=[rnd(), rnd(), rnd()])
    pe = lambda v: ff.pack_elements(v, r, L)
    key = gpu.PlonkKey(c.curve_id, logn, pe(circ.ql), pe(circ.qr), pe(circ.qm), pe(circ.qo), pe(circ.qk),
                       np.array(circ.perm, dtype=np.int64), ec.pack_points(c, 1, mono[:n + 3]))
    pts, vals = key.prove(pe(l), pe(rr), pe(o), pe([ch.gamma]), pe([ch.beta]), pe([ch.alpha]), pe([ch.zeta]), pe([ch.v]),
                          pe(ch.bl), pe(ch.br), pe(ch.bo), pe(ch.bz))
    key.free()
    F = ff.Fp(c.p)

    def cpp_msm(points, scalars):
        out = corelib.msm(c, 1, ec.pack_points(c, 1, points), pe(scalars))
        return ec.from_jac(F, ec.unpack_points(c, 1, out, ncoords=3)[0])
    proof_pts = [jac_to_affine(c, 1, pts[k]) for k in range(10)]
    got = ff.unpack_elements(vals, r, L)
    assert pp.verify_pairing(c, circ, proof_pts, got, ch, srs_g1=mono, tau_g2=g2[1], msm=cpp_msm)
    assert not pp.verify_pairing(c, circ, proof_pts, got, ch, srs_g1=mono, tau_g2=g2[2], msm=cpp_msm)


@pytest.mark.parametrize("n_commit", (1, 2))
def test_plonk_prove_bsb22(gpu, n_commit):
    """b200_plonk_prove on a key with BSB22 commitment gates against the oracle prover: digests (incl. [PI2_j]) and the
    7 + n_commit opened values"""
    from oracle import corelib, plonk_prover as pp
    c = CURVES["bn254"]
    logn = 5
    rng = random.Random(5000 + n_commit)
    r, L = c.r, c.fr_limbs
    n = 1 << logn
    circ, l, rr, o, pi2 = pp.random_satisfied_instance(c, n, seed=71, n_commit=n_commit)
    rnd = lambda: rng.randrange(r)
    ch = pp.Challenges(gamma=rnd(), beta=rnd(), alpha=rnd(), zeta=rnd(), v=rnd(), bl=[rnd(), rnd()], br=[rnd(), rnd()],
                       bo=[rnd(), rnd()], bz=[rnd(), rnd(), rnd()])
    tau = rnd()
    want = pp.prove(c, circ, l, rr, o, ch, tau, pi2=pi2)
    assert pp.verify(c, circ, want, ch, tau)
    pe = lambda v: ff.pack_elements(v, r, L)
    srs = corelib.fixed_base(c, 1, ec.pack_points(c, 1, [c.g1]), pe([pow(tau, i, r) for i in range(n + 3)]))
    key = gpu.PlonkKey(c.curve_id, logn, pe(circ.ql), pe(circ.qr), pe(circ.qm), pe(circ.qo), pe(circ.qk),
                       np.array(circ.perm, dtype=np.int64), srs, qcp=[pe(v) for v in circ.qcp])
    pts, vals, bsb = key.prove(pe(l), pe(rr), pe(o), pe([ch.gamma]), pe([ch.beta]), pe([ch.alpha]), pe([ch.zeta]),
                               pe([ch.v]), pe(ch.bl), pe(ch.br), pe(ch.bo), pe(ch.bz), pi2=[pe(v) for v in pi2])
    F = ff.Fp(c.p)
    dl = [want.L, want.R, want.O, want.Z, want.H[0], want.H[1], want.H[2], want.lin, want.batch_opening, want.z_opening]
    for k in range(10):
        assert jac_to_affine(c, 1, pts[k]) == ec.scalar_mul(F, dl[k], c.g1), k
    for j in range(n_commit):
        assert jac_to_affine(c, 1, bsb[j]) == ec.scalar_mul(F, want.bsb22[j], c.g1)
    got = ff.unpack_elements(vals, r, L)
    assert got[:6] + got[7:] == want.claimed and got[6] == want.zu
    key.free()


@pytest.mark.parametrize("cname", ["bn254", "bls12-381"])
def test_plonk_prove_reproduces_golden(gpu, cname):
    """the committed PLONK known-answer vector (tests/golden/kat_plonk_v1.json) through b200_plonk_prove on the GPU"""
    from oracle import corelib
    from test_golden import _plonk_case
    c, circ, l, rr, o, pi2, ch, tau, want = _plonk_case(cname)
    r, L = c.r, c.fr_limbs
    n, logn = circ.n, circ.n.bit_length() - 1
    pe = lambda v: ff.pack_elements(v, r, L)
    srs = corelib.fixed_base(c, 1, ec.pack_points(c, 1, [c.g1]), pe([pow(tau, i, r) for i in range(n + 3)]))
    key = gpu.PlonkKey(c.curve_id, logn, pe(circ.ql), pe(circ.qr), pe(circ.qm), pe(circ.qo), pe(circ.qk),
                       np.array(circ.perm, dtype=np.int64), srs, qcp=[pe(v) for v in circ.qcp])
    pts, vals, bsb = key.prove(pe(l), pe(rr), pe(o), pe([ch.gamma]), pe([ch.beta]), pe([ch.alpha]), pe([ch.zeta]),
                               pe([ch.v]), pe(ch.bl), pe(ch.br), pe(ch.bo), pe(ch.bz), pi2=[pe(v) for v in pi2])
    F = ff.Fp(c.p)
    dl = [H(want[k]) for k in ("L", "R", "O", "Z")] + [H(x) for x in want["H"]] + [H(want["lin"]), H(want["batch_opening"]),
                                                                                  H(want["z_opening"])]
    for k in range(10):
        assert jac_to_affine(c, 1, pts[k]) == ec.scalar_mul(F, dl[k], c.g1), k
    assert jac_to_affine(c, 1, bsb[0]) == ec.scalar_mul(F, H(want["bsb22"][0]), c.g1)
    got = ff.unpack_elements(vals, r, L)
    assert got[:6] + got[7:] == [H(x) for x in want["claimed"]] and got[6] == H(want["zu"])
    key.free()


def test_groth16_committed_wires_filtered_from_k(gpu):
    """Groth16 keys with Pedersen/BSB22 commitments: the committed private wires have no base in G1.K and are
    dropped from the Krs scalars (filterHeap, prove.go:231-239,321-344).  The K MSM must equal
    sum over the remaining private wires of w_i * K_i; the other four MSMs are unchanged."""
    from gnark_b200 import groth16 as b200
    from oracle import groth16 as g16
    from util import build_groth16_pk, pack_solution
    c = CURVES["bn254"]
    m_ = 300
    cs, W = g16.square_chain_r1cs(m_), g16.square_chain_witness(c.r, m_)
    pk, pkd, (F1, g1), (F2, g2) = build_groth16_pk(c, cs, g16.random_toxic(c, 3), 3)
    rng = random.Random(3)
    nb_pub = cs.nb_public
    nb_wires = len(W)
    removed = sorted(rng.sample(range(nb_pub, nb_wires), 17))
    keep = [i for i in range(nb_pub, nb_wires) if i not in set(removed)]
    per = 2 * c.fp_limbs
    K_full = pk.G1_K.reshape(-1, per)
    pk2 = b200.ProvingKey.from_arrays(
        c.curve_id, pk.domain_size, pk.G1_Alpha, pk.G1_Beta, pk.G1_Delta, pk.G1_A, pk.G1_B, pk.G1_Z,
        np.ascontiguousarray(K_full[[i - nb_pub for i in keep]]), pk.G2_Beta, pk.G2_Delta, pk.G2_B, pk.InfinityA, pk.InfinityB,
        nb_pub, committed_private_wires=removed)
    rs = [rng.randrange(c.r), rng.randrange(c.r)]
    it = iter(rs)
    proof = b200.ProveSolution(pk2, pack_solution(c, cs, W), b200.WithDeviceID(0), b200.WithRandomness(lambda q: next(it)),
                               keep_msm=True)
    want = g16.prove_dlog(c, cs, pkd, W, rs[0], rs[1])
    Lj = 3 * c.fp_limbs
    msm = proof.msm
    for k, dlog in ((0, want.msm_a), (1, want.msm_b), (2, want.msm_z)):
        assert ec.from_jac(F1, ec.unpack_points(c, 1, msm[k * Lj:(k + 1) * Lj], ncoords=3)[0]) == ec.scalar_mul(F1, dlog, g1)
    k_dlog = sum(W[i] * pkd.K[i - nb_pub] for i in keep) % c.r
    assert ec.from_jac(F1, ec.unpack_points(c, 1, msm[3 * Lj:4 * Lj], ncoords=3)[0]) == ec.scalar_mul(F1, k_dlog, g1)
    pk2.free_gpu_resources()


@pytest.mark.parametrize("cname,logn", [("bn254", 22), ("bls12-381", 24)])
def test_ntt_full_size_identities(gpu, cname, logn):
    """SURVEY.md §8c-4 at BASELINE sizes (2^22, 2^24), where no CPU oracle run is affordable: the inverse transform
    undoes the forward one bit for bit, and X[k] = p(w^k) at a few random k (Horner evaluation of the 2^logn
    coefficients by b200_poly_eval against the NTT output, plain and on the coset)."""
    import torch
    from oracle import ntt
    c = CURVES[cname]
    L = c.fr_limbs
    n = 1 << logn
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randint(0, 1 << 62, (n, L), dtype=torch.int64, device="cuda", generator=g)
    x[:, L - 1] &= (1 << 56) - 1                      # < r: valid Montgomery residues
    x = x.reshape(-1).contiguous()
    d = gpu.Domain(c.curve_id, logn)
    dom = ntt.Domain(c, n)                             # generator / coset constants only
    rng = random.Random(8)
    for on_coset in (False, True):
        y = x.clone()
        # the library runs on its own non-blocking stream (no b200_set_stream here): torch's producer kernels must have
        # finished before it reads y.  Round 1's failure of [bls12-381-24] was this race in the TEST (the 512 MiB clone
        # was still in flight when the first NTT pass started), not a kernel fault - see test_ntt_large_vs_cpp_oracle.
        torch.cuda.synchronize()
        d.ntt_async(y, inverse=False, decimation=gpu.DIF, on_coset=on_coset)      # natural -> bit-reversed
        gpu.sync(0)
        for _ in range(3):
            k = rng.randrange(n)
            point = pow(dom.generator, k, c.r) * (dom.coset_gen if on_coset else 1) % c.r
            want = gpu.poly_eval(0, c.curve_id, x, n, ff.pack_elements([point], c.r, L))
            pos = ntt.bitrev(k, logn)
            got = y[pos * L:(pos + 1) * L].cpu().numpy().view(np.uint64)
            assert np.array_equal(got, want.reshape(-1)), (cname, logn, on_coset, k)
        d.ntt_async(y, inverse=True, decimation=gpu.DIT, on_coset=on_coset)       # bit-reversed -> natural
        gpu.sync(0)
        assert torch.equal(y, x), (cname, logn, on_coset)
    d.free()


@pytest.mark.parametrize("cname,logn", [("bls12-381", 22), ("bls12-381", 24), ("bn254", 24)])
def test_ntt_large_vs_cpp_oracle(gpu, cname, logn):
    """three-pass plans (2^22: PLONK config 4's domain, 2^24: its 4n quotient domain) limb for limb against the
    multi-threaded C++ oracle, forward DIF plain and inverse DIT on the coset, host buffers through b200_ntt"""
    from oracle import corelib
    c = CURVES[cname]
    n = 1 << logn
    rs = np.random.RandomState(logn)
    a = rs.randint(0, 1 << 62, size=(n, c.fr_limbs), dtype=np.int64).astype(np.uint64)
    a[:, -1] &= np.uint64((1 << 56) - 1)
    d = gpu.Domain(c.curve_id, logn)
    for inv, dec, cos in ((False, gpu.DIF, False), (True, gpu.DIT, True)):
        want = corelib.ntt(c, a.copy(), logn, inv, dec, cos)
        got = d.ntt(a.copy(), inverse=inv, decimation=dec, on_coset=cos)
        assert np.array_equal(got, want), (cname, logn, inv, dec, cos)
    d.free()


def test_sharded_ntt_single_rank(gpu):
    """gnark_b200/parallel_ntt.py with world = 1 on the GPU: no exchange, but the stream scoping, the local
    transform + bit reversal and the coset scaling are the ones every rank runs (multi-rank: tools/bench_sharded_ntt.py)"""
    import torch
    from gnark_b200 import parallel_ntt as pn
    from oracle import ntt
    c = CURVES["bn254"]
    logn = 10
    n = 1 << logn
    rng = random.Random(5)
    x = [rng.randrange(c.r) for _ in range(n)]
    X = ff.pack_elements(x, c.r, c.fr_limbs).reshape(n, c.fr_limbs)
    dom = ntt.Domain(c, n)
    sd = pn.ShardedDomain(c.curve_id, logn, 0, 1)
    for on_coset in (False, True):
        d = torch.from_numpy(X.view(np.int64).reshape(-1).copy()).cuda()
        got = sd.forward(d, on_coset=on_coset).cpu().numpy().view(np.uint64)
        want = ntt.bit_reverse(dom.fft(list(x), ntt.DIF, on_coset=on_coset))
        assert ff.unpack_elements(got, c.r, c.fr_limbs) == want
        back = sd.inverse(sd.forward(torch.from_numpy(X.view(np.int64).reshape(-1).copy()).cuda(), on_coset=on_coset),
                          on_coset=on_coset).cpu().numpy().view(np.uint64)
        assert ff.unpack_elements(back, c.r, c.fr_limbs) == x
    sd.free()


def test_msm_submit_stream_of_msms(gpu):
    """b200_msm_submit: a stream of MSMs from pinned host buffers (different scalars, different ranges), results
    after b200_sync, each against the known-dlog oracle"""
    import torch
    from util import known_dlog_instance
    c = CURVES["bn254"]
    n = 6000
    F, base, pts, sc, expected = known_dlog_instance(c, 1, n, seed=77)
    t = gpu.Table(c.curve_id, 1, pts, precomp=True)
    h_sc = torch.from_numpy(sc.view(np.int64).copy()).pin_memory()
    K = 6
    h_out = torch.zeros((K, 12), dtype=torch.int64).pin_memory()
    for i in range(K):
        t.msm_submit(h_sc, h_out[i], n=n)
    gpu.sync(0)
    for i in range(K):
        assert jac_to_affine(c, 1, h_out[i].numpy().view(np.uint64)) == expected
    # a sub-range and the empty sum
    half = n // 2
    h2 = torch.zeros((2, 12), dtype=torch.int64).pin_memory()
    t.msm_submit(h_sc.view(n, 4)[:half], h2[0], n=half)
    t.msm_submit(h_sc, h2[1], n=0)
    gpu.sync(0)
    want_half = jac_to_affine(c, 1, t.msm(sc[:half].copy(), n=half))
    assert jac_to_affine(c, 1, h2[0].numpy().view(np.uint64)) == want_half
    assert jac_to_affine(c, 1, h2[1].numpy().view(np.uint64)) is None
    t.free()


@pytest.mark.parametrize("c", ALL, ids=lambda c: c.name)
@pytest.mark.parametrize("group", (1, 2))
def test_fixed_base_batch(gpu, c, group):
    """b200_fixed_base_batch (curve.BatchScalarMultiplicationG1/G2, setup.go:233,302) against the C++ oracle's
    fixed-base batch, bit-exact affine points; host and device I/O; edge scalars"""
    import torch
    from oracle import corelib
    from util import pick_base
    rng = random.Random(61 + group)
    F, base = pick_base(c, group, rng)
    n = 3001
    ks = [rng.randrange(c.r) for _ in range(n)]
    ks[0], ks[1], ks[2] = 0, 1, c.r - 1
    KS = ff.pack_elements(ks, c.r, c.fr_limbs)
    BA = ec.pack_points(c, group, [base])
    want = corelib.fixed_base(c, group, BA, KS)
    got = gpu.fixed_base_batch(c.curve_id, group, BA, KS)
    assert np.array_equal(got.reshape(want.shape), want)
    d_ks = torch.from_numpy(KS.view(np.int64)).cuda()
    d_out = torch.zeros(want.size, dtype=torch.int64, device="cuda")
    gpu.fixed_base_batch(c.curve_id, group, BA, d_ks, n=n, out=d_out)
    assert np.array_equal(d_out.cpu().numpy().view(np.uint64).reshape(want.shape), want)
    assert ec.unpack_points(c, group, got)[2] == ec.scalar_mul(F, c.r - 1, base)


def test_tables_straight_from_a_dump_file(gpu, tmp_path):
    """b200_table_upload_file and the dump_path form of b200_groth16_pk_load (SURVEY.md §8f-1): point slices written the
    way ProvingKey.WriteDump writes them (8-byte little-endian length, then the raw memory image) are read from the file
    into HBM; MSM results and a whole proof must equal those of the in-memory path, also for a point-range shard."""
    import struct
    from gnark_b200 import groth16 as b200
    from oracle import groth16 as g16o
    from util import build_groth16_pk, known_dlog_instance, pack_solution
    c = CURVES["bn254"]
    # 1. one table
    _, _, pts, sc, expected = known_dlog_instance(c, 1, 70000, seed=5)
    f = tmp_path / "slice.bin"
    with open(f, "wb") as fh:
        fh.write(b"HEADER-OF-ANOTHER-KIND" + struct.pack("<Q", 70000))
        off = fh.tell()
        fh.write(np.ascontiguousarray(pts).tobytes())
        fh.write(b"trailer")
    for precomp in (False, True):
        t = gpu.Table.from_file(c.curve_id, 1, str(f), off, 70000, precomp=precomp)
        assert jac_to_affine(c, 1, t.msm(sc)) == expected
        t.free()
    per = 2 * c.fp_limbs * 8
    t = gpu.Table.from_file(c.curve_id, 1, str(f), off + 1000 * per, 3000)                 # a point range of the slice
    want = gpu.Table(c.curve_id, 1, np.ascontiguousarray(pts[1000:4000]))
    sub = np.ascontiguousarray(sc[:3000])
    assert jac_to_affine(c, 1, t.msm(sub)) == jac_to_affine(c, 1, want.msm(sub))
    t.free(); want.free()
    with pytest.raises(gpu.B200Error):
        gpu.Table.from_file(c.curve_id, 1, str(f), off, 70001 + 10)                          # exceeds the file
    # 2. a whole key
    m = 2000
    cs, W = g16o.square_chain_r1cs(m), g16o.square_chain_witness(c.r, m)
    pk, pkd, _, _ = build_groth16_pk(c, cs, g16o.random_toxic(c, 21), 21)
    sol = pack_solution(c, cs, W)
    rs = [111, 222]
    ref = b200.ProveSolution(pk, sol, b200.WithDeviceID(0), b200.WithRandomness(lambda q, it=iter(rs): next(it)))
    dump = tmp_path / "pk.dump"
    offs = {}
    with open(dump, "wb") as fh:
        fh.write(b"marker+domain+alpha..")                                                 # whatever precedes the slices
        for name, arr in (("a", pk.G1_A), ("b", pk.G1_B), ("z", pk.G1_Z), ("k", pk.G1_K), ("b2", pk.G2_B)):
            fh.write(struct.pack("<Q", 0))                                                 # the slice's length prefix
            offs[name] = fh.tell()
            fh.write(np.ascontiguousarray(arr).tobytes())
    pk.use_dump_file(str(dump), offs["a"], offs["b"], offs["z"], offs["k"], offs["b2"])
    got = b200.ProveSolution(pk, sol, b200.WithDeviceID(0), b200.WithRandomness(lambda q, it=iter(rs): next(it)))
    assert np.array_equal(ref.Ar, got.Ar) and np.array_equal(ref.Bs, got.Bs) and np.array_equal(ref.Krs, got.Krs)
    pk.free_gpu_resources()


def test_groth16_with_devices_in_one_process(gpu):
    """WithDevices: every visible GPU holds one point-range shard of the key, the device parts run concurrently from
    one process (what a Go caller does with a goroutine per device); the proof must equal the single-device proof."""
    import torch
    from gnark_b200 import groth16 as b200
    from oracle import groth16 as g16o
    from util import build_groth16_pk, pack_solution
    nd = torch.cuda.device_count()
    if nd < 2:
        pytest.skip("needs at least two GPUs")
    c = CURVES["bn254"]
    m = 3000
    cs, W = g16o.square_chain_r1cs(m), g16o.square_chain_witness(c.r, m)
    pk, pkd, _, _ = build_groth16_pk(c, cs, g16o.random_toxic(c, 17), 17)
    sol = pack_solution(c, cs, W)
    rs = [12345, 67890]
    one = b200.ProveSolution(pk, sol, b200.WithDeviceID(0), b200.WithRandomness(lambda q, it=iter(rs): next(it)))
    many = b200.ProveSolution(pk, sol, b200.WithDevices(*range(nd)), b200.WithRandomness(lambda q, it=iter(rs): next(it)))
    assert np.array_equal(one.Ar, many.Ar) and np.array_equal(one.Bs, many.Bs) and np.array_equal(one.Krs, many.Krs)
    pk.free_gpu_resources()


def test_groth16_threaded_staging_of_pageable_inputs(gpu):
    """GB200_STAGE_THREADS: W, A, B, C uploaded from pageable memory through two pinned slots filled by several
    threads; the proof must be identical to the plain path (domain 2^18 so that the vectors exceed the 4 MiB
    threshold and span several 16 MiB slots... 8 MiB each: one slot, ragged)"""
    import subprocess
    import sys
    code = r'''
import os, sys, random
import numpy as np
sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
from gnark_b200 import groth16 as b200
from oracle import groth16 as g16
from oracle.params import CURVES
from util import build_groth16_pk, pack_solution
c = CURVES["bn254"]
m = (1 << 18) - 5
cs, W = g16.square_chain_r1cs(m), g16.square_chain_witness(c.r, m)
pk, pkd, _, _ = build_groth16_pk(c, cs, g16.random_toxic(c, 9), 9)
sol = pack_solution(c, cs, W)
outs = []
for threads in ("0", "4"):
    os.environ["GB200_STAGE_THREADS"] = threads   # read once per process: the second value needs a fresh process
    it = iter([123456789, 987654321])
    p = b200.ProveSolution(pk, sol, b200.WithDeviceID(0), b200.WithRandomness(lambda q: next(it)), keep_msm=True)
    outs.append(np.concatenate([p.msm, p.Ar.reshape(-1), p.Bs.reshape(-1), p.Krs.reshape(-1)]))
print("EQUAL" if np.array_equal(outs[0], outs[1]) else "DIFFERENT")
'''
    # the knob is latched at first use, so each setting runs in its own interpreter and prints a digest
    res = {}
    for threads in ("0", "4"):
        env = dict(os.environ, GB200_STAGE_THREADS=threads)
        body = code.replace('for threads in ("0", "4"):', 'for threads in ("%s",):' % threads).replace(
            'print("EQUAL" if np.array_equal(outs[0], outs[1]) else "DIFFERENT")',
            'import hashlib; print("DIGEST", hashlib.sha256(outs[0].tobytes()).hexdigest())')
        out = subprocess.run([sys.executable, "-c", body], env=env, capture_output=True, text=True, timeout=900,
                             cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        assert out.returncode == 0, out.stderr[-2000:]
        res[threads] = [ln for ln in out.stdout.splitlines() if ln.startswith("DIGEST")][0]
    assert res["0"] == res["4"]
