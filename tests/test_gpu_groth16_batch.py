"""Batched Groth16 proving (b200_groth16_prove_batch, gnark_b200.groth16.ProveSolutionBatch) and the batched NTT
(b200_ntt_batch).  Each proof of a batch is checked against the big-int oracle's discrete logs (five MSM results and
three proof points), against the pairing, and byte for byte against b200_groth16_prove of the same witness and r, s.

The first tests need no GPU: the strided batch decompose emulated on the CPU, and the Python wrapper against a fake C
library (pointer arrays, the order r0, s0, r1, s1, ..., how the outputs become Proofs, the refusals)."""
import ctypes
import dataclasses
import os
import random
import subprocess

import numpy as np
import pytest

from oracle import ec, ff
from oracle import groth16 as g16
from oracle.params import CURVES
from util import build_groth16_pk, jac_to_affine, pack_solution

ALL = list(CURVES.values())
BN254 = CURVES["bn254"]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- CPU: the strided batch decompose ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def strideemu():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "gnark_b200", "csrc"), "../../tests/_build/libgb200_msmstrideemu.so"])
    lib = ctypes.CDLL(os.path.join(ROOT, "tests", "_build", "libgb200_msmstrideemu.so"))
    u32, i, vp = ctypes.c_uint32, ctypes.c_int, ctypes.c_void_p
    lib.emu_decompose_batch.argtypes = [i, u32, u32, vp, u32, u32, u32, i, i, i, vp, vp]
    return lib


def _decompose(lib, curve, sc, n, batch, stride, c, precomp, back_to_back):
    nwin = curve.r.bit_length() // c + 1
    keys = np.full(n * batch * nwin, 7, dtype=np.uint32)
    vals = np.full_like(keys, 7)
    P = lambda a: a.ctypes.data
    assert lib.emu_decompose_batch(curve.curve_id, 1000, 3, P(sc), n, batch, stride, c, precomp, back_to_back,
                                   P(keys), P(vals)) == 0
    return keys, vals


def _scalars(curve, count, rng):
    return ff.pack_elements([rng.randrange(curve.r) for _ in range(count)], curve.r, curve.fr_limbs)


@pytest.mark.parametrize("precomp", (0, 1), ids=("plain", "precomp"))
@pytest.mark.parametrize("curve", ALL, ids=lambda c: c.name)
def test_strided_decompose_emulated(strideemu, curve, precomp):
    """stride = n: exactly the entries of the items read back to back; stride > n: exactly the entries of the
    compacted scalars (the first n of every stride-long row), whatever the rows hold past n"""
    rng = random.Random(f"stride-{curve.name}-{precomp}")
    for c in (4, 7):
        for n, batch in ((1, 5), (37, 3), (64, 4)):
            sc = _scalars(curve, n * batch, rng)
            want = _decompose(strideemu, curve, sc, n, batch, 0, c, precomp, back_to_back=1)
            assert all(np.array_equal(x, y) for x, y in zip(_decompose(strideemu, curve, sc, n, batch, n, c, precomp, 0), want))
            for stride in (n + 1, 2 * n + 3):
                rows = _scalars(curve, stride * batch, rng).reshape(batch, stride, -1)
                compact = np.ascontiguousarray(rows[:, :n]).reshape(n * batch, -1)
                want = _decompose(strideemu, curve, compact, n, batch, 0, c, precomp, back_to_back=1)
                got = _decompose(strideemu, curve, np.ascontiguousarray(rows), n, batch, stride, c, precomp, 0)
                assert all(np.array_equal(x, y) for x, y in zip(got, want)), (curve.name, c, n, batch, stride)


# ---- CPU: the Python wrapper against a fake C library ------------------------------------------------------------------
class _FakeC:
    def __init__(self, frl, fpl, deg):
        self.frl, self.fpl, self.deg = frl, fpl, deg
        self.calls = []

    def b200_groth16_pk_load(self, dev, desc_ref, out_ref):
        out_ref._obj.value = 42
        self.calls.append(("load", dev, desc_ref._obj.shard_world))
        return 0

    def b200_groth16_pk_free(self, h):
        return 0

    def b200_groth16_prove_batch(self, h, k, w, a, b, c, n, r, s, ar, bs, krs, msm):
        u64 = lambda p, count: np.ctypeslib.as_array((ctypes.c_uint64 * count).from_address(p.value))
        frl, fpl, deg = self.frl, self.fpl, self.deg
        self.calls.append(("prove_batch", h.value, k, n, [w[i] for i in range(k)], [a[i] for i in range(k)],
                           [b[i] for i in range(k)], [c[i] for i in range(k)],
                           u64(r, k * frl).copy(), u64(s, k * frl).copy()))
        for i in range(k):                 # recognisable outputs: item i's words hold i + 1 (Ar), 100 + i, 200 + i
            u64(ar, k * 2 * fpl)[i * 2 * fpl:(i + 1) * 2 * fpl] = i + 1
            u64(bs, k * 2 * fpl * deg)[i * 2 * fpl * deg:(i + 1) * 2 * fpl * deg] = 100 + i
            u64(krs, k * 2 * fpl)[i * 2 * fpl:(i + 1) * 2 * fpl] = 200 + i
            if msm.value:
                per = 4 * 3 * fpl + 3 * fpl * deg
                u64(msm, k * per)[i * per:(i + 1) * per] = 300 + i
        return 0


class _FakeLib:
    def __init__(self):
        from gnark_b200 import lib as real
        self.real = real
        self.CURVE_SHAPES, self.TABLE_PRECOMP, self.Groth16PkDesc = real.CURVE_SHAPES, real.TABLE_PRECOMP, real.Groth16PkDesc
        self.c = _FakeC(*real.CURVE_SHAPES[real.BN254])

    def load(self):
        return self.c

    def ptr(self, a):
        return self.real.ptr(a)

    @staticmethod
    def check(rc):
        assert rc == 0


@pytest.fixture
def fake(monkeypatch):
    from gnark_b200 import groth16 as b200
    f = _FakeLib()
    monkeypatch.setattr(b200, "_lib", f)
    return f


def _fake_key_and_solutions(k, n_constraints=3):
    from gnark_b200 import groth16 as b200
    from gnark_b200 import lib as real
    frl, fpl, deg = real.CURVE_SHAPES[real.BN254]
    z = lambda n: np.zeros(n, dtype=np.uint64)
    nb_wires = 5
    pk = b200.ProvingKey.from_arrays(real.BN254, 4, z(2 * fpl), z(2 * fpl), z(2 * fpl), z(2 * fpl * nb_wires),
                                     z(2 * fpl * nb_wires), z(2 * fpl * 3), z(2 * fpl * 3), z(2 * fpl * deg),
                                     z(2 * fpl * deg), z(2 * fpl * deg * nb_wires), [0] * nb_wires, [0] * nb_wires, 2)
    sols = [b200.R1CSSolution(W=np.full(frl * nb_wires, i, dtype=np.uint64), A=z(frl * n_constraints),
                              B=z(frl * n_constraints), C=z(frl * n_constraints)) for i in range(k)]
    return pk, sols


def test_wrapper_passes_pointer_arrays_and_splits_outputs(fake):
    from gnark_b200 import groth16 as b200
    pk, sols = _fake_key_and_solutions(3)
    draws = iter(range(1, 7))
    proofs = b200.ProveSolutionBatch(pk, sols, b200.WithRandomness(lambda q: next(draws)), keep_msm=True)
    assert fake.c.calls[0] == ("load", 0, 1)
    _, h, k, n, w, a, b, c, r, s = fake.c.calls[1]
    assert (h, k, n) == (42, 3, 3)
    assert w == [sol.W.ctypes.data for sol in sols]              # the solutions' own buffers, not a copy
    assert a == [sol.A.ctypes.data for sol in sols] and b == [sol.B.ctypes.data for sol in sols]
    assert c == [sol.C.ctypes.data for sol in sols]
    # WithRandomness is drawn r0, s0, r1, s1, r2, s2
    mont = lambda x: b200._fr_to_mont_limbs(x, b200.BN254)
    assert np.array_equal(r.reshape(3, -1), np.stack([mont(1), mont(3), mont(5)]))
    assert np.array_equal(s.reshape(3, -1), np.stack([mont(2), mont(4), mont(6)]))
    assert len(proofs) == 3
    for i, p in enumerate(proofs):
        assert (p.Ar == i + 1).all() and (p.Bs == 100 + i).all() and (p.Krs == 200 + i).all() and (p.msm == 300 + i).all()
    assert b200.ProveSolutionBatch(pk, []) == []

    class Solver:
        def Solve(self, w):
            return sols[w]
    assert len(b200.ProveBatch(Solver(), pk, [2, 0], b200.WithRandomness(lambda q: 9))) == 2
    assert fake.c.calls[-1][4] == [sols[2].W.ctypes.data, sols[0].W.ctypes.data]


def test_wrapper_refusals(fake):
    from gnark_b200 import groth16 as b200
    pk, sols = _fake_key_and_solutions(2)
    with pytest.raises(ValueError):
        b200.ProveSolutionBatch(pk, sols, b200.WithDevices(0, 1))
    with pytest.raises(ValueError):
        b200.ProveSolutionBatch(pk, sols, b200.WithSharding(0, 2))
    bad = dataclasses.replace(sols[1], W=sols[1].W[:-1])
    with pytest.raises(ValueError, match="witness size"):
        b200.ProveSolutionBatch(pk, [sols[0], bad])
    _, other = _fake_key_and_solutions(1, n_constraints=2)
    with pytest.raises(ValueError, match="constraint counts"):
        b200.ProveSolutionBatch(pk, [sols[0], other[0]])
    assert not [c for c in fake.c.calls if c[0] == "prove_batch"]


# ---- GPU ----------------------------------------------------------------------------------------------------------------
def _check_item(c, cs, pkd, g1, g2, W, rr, ss, proof, pairing):
    F1, F2 = ff.Fp(c.p), ff.base_field(c, 2)
    want = g16.prove_dlog(c, cs, pkd, W, rr, ss)
    L = 3 * c.fp_limbs
    m = proof.msm
    for k, dlog in enumerate((want.msm_a, want.msm_b, want.msm_z, want.msm_k)):
        assert ec.from_jac(F1, ec.unpack_points(c, 1, m[k * L:(k + 1) * L], ncoords=3)[0]) == ec.scalar_mul(F1, dlog, g1), k
    assert ec.from_jac(F2, ec.unpack_points(c, 2, m[4 * L:], ncoords=3)[0]) == ec.scalar_mul(F2, want.msm_b, g2)
    ar, bs, krs = (ec.unpack_points(c, 1, proof.Ar)[0], ec.unpack_points(c, 2, proof.Bs)[0],
                   ec.unpack_points(c, 1, proof.Krs)[0])
    assert ar == ec.scalar_mul(F1, want.ar, g1)
    assert bs == ec.scalar_mul(F2, want.bs, g2)
    assert krs == ec.scalar_mul(F1, want.krs, g1)
    if pairing:
        assert g16.verify_pairing(c, pkd, ar, bs, krs, W)


def _randomness(c, k, seed):
    rng = random.Random(repr(seed))
    return [rng.randrange(1, c.r) for _ in range(2 * k)]


def _prove_batch(pk, sols, rs, precomp=True, keep_msm=True):
    from gnark_b200 import groth16 as b200
    it = iter(rs)
    return b200.ProveSolutionBatch(pk, sols, b200.WithDeviceID(0), b200.WithPrecompute(precomp),
                                   b200.WithRandomness(lambda q: next(it)), keep_msm=keep_msm)


@pytest.mark.gpu
@pytest.mark.parametrize("precomp", (False, True), ids=("plain", "precomp"))
@pytest.mark.parametrize("c", ALL, ids=lambda c: c.name)
def test_batch_against_dlogs(gpu, c, precomp):
    """cubic and square-chain circuits, k = 1, 2, 5, 33 distinct witnesses: every item's five MSM results and three
    proof points equal prove_dlog; on BN254 and BLS12-381 the pairing equation holds (every item of the small batches,
    the first and last of 33)"""
    m = 200
    for cs, wit, seed in ((g16.cubic_r1cs(), lambda x: g16.cubic_witness(c.r, x), 21),
                          (g16.square_chain_r1cs(m), lambda x: g16.square_chain_witness(c.r, m, x0=x), 22)):
        pk, pkd, (F1, g1), (F2, g2) = build_groth16_pk(c, cs, g16.random_toxic(c, seed), seed)
        for k in (1, 2, 5, 33):
            Ws = [wit(3 + 7 * i) for i in range(k)]
            rs = _randomness(c, k, (seed, k))
            proofs = _prove_batch(pk, [pack_solution(c, cs, W) for W in Ws], rs, precomp)
            assert len(proofs) == k
            for i, (W, p) in enumerate(zip(Ws, proofs)):
                pairing = c.name in ("bn254", "bls12-381") and (k <= 5 or i in (0, k - 1))
                _check_item(c, cs, pkd, g1, g2, W, rs[2 * i], rs[2 * i + 1], p, pairing)
        pk.free_gpu_resources()


def _msm_affine(c, msm):
    L = 3 * c.fp_limbs
    return [jac_to_affine(c, 1, msm[k * L:(k + 1) * L]) for k in range(4)] + [jac_to_affine(c, 2, msm[4 * L:])]


@pytest.mark.gpu
@pytest.mark.parametrize("m", (1000, 1024), ids=("padded", "full-domain"))
def test_batch_equals_single_proofs(gpu, m):
    """with the same r, s, item b's Ar, Bs, Krs are byte-identical to b200_groth16_prove of witness b and its five MSM
    results the same points, at k = 3 and k = 1, with n_constraints < n and = n; identical witnesses in one batch give
    equal MSM results"""
    from gnark_b200 import groth16 as b200
    c = BN254
    cs = g16.square_chain_r1cs(m)
    pk, pkd, (F1, g1), (F2, g2) = build_groth16_pk(c, cs, g16.random_toxic(c, 31), 31)
    assert (m < pk.domain_size) == (m == 1000)
    sols = [pack_solution(c, cs, g16.square_chain_witness(c.r, m, x0=5 + i)) for i in range(3)]
    for k in (3, 1):
        rs = _randomness(c, k, ("eq", m, k))
        batch = _prove_batch(pk, sols[:k], rs)
        for i in range(k):
            it = iter(rs[2 * i:2 * i + 2])
            one = b200.ProveSolution(pk, sols[i], b200.WithDeviceID(0), b200.WithRandomness(lambda q: next(it)),
                                     keep_msm=True)
            for f in ("Ar", "Bs", "Krs"):
                assert np.array_equal(getattr(batch[i], f), getattr(one, f)), (k, i, f)
            # the MSM results are the same points; their Jacobian coordinates may differ (the batch groups the bucket
            # entries into tasks of another length)
            assert _msm_affine(c, batch[i].msm) == _msm_affine(c, one.msm), (k, i)
    same = _prove_batch(pk, [sols[0]] * 4, _randomness(c, 4, "same"))
    assert all(np.array_equal(p.msm, same[0].msm) for p in same[1:])
    pk.free_gpu_resources()


@pytest.mark.gpu
def test_batch_committed_wires_filtered_from_k(gpu):
    """a key with committed private wires (the K scalars go through the batched gather): every item's K MSM is the
    sum over the remaining private wires, the other four MSMs are unchanged"""
    from gnark_b200 import groth16 as b200
    c = BN254
    m_ = 300
    cs = g16.square_chain_r1cs(m_)
    pk, pkd, (F1, g1), (F2, g2) = build_groth16_pk(c, cs, g16.random_toxic(c, 3), 3)
    rng = random.Random(3)
    nb_pub, nb_wires = cs.nb_public, pk.nb_wires
    removed = sorted(rng.sample(range(nb_pub, nb_wires), 17))
    keep = [i for i in range(nb_pub, nb_wires) if i not in set(removed)]
    K_full = pk.G1_K.reshape(-1, 2 * c.fp_limbs)
    pk2 = b200.ProvingKey.from_arrays(
        c.curve_id, pk.domain_size, pk.G1_Alpha, pk.G1_Beta, pk.G1_Delta, pk.G1_A, pk.G1_B, pk.G1_Z,
        np.ascontiguousarray(K_full[[i - nb_pub for i in keep]]), pk.G2_Beta, pk.G2_Delta, pk.G2_B, pk.InfinityA,
        pk.InfinityB, nb_pub, committed_private_wires=removed)
    Ws = [g16.square_chain_witness(c.r, m_, x0=4 + i) for i in range(4)]
    rs = _randomness(c, 4, "committed")
    proofs = _prove_batch(pk2, [pack_solution(c, cs, W) for W in Ws], rs)
    Lj = 3 * c.fp_limbs
    for W, rr, ss, p in zip(Ws, rs[0::2], rs[1::2], proofs):
        want = g16.prove_dlog(c, cs, pkd, W, rr, ss)
        for k, dlog in ((0, want.msm_a), (1, want.msm_b), (2, want.msm_z)):
            assert ec.from_jac(F1, ec.unpack_points(c, 1, p.msm[k * Lj:(k + 1) * Lj], ncoords=3)[0]) == ec.scalar_mul(F1, dlog, g1)
        k_dlog = sum(W[i] * pkd.K[i - nb_pub] for i in keep) % c.r
        assert ec.from_jac(F1, ec.unpack_points(c, 1, p.msm[3 * Lj:4 * Lj], ncoords=3)[0]) == ec.scalar_mul(F1, k_dlog, g1)
    pk2.free_gpu_resources()
    pk.free_gpu_resources()


@pytest.mark.gpu
def test_batch_full_size(gpu):
    """BN254 2^20, k = 4: the witnesses of satisfied_instance at four seeds on the key of the first; every proof passes
    the verifier's equation with a real pairing"""
    from gnark_b200 import groth16 as b200
    from oracle import groth16_fast as gf
    c = BN254
    seeds = (40, 41, 42, 43)
    inst0 = gf.satisfied_instance(c, 20, seed=seeds[0])
    fb = lambda group, dl: gpu.fixed_base_batch(c.curve_id, group, ec.pack_points(c, group, [c.g1 if group == 1 else c.g2]),
                                                np.ascontiguousarray(dl))
    kp = gf.key_points(inst0, fb)
    pk = b200.ProvingKey.from_arrays(c.curve_id, inst0.n, kp["alpha"], kp["beta"], kp["delta"], kp["A"], kp["B"], kp["Z"],
                                     kp["K"], kp["beta2"], kp["delta2"], kp["B2"], inst0.inf_a, inst0.inf_b, inst0.nb_public)
    insts = [inst0] + [dataclasses.replace(inst0, v=gf.satisfied_instance(c, 20, seed=s).v) for s in seeds[1:]]
    sols = []
    for inst in insts:
        assert gf.check_satisfied(inst)
        a, b, cc = inst.solution_abc()
        sols.append(b200.R1CSSolution(W=inst.wires(), A=a, B=b, C=cc))
    rs = _randomness(c, 4, "full")
    proofs = _prove_batch(pk, sols, rs, keep_msm=False)
    for inst, rr, ss, p in zip(insts, rs[0::2], rs[1::2], proofs):
        e = gf.expected(inst, rr, ss)
        assert gf.verify_points(inst, ec.unpack_points(c, 1, p.Ar)[0], ec.unpack_points(c, 2, p.Bs)[0],
                                ec.unpack_points(c, 1, p.Krs)[0], e, with_pairing=True)
    pk.free_gpu_resources()


@pytest.mark.gpu
def test_batch_after_other_work(gpu):
    """a batch enqueued after pipelined MSMs that were not joined, and a batch right after a single prove on the same
    key, both give the oracle's proofs (and the pipelined MSMs theirs)"""
    import torch
    from gnark_b200 import groth16 as b200
    c = BN254
    m = 500
    cs = g16.square_chain_r1cs(m)
    pk, pkd, (F1, g1), (F2, g2) = build_groth16_pk(c, cs, g16.random_toxic(c, 51), 51)
    Ws = [g16.square_chain_witness(c.r, m, x0=9 + i) for i in range(3)]
    sols = [pack_solution(c, cs, W) for W in Ws]
    # pipelined MSMs over the key's own A points, left unjoined
    rng = random.Random(5)
    pts = np.ascontiguousarray(pk.G1_A.reshape(-1, 2 * c.fp_limbs)[:256])
    t = gpu.Table(c.curve_id, 1, pts)
    scs = [ff.pack_elements([rng.randrange(c.r) for _ in range(256)], c.r, c.fr_limbs) for _ in range(3)]
    d_sc = [torch.from_numpy(s.view(np.int64)).cuda() for s in scs]
    d_out = [torch.zeros(3 * c.fp_limbs, dtype=torch.int64, device="cuda") for _ in scs]
    torch.cuda.synchronize()
    for s, o in zip(d_sc, d_out):
        t.msm_pipelined(s, o, n=256)
    rs = _randomness(c, 3, "after-msm")
    proofs = _prove_batch(pk, sols, rs)
    for W, rr, ss, p in zip(Ws, rs[0::2], rs[1::2], proofs):
        _check_item(c, cs, pkd, g1, g2, W, rr, ss, p, pairing=False)
    t.join()
    gpu.sync(0)
    for s, o in zip(scs, d_out):
        assert jac_to_affine(c, 1, o.cpu().numpy().view(np.uint64)) == jac_to_affine(c, 1, t.msm(s))
    t.free()
    # a single prove, then a batch on the same key
    it = iter(rs[:2])
    b200.ProveSolution(pk, sols[0], b200.WithDeviceID(0), b200.WithRandomness(lambda q: next(it)))
    proofs = _prove_batch(pk, sols, rs)
    for W, rr, ss, p in zip(Ws, rs[0::2], rs[1::2], proofs):
        _check_item(c, cs, pkd, g1, g2, W, rr, ss, p, pairing=False)
    pk.free_gpu_resources()


@pytest.mark.gpu
def test_batch_refusals(gpu):
    """null arguments, a sharded key, n_constraints > n and a batch past the device indices are refused before anything
    runs, with every output untouched; batch = 0 writes nothing"""
    from gnark_b200 import groth16 as b200
    c = BN254
    m = 1000
    cs = g16.square_chain_r1cs(m)
    pk, pkd, _, _ = build_groth16_pk(c, cs, g16.random_toxic(c, 61), 61)
    pk.setup_device_pointers(b200.NewConfig(b200.WithDeviceID(0)))
    L = gpu.load()
    k = 2
    sols = [pack_solution(c, cs, g16.square_chain_witness(c.r, m, x0=3 + i)) for i in range(k)]
    arr = lambda name: (ctypes.c_void_p * k)(*[getattr(s, name).ctypes.data for s in sols])
    W, A, B, C = arr("W"), arr("A"), arr("B"), arr("C")
    rs = np.stack([b200._fr_to_mont_limbs(x, c.curve_id) for x in _randomness(c, k, "refuse")])
    r, s = np.ascontiguousarray(rs[0::2]), np.ascontiguousarray(rs[1::2])
    fpl, deg = c.fp_limbs, 2
    outs = [np.full(k * 2 * fpl, 7, dtype=np.uint64), np.full(k * 2 * fpl * deg, 7, dtype=np.uint64),
            np.full(k * 2 * fpl, 7, dtype=np.uint64), np.full(k * (12 * fpl + 3 * fpl * deg), 7, dtype=np.uint64)]
    P = gpu.ptr
    null = ctypes.c_void_p(0)

    def call(h, batch=k, w=W, a=A, n=m, rp=r, ar=None):
        return L.b200_groth16_prove_batch(h, batch, w, a, B, C, n, P(rp), P(s), ar if ar is not None else P(outs[0]),
                                          P(outs[1]), P(outs[2]), P(outs[3]))

    def fails(match, rc):
        assert rc != 0
        assert match in L.b200_last_error().decode(), L.b200_last_error()
        assert all((o == 7).all() for o in outs), "an output was written"

    fails("prove_batch: null proving key", call(null))
    fails("prove_batch: null argument", call(pk._handle, w=None))
    fails("prove_batch: null argument", call(pk._handle, rp=None))
    fails("prove_batch: null argument", call(pk._handle, ar=null))
    holed = (ctypes.c_void_p * k)(A[0], None)
    fails("prove_batch: null witness vector of item 1", call(pk._handle, a=holed))
    fails("prove_batch: more constraints than the domain holds", call(pk._handle, n=pk.domain_size + 1))
    # the largest batch the key takes, then one more: refused before any item pointer is read
    rc = call(pk._handle, batch=1 << 40)
    msg = L.b200_last_error().decode()
    fails("the largest batch this key takes is", rc)
    fits = int(msg.rsplit(" ", 1)[1])
    assert 0 < fits < (1 << 31)
    fails(f"a batch of {fits + 1} proofs exceeds", call(pk._handle, batch=fits + 1))
    gpu.check(call(pk._handle, batch=0))
    assert all((o == 7).all() for o in outs)
    # a sharded key
    sh = pk._load(0, 0, 2, True)
    fails("prove_batch: sharded keys are not supported", call(sh))
    gpu.check(call(pk._handle))                                  # a valid call still works
    assert not (outs[0] == 7).all()
    pk.free_gpu_resources()


# ---- GPU: b200_ntt_batch -----------------------------------------------------------------------------------------------
MODES = [(inv, dec, cos) for inv in (False, True) for dec in (0, 1) for cos in (False, True)]


def _random_fr(c, count, rng):
    x = rng.integers(0, 1 << 63, size=(count, c.fr_limbs), dtype=np.uint64)
    x[:, c.fr_limbs - 1] &= np.uint64((1 << 56) - 1)             # < r: valid Montgomery residues
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("c", ALL, ids=lambda c: c.name)
def test_ntt_batch_matches_single(gpu, c):
    """every inverse x decimation x coset mode: batches of 1, 3 and 70 000 at 2^4 (past a grid's 65 535 rows), 4 x 2^20,
    and the n = 1 domain, on host data; 3 x 2^10 on device data.  Every vector equals b200_ntt of it (for 70 000: the
    vectors around the split and at the ends)"""
    import torch
    rng = np.random.default_rng(c.curve_id)
    L = c.fr_limbs
    cases = [(4, 1, None), (4, 3, None), (4, 70000, [0, 1, 65534, 65535, 65536, 69999]), (20, 4, None), (0, 5, None)]
    for logn, batch, check in cases:
        d = gpu.Domain(c.curve_id, logn)
        n = 1 << logn
        x = _random_fr(c, batch * n, rng)
        for inv, dec, cos in MODES:
            got = d.ntt_batch(x.copy(), inverse=inv, decimation=dec, on_coset=cos).reshape(batch, n, L)
            for b in (check if check is not None else range(batch)):
                want = d.ntt(np.ascontiguousarray(x[b * n:(b + 1) * n]), inverse=inv, decimation=dec, on_coset=cos)
                assert np.array_equal(got[b], want.reshape(n, L)), (logn, batch, b, inv, dec, cos)
        d.free()
    d = gpu.Domain(c.curve_id, 10)
    x = _random_fr(c, 3 * 1024, rng)
    for inv, dec, cos in MODES:
        t = torch.from_numpy(x.view(np.int64).reshape(-1).copy()).cuda()
        torch.cuda.synchronize()
        d.ntt_batch(t, inverse=inv, decimation=dec, on_coset=cos, on_device=True)
        got = t.cpu().numpy().view(np.uint64).reshape(3, 1024, L)
        for b in range(3):
            want = d.ntt(np.ascontiguousarray(x[b * 1024:(b + 1) * 1024]), inverse=inv, decimation=dec, on_coset=cos)
            assert np.array_equal(got[b], want.reshape(1024, L)), (b, inv, dec, cos)
    # batch = 0 does nothing
    gpu.check(gpu.load().b200_ntt_batch(d.handle, None, 0, 0, 0, 0, 0))
    d.free()
