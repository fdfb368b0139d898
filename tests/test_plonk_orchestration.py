"""The ORCHESTRATION of the device PLONK prover (gnark_b200/plonk.py) on the CPU: every C-ABI call the
orchestrator makes is replaced by a mock that computes the same documented result with the big-int oracle
on host tensors, so what is exercised here is the stage order, layouts (regular / bit-reversed), blinding
patches, coset handles, slice arithmetic and the linearised-polynomial / batch-opening algebra of
backend/plonk/bn254/prove.go:404-837 - against oracle/plonk_prover.py with the same injected challenges.

The C-ABI entry points themselves are pinned on hardware by tests/test_gpu_plonk.py; the two together are
what tests/test_gpu_zz_late.py::test_full_prover_vs_oracle checks in one piece on an H100.  Nothing here is a
product code path: the mock lives in this test file only.
"""
import contextlib
import random
import types

import numpy as np
import pytest

from oracle import corelib, ec, ff, ntt, plonk, plonk_prover as pp
from oracle.params import CURVES
from util import jac_to_affine

BY_ID = {c.curve_id: c for c in CURVES.values()}


def _ints(c, t, count=None):
    a = t.detach().cpu().numpy().reshape(-1).view(np.uint64)
    if count is not None:
        a = a[:count * c.fr_limbs]
    return ff.unpack_elements(a, c.r, c.fr_limbs)


def _store(c, t, vals, offset=0):
    import torch
    a = ff.pack_elements(vals, c.r, c.fr_limbs).reshape(-1).view(np.int64)
    flat = t.view(-1)
    flat[offset * c.fr_limbs:offset * c.fr_limbs + a.size] = torch.from_numpy(a.copy())


def _scalar(c, a):
    return ff.unpack_elements(np.ascontiguousarray(a, dtype=np.uint64), c.r, c.fr_limbs)[0]


def make_mock_lib(real_lib, calls):
    m = types.SimpleNamespace()
    for k in ("BN254", "BLS12_381", "BLS12_377", "BW6_761", "CURVE_SHAPES", "DIF", "DIT"):
        setattr(m, k, getattr(real_lib, k))

    class Domain:
        def __init__(self, curve, log2n, dev=0, generator=None, coset_gen=None):
            self.c = BY_ID[curve]
            self.curve, self.log2n, self.n, self.dev = curve, log2n, 1 << log2n, dev
            self.fr_limbs = self.c.fr_limbs
            self.o = ntt.Domain(self.c, self.n, coset_gen=None if coset_gen is None else _scalar(self.c, coset_gen))

        def ntt_async(self, d, inverse=False, decimation=0, on_coset=False):
            calls.append("ntt")
            a = _ints(self.c, d, self.n)
            out = (self.o.fft_inverse if inverse else self.o.fft)(a, decimation, on_coset=on_coset)
            _store(self.c, d, out)

        def free(self):
            pass

    class Table:
        def __init__(self, curve, group, points, dev=0, precomp=True, n=None, on_device=False):
            self.c, self.group, self.points = BY_ID[curve], group, np.ascontiguousarray(points)

        def msm(self, scalars, off=0, n=None, on_device=False):
            calls.append("msm")
            assert on_device and off == 0
            sc = scalars.detach().cpu().numpy().reshape(-1).view(np.uint64)[:n * self.c.fr_limbs].copy()
            pts = self.points.reshape(-1)[:n * 2 * self.c.fp_limbs].copy()
            return corelib.msm(self.c, self.group, pts, sc, n=n, c=4).reshape(-1)

        def free(self):
            pass

    def vec_bit_reverse(dev, curve, d, log2n):
        c = BY_ID[curve]
        _store(c, d, ntt.bit_reverse(_ints(c, d, 1 << log2n)))

    def plonk_build_z(dom0, d_l, d_r, d_o, d_perm, beta, gamma, d_z):
        c = dom0.c
        z = plonk.build_ratio_copy_constraint(c, dom0.o, _ints(c, d_l), _ints(c, d_r), _ints(c, d_o),
                                              [int(x) for x in d_perm.tolist()], _scalar(c, beta), _scalar(c, gamma))
        _store(c, d_z, z)

    def plonk_constraints_coset(dom0, big_coset_gen, big_gen, polys, alpha, beta, gamma, blind, coset_index, rho, d_out):
        """documented result of b200_plonk_constraints_coset: allConstraints (prove.go:968-1001) at the n points of
        coset g*w4^i, inputs already ON that coset, written to cres[bitrev(rho*j + i)]"""
        calls.append("constraints")
        c, n, r = dom0.c, dom0.n, dom0.c.r
        g, w4 = _scalar(c, big_coset_gen), _scalar(c, big_gen)
        coset = g * pow(w4, coset_index, r) % r
        assert dom0.o.coset_gen == coset, "constraint call on a domain handle of another coset"
        vals = {k: _ints(c, polys[k], n) for k in plonk.POLYS}
        bl = {k: ([] if blind.get(k) is None else ff.unpack_elements(blind[k], r, c.fr_limbs)) for k in ("l", "r", "o", "z")}
        w = dom0.o.generator
        xn1 = (pow(coset, n, r) - 1) % r
        logm = (rho * n).bit_length() - 1
        for j in range(n):
            u = {k: vals[k][j] for k in plonk.POLYS}
            u["zs"] = vals["z"][(j + 1) % n]
            x, x1 = coset * pow(w, j, r) % r, coset * pow(w, (j + 1) % n, r) % r
            v = plonk.all_constraints(r, n, dom0.o.cardinality_inv, u, x, x1, _scalar(c, alpha), _scalar(c, beta),
                                      _scalar(c, gamma), g, bl, xn1)
            _store(c, d_out, [v], offset=ntt.bitrev(rho * j + coset_index, logm))

    def plonk_bsb22_coset(dom0, d_qcp, d_pi2, coset_index, rho, d_out):
        """documented result of b200_plonk_bsb22_coset: out[slot of point j] += qcp[j] * pi2[j]"""
        calls.append("bsb22")
        c, n = dom0.c, dom0.n
        qv, pv = _ints(c, d_qcp, n), _ints(c, d_pi2, n)
        logm = (rho * n).bit_length() - 1
        cur = _ints(c, d_out, rho * n)
        for j in range(n):
            k = ntt.bitrev(rho * j + coset_index, logm)
            _store(c, d_out, [(cur[k] + qv[j] * pv[j]) % c.r], offset=k)

    def plonk_divide_by_zh(dom1, domain0_log2n, d):
        c = dom1.c
        n = 1 << domain0_log2n
        _store(c, d, plonk.divide_by_zh(c, n, dom1.n // n, _ints(c, d, dom1.n)))

    def poly_eval(dev, curve, d, n, x):
        c = BY_ID[curve]
        return ff.pack_elements([ntt.poly_eval(c.r, _ints(c, d, n), _scalar(c, x))], c.r, c.fr_limbs).reshape(-1)

    def poly_div_by_linear(dev, curve, d, n, z):
        c = BY_ID[curve]
        q_, rem = plonk.div_by_linear(c.r, _ints(c, d, n), _scalar(c, z))
        _store(c, d, q_ + [0])          # b200_poly_div_by_linear: quotient in [0, n-1), top slot cleared
        return ff.pack_elements([rem], c.r, c.fr_limbs).reshape(-1)

    def vec_axpy(dev, curve, d_y, a, d_x, n):
        c = BY_ID[curve]
        s = _scalar(c, a)
        y, x = _ints(c, d_y, n), _ints(c, d_x, n)
        _store(c, d_y, [(yy + s * xx) % c.r for yy, xx in zip(y, x)])

    def vec_scale_powers(dev, curve, d, n, s_mont, g_mont):
        c = BY_ID[curve]
        s_, g_ = _scalar(c, s_mont), _scalar(c, g_mont)
        _store(c, d, [x * s_ * pow(g_, i, c.r) % c.r for i, x in enumerate(_ints(c, d, n))])

    def vec_op(dev, curve, op, d_out, d_a, d_b, n):
        c = BY_ID[curve]
        a, b = _ints(c, d_a, n), _ints(c, d_b, n)
        f = (lambda x, y: x * y, lambda x, y: x + y, lambda x, y: x - y)[op]
        _store(c, d_out, [f(x, y) % c.r for x, y in zip(a, b)])

    m.vec_scale_powers, m.vec_op = vec_scale_powers, vec_op
    m.plonk_bsb22_coset = plonk_bsb22_coset
    m.Domain, m.Table = Domain, Table
    m.vec_bit_reverse, m.plonk_build_z, m.plonk_constraints_coset = vec_bit_reverse, plonk_build_z, plonk_constraints_coset
    m.plonk_divide_by_zh, m.poly_eval, m.poly_div_by_linear, m.vec_axpy = plonk_divide_by_zh, poly_eval, poly_div_by_linear, vec_axpy
    m.set_stream = lambda dev, s: calls.append(("set_stream", s))
    m.sync = lambda dev=0: None
    return m


@pytest.mark.parametrize("cname,logn", [("bn254", 3), ("bn254", 5), ("bls12-381", 4)])
def test_orchestration_against_oracle_prover(monkeypatch, cname, logn):
    from gnark_b200 import lib as real_lib, plonk as b200_plonk
    c = CURVES[cname]
    calls = []
    monkeypatch.setattr(b200_plonk, "_lib", make_mock_lib(real_lib, calls))
    monkeypatch.setattr(b200_plonk, "_device", lambda dev: "cpu")
    monkeypatch.setattr(b200_plonk, "_new_stream",
                        lambda torch, dev: types.SimpleNamespace(cuda_stream=1234, synchronize=lambda: None))
    monkeypatch.setattr(b200_plonk, "_stream_ctx", lambda torch, s: contextlib.nullcontext())

    rng = random.Random(500 + logn)
    r, L = c.r, c.fr_limbs
    n = 1 << logn
    circ, l, rr, o = pp.random_satisfied_instance(c, n, seed=logn)
    rnd = lambda: rng.randrange(r)
    ch = pp.Challenges(gamma=rnd(), beta=rnd(), alpha=rnd(), zeta=rnd(), v=rnd(), bl=[rnd(), rnd()], br=[rnd(), rnd()],
                       bo=[rnd(), rnd()], bz=[rnd(), rnd(), rnd()])
    tau = rnd()
    want = pp.prove(c, circ, l, rr, o, ch, tau)
    assert pp.verify(c, circ, want, ch, tau)
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
    # the library was pointed at the orchestrator's stream for the duration and handed back afterwards
    streams = [x[1] for x in calls if isinstance(x, tuple)]
    assert streams == [1234, 0, 1234, 0]
    # key load: 8 canonical conversions + 8 x 4 cached coset evaluations; per proof: 4 canonical conversions and
    # 4 polys x 4 cosets; 4 constraint calls; 10 commitments
    assert calls.count("ntt") == (8 + 32) + (4 + 16) and calls.count("constraints") == 4 and calls.count("msm") == 10
    pk.free()


@pytest.mark.parametrize("n_commit", (1, 2))
@pytest.mark.parametrize("coset_cache", ("1", "0"))
def test_orchestration_with_bsb22_commitments(monkeypatch, n_commit, coset_cache):
    """BSB22 commitment gates through the orchestrator: gate term on every coset, [PI2_j], the linearised-polynomial
    term sum_j Qcp_j(zeta) PI2_j(X) and the extra Qcp openings - against the oracle prover (whose proof passes the
    extended verifier equations)"""
    from gnark_b200 import lib as real_lib, plonk as b200_plonk
    monkeypatch.setenv("GB200_PLONK_COSET_CACHE", coset_cache)
    c = CURVES["bn254"]
    calls = []
    monkeypatch.setattr(b200_plonk, "_lib", make_mock_lib(real_lib, calls))
    monkeypatch.setattr(b200_plonk, "_device", lambda dev: "cpu")
    monkeypatch.setattr(b200_plonk, "_new_stream",
                        lambda torch, dev: types.SimpleNamespace(cuda_stream=1234, synchronize=lambda: None))
    monkeypatch.setattr(b200_plonk, "_stream_ctx", lambda torch, s: contextlib.nullcontext())
    logn = 4
    rng = random.Random(900 + n_commit)
    r, L = c.r, c.fr_limbs
    n = 1 << logn
    circ, l, rr, o, pi2 = pp.random_satisfied_instance(c, n, seed=31, n_commit=n_commit)
    rnd = lambda: rng.randrange(r)
    ch = pp.Challenges(gamma=rnd(), beta=rnd(), alpha=rnd(), zeta=rnd(), v=rnd(), bl=[rnd(), rnd()], br=[rnd(), rnd()],
                       bo=[rnd(), rnd()], bz=[rnd(), rnd(), rnd()])
    tau = rnd()
    want = pp.prove(c, circ, l, rr, o, ch, tau, pi2=pi2)
    assert pp.verify(c, circ, want, ch, tau)
    pe = lambda v: ff.pack_elements(v, r, L)
    srs = corelib.fixed_base(c, 1, ec.pack_points(c, 1, [c.g1]), pe([pow(tau, i, r) for i in range(n + 3)]))
    pk = b200_plonk.ProvingKey.from_trace(c.curve_id, logn, pe(circ.ql), pe(circ.qr), pe(circ.qm), pe(circ.qo),
                                         pe(circ.qk), np.array(circ.perm, dtype=np.int64), srs,
                                         qcp=[pe(v) for v in circ.qcp])
    got = b200_plonk.Prove(pk, pe(l), pe(rr), pe(o),
                           b200_plonk.Challenges(gamma=ch.gamma, beta=ch.beta, alpha=ch.alpha, zeta=ch.zeta, v=ch.v,
                                                 bl=ch.bl, br=ch.br, bo=ch.bo, bz=ch.bz), pi2=[pe(v) for v in pi2])
    F = ff.Fp(c.p)
    pt = lambda dlog: ec.scalar_mul(F, dlog, c.g1)
    for name, g_, w_ in (("L", got.LRO[0], want.L), ("Z", got.Z, want.Z), ("H1", got.H[0], want.H[0]),
                         ("H3", got.H[2], want.H[2]), ("lin", got.LinearizedDigest, want.lin),
                         ("batch", got.BatchedProofH, want.batch_opening), ("zopen", got.ZShiftedOpeningH, want.z_opening)):
        assert jac_to_affine(c, 1, g_) == pt(w_), name
    for j in range(n_commit):
        assert jac_to_affine(c, 1, got.Bsb22Commitments[j]) == pt(want.bsb22[j])
    assert got.BatchedClaimedValues == want.claimed and len(want.claimed) == 6 + n_commit
    assert got.ZShiftedClaimedValue == want.zu
    assert calls.count("bsb22") == 4 * n_commit
    with pytest.raises(ValueError):
        b200_plonk.Prove(pk, pe(l), pe(rr), pe(o), b200_plonk.Challenges(gamma=1, beta=2, alpha=3, zeta=4, v=5))
