"""Device-resident PLONK prover: host orchestration over the C ABI (include/gnark_b200.h).

The reference has no accelerated PLONK (SURVEY.md §0.3); this is the twin of the CPU prover
backend/plonk/bn254/prove.go, stage by stage, with every polynomial kept in HBM between the
MSM / NTT stages and only digests, challenges and opened values crossing to the host - the four
mandatory sync points of the Fiat-Shamir transcript (SURVEY.md Appendix A).

    pk = ProvingKey.from_trace(curve, log2n, ql, qr, qm, qo, qk, perm, srs_canonical)   # setupDevicePointers
    proof = Prove(pk, l, r, o, challenges)

Stages (reference line numbers in backend/plonk/bn254/prove.go):
  commitToLRO :404-489           canonical forms (iNTT), blinding :1211-1220, 3 MSMs on the SRS
  buildRatioCopyConstraint :635  b200_plonk_build_z, commit Z
  computeQuotient :558-633       48 coset NTTs + fused constraint kernel x4 :841-1123, divideByZH :1287,
                                 commitToQuotient :1263-1282 (3 MSMs of n+2)
  openZ :670-687, computeLinearizedPolynomial :724-794 (+ :1366-1487), batchOpening :796-837

Digests are computed from canonical coefficients against the canonical SRS: [p + b(X^n - 1)] is one MSM of
n + deg(b) + 1 points, the same group element the reference obtains from its Lagrange-SRS MSM plus
commitBlindingFactor (:1223-1236).  BSB22 commitment gates (:867-884) are supported with the committed polynomials
PI2_i given by the caller (in the reference they come out of the solver hint :280-318): their selectors Qcp_i are
part of the key, the gate term, the linearised-polynomial term sum_i Qcp_i(zeta) PI2_i(X) (:1457) and the Qcp openings
(:805-817) are added, and the digests [PI2_i] are returned.  StatisticalZK is not supported.

Challenges and blinding coefficients are taken from the caller (`Challenges`): the Fiat-Shamir transcript
encoding is gnark-crypto's (absent here); a Go shim derives them exactly as prove.go:492-555 does and passes
them in, which also makes every intermediate result reproducible (parity tests).
Host language note: the reference's prover is Go orchestrating gnark-crypto calls; with no Go toolchain in this
image the orchestration is Python over the same C ABI a Go shim would call (INTEGRATION.md §4).
"""

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from . import lib as _lib

_FR_MODULUS = {
    _lib.BN254: 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001,
    _lib.BLS12_381: 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001,
    _lib.BLS12_377: 0x12ab655e9a2ca55660b44d1e5c37b00159aa76fed00000010a11800000000001,
    _lib.BW6_761: 0x1ae3a4617c510eac63b05c06ca1493b1a22d9f300f5138f1ef3622fba094800170b5d44300000008508c00000000001,
}
# gnark-crypto fft.Domain constants (2-adicity, root of unity, FrMultiplicativeGen) - as params_gen.cuh
_FR_DOMAIN = {
    _lib.BN254: (28, 19103219067921713944291392827692070036145651957329286315305642004821462161904, 5),
    _lib.BLS12_381: (32, 10238227357739495823651030575849232062558860180284477541189508159991286009131, 7),
    _lib.BLS12_377: (47, 8065159656716812877374967518403273466521432693661810619979959746626482506078, 22),
    _lib.BW6_761: (46, 32863578547254505029601261939868325669770508939375122462904745766352256812585773382134936404344547323199885654433, 15),
}


# device plumbing, gathered here so that tests/test_plonk_orchestration.py can run the ORCHESTRATION (ordering,
# layouts, blinding, index conventions) on host tensors against a mock of the C ABI; the product always
# runs on CUDA and there is no CPU implementation of any library call
def _device(dev: int) -> str:
    return f"cuda:{dev}"


def _new_stream(torch, dev: int):
    return torch.cuda.Stream(device=dev)


def _stream_ctx(torch, stream):
    return torch.cuda.stream(stream)


@dataclass
class Challenges:
    gamma: int
    beta: int
    alpha: int
    zeta: int
    v: int
    bl: List[int] = field(default_factory=lambda: [0, 0])
    br: List[int] = field(default_factory=lambda: [0, 0])
    bo: List[int] = field(default_factory=lambda: [0, 0])
    bz: List[int] = field(default_factory=lambda: [0, 0, 0])


@dataclass
class Proof:
    """backend/plonk/bn254/prove.go:77-96.  Digests are Jacobian points in gnark layout (uint64 limbs)."""
    LRO: List[np.ndarray]
    Z: np.ndarray
    H: List[np.ndarray]
    LinearizedDigest: np.ndarray
    BatchedProofH: np.ndarray
    BatchedClaimedValues: List[int]
    ZShiftedOpeningH: np.ndarray
    ZShiftedClaimedValue: int
    Bsb22Commitments: List[np.ndarray] = field(default_factory=list)
    timings_ms: dict = field(default_factory=dict)


class _Fr:
    """tiny host-side helper: canonical int <-> fr.Element limbs (Montgomery)"""

    def __init__(self, curve):
        self.q = _FR_MODULUS[curve]
        self.limbs = _lib.CURVE_SHAPES[curve][0]
        self.R = 1 << (64 * self.limbs)
        self.Rinv = pow(self.R, -1, self.q)

    def enc(self, x: int) -> np.ndarray:
        v = (x % self.q) * self.R % self.q
        return np.frombuffer(v.to_bytes(8 * self.limbs, "little"), dtype=np.uint64).copy()

    def enc_many(self, xs) -> np.ndarray:
        return np.concatenate([self.enc(x) for x in xs]) if len(xs) else np.zeros(0, dtype=np.uint64)

    def dec(self, a) -> int:
        return int.from_bytes(np.ascontiguousarray(a, dtype=np.uint64).tobytes(), "little") * self.Rinv % self.q


class ProvingKey:
    """Device-resident PLONK proving key (backend/plonk/bn254/setup.go:88-93 ProvingKey + Trace :67-86)."""

    def __init__(self, curve: int, log2n: int, dev: int = 0, shard=None):
        """shard = (rank, world, process_group): one process per GPU.  Polynomials and the O(n) stages are
        replicated; the two things that dominate a proof are split (SURVEY.md §8e): every KZG commitment is a
        point-range-sharded MSM (this rank holds SRS points [off, off+cnt), partial digests all-gathered and
        summed on the host, as parallel.sharded_msm), and coset i of the quotient numerator is evaluated by rank
        i mod world, the disjoint quarter results merged with one all-reduce."""
        import torch
        self.torch = torch
        self.curve, self.log2n, self.dev = curve, log2n, dev
        self.rank, self.world, self.pg = (0, 1, None) if shard is None else shard
        if not (0 <= self.rank < self.world):
            raise ValueError(f"invalid shard {self.rank}/{self.world}")
        self.n = 1 << log2n
        self.fr = _Fr(curve)
        s, root, g = _FR_DOMAIN[curve]
        q = self.fr.q
        self.g = g
        self.w = pow(root, 1 << (s - log2n), q)                 # domain0.Generator
        self.w4 = pow(root, 1 << (s - log2n - 2), q)            # domain1.Generator
        # domain0 handles for the four cosets g * w4^i (computeNumerator :943-948) and the big domain
        self.dom0 = [_lib.Domain(curve, log2n, dev=dev, coset_gen=self.fr.enc(g * pow(self.w4, i, q) % q)) for i in range(4)]
        self.dom1 = _lib.Domain(curve, log2n + 2, dev=dev)
        # ONE stream for everything: torch tensor ops (clone, slice copies, H2D/D2H) and the library's kernels
        # must be ordered with respect to each other, so the library is pointed at this torch stream while a
        # key method / Prove runs (the library's own stream is non-blocking and would race with torch's)
        self.stream = _new_stream(torch, dev)
        self.polys = {}        # name -> device tensor, CANONICAL coefficients in BIT-REVERSED layout (n)
        self.canon = {}        # name -> canonical, regular layout (for evaluations / linearised polynomial)
        self.perm = None
        self.srs = None

    def _dev(self, arr):
        return self.torch.from_numpy(np.ascontiguousarray(arr).view(np.int64)).to(_device(self.dev))

    def on_stream(self):
        """context manager: torch's current stream and the library's stream are both self.stream"""
        pk = self

        class _Ctx:
            def __enter__(self_inner):
                self_inner.cm = _stream_ctx(pk.torch, pk.stream)
                self_inner.cm.__enter__()
                _lib.set_stream(pk.dev, pk.stream.cuda_stream)
                return pk

            def __exit__(self_inner, *exc):
                pk.stream.synchronize()
                _lib.set_stream(pk.dev, 0)          # back to the library's own stream
                return self_inner.cm.__exit__(*exc)
        return _Ctx()

    @classmethod
    def from_trace(cls, curve, log2n, ql, qr, qm, qo, qk, perm, srs_canonical, dev=0, shard=None, qcp=()):
        """ql..qk: (n, limbs) uint64 Lagrange/regular (Montgomery); perm: int64[3n]; srs_canonical: (n+3) G1Affine
        (the FULL SRS on every rank; a sharded key uploads only its own point range)."""
        pk = cls(curve, log2n, dev, shard=shard)
        with pk.on_stream():
            pk._load(ql, qr, qm, qo, qk, perm, srs_canonical, qcp)
        return pk

    def _load(self, ql, qr, qm, qo, qk, perm, srs_canonical, qcp=()):
        pk, curve, log2n, dev = self, self.curve, self.log2n, self.dev
        t = pk.torch
        n, L, q = pk.n, pk.fr.limbs, pk.fr.q
        pk.perm = t.from_numpy(np.ascontiguousarray(perm, dtype=np.int64)).to(_device(dev))
        # sigma polynomials from the permutation: s_j[i] = supp[perm[j n + i]], supp = <w> || g<w> || g^2<w>
        # (setup.go:289-392, getSupportPermutation :377-392) - built on the device: powers of w by
        # b200_vec_scale_powers on a vector of ones, the two cosets by a constant scaling, then one gather
        one = pk.fr.enc(1)
        d_w = pk._dev(np.tile(one, (n, 1))).reshape(-1)
        _lib.vec_scale_powers(dev, curve, d_w, n, one, pk.fr.enc(pk.w))
        supp = t.empty((3 * n, L), dtype=t.int64, device=d_w.device)
        supp[:n] = d_w.view(n, L)
        for j in (1, 2):
            blk = d_w.clone()
            _lib.vec_scale_powers(dev, curve, blk, n, pk.fr.enc(pow(pk.g, j, q)), one)
            supp[j * n:(j + 1) * n] = blk.view(n, L)
        lag = {"ql": ql, "qr": qr, "qm": qm, "qo": qo, "qk": qk}
        pk.n_commit = len(qcp)
        for j, v in enumerate(qcp):                  # trace.Qcp: selectors of the BSB22 commitment gates
            lag[f"qcp{j}"] = v
        sigma = {name: supp[pk.perm[j * n:(j + 1) * n]].contiguous() for j, name in enumerate(("s1", "s2", "s3"))}
        del supp, d_w
        for name in ("ql", "qr", "qm", "qo", "qk", "s1", "s2", "s3") + tuple(f"qcp{j}" for j in range(pk.n_commit)):
            d = pk._dev(lag[name]) if name in lag else sigma[name]
            pk.dom0[0].ntt_async(d, inverse=True, decimation=_lib.DIF)       # Lagrange/regular -> canonical/bit-reversed
            pk.polys[name] = d
            c = d.clone()
            _lib.vec_bit_reverse(dev, curve, c, log2n)
            pk.canon[name] = c
        # the key polynomials never change between proofs: keep their evaluations on the four quotient cosets in
        # HBM ((8 + n_commit) x 4 x n elements; 4 GiB at n = 2^22), so a proof runs 16 coset NTTs instead of 48.
        # A sharded key keeps only the cosets this rank evaluates.  GB200_PLONK_COSET_CACHE=0 turns it off.
        import os
        pk.key_cos = {}
        if os.environ.get("GB200_PLONK_COSET_CACHE", "1") != "0":
            for i in range(4):
                if i % pk.world != pk.rank:
                    continue
                for name, d in pk.polys.items():
                    e = d.clone()
                    pk.dom0[i].ntt_async(e, inverse=False, decimation=_lib.DIT, on_coset=True)
                    pk.key_cos[(i, name)] = e
        from .parallel import shard_range
        srs = np.ascontiguousarray(srs_canonical).reshape(n + 3, -1)
        pk.srs_off, pk.srs_cnt = shard_range(n + 3, pk.world, pk.rank)
        pk.srs = _lib.Table(curve, 1, np.ascontiguousarray(srs[pk.srs_off:pk.srs_off + pk.srs_cnt]), dev=dev, precomp=True,
                            n=pk.srs_cnt)
        _lib.sync(dev)

    def free(self):
        for d in self.dom0:
            d.free()
        self.dom1.free()
        if self.srs is not None:
            self.srs.free()


def bsb22_commitment(lagrange_table, nb_public: int, committed, values, blind2):
    """The commitment of the BSB22 solver hint (bsb22Hint, backend/plonk/bn254/prove.go:280-315) and its committed
    polynomial.  The hint's vector has n = lagrange_table.n entries (Lagrange form, regular layout) and is zero except:
      nb_public + committed[i]  <- values[i]     (the committed wires, ci.Committed)
      nb_public + p             <- v             for each (p, v) of blind2: the two blinding values, at the commitment
                                                 constraint ci.CommitmentIndex and at the last constraint nbConstraints - 1
    written in that order (a later write replaces an earlier one, as in the hint).  The digest kzg.Commit(vector,
    pk.KzgLagrange) is one indexed MSM over those few entries (Table.msm_indexed), not an MSM over n scalars.
    values: (len(committed), fr_limbs) Montgomery; blind2: two (constraint index, Montgomery value).
    Returns (digest as a Jacobian point in gnark layout, the dense (n, fr_limbs) vector that Prove(..., pi2=) takes)."""
    L = lagrange_table.fr_limbs
    values = np.ascontiguousarray(values, dtype=np.uint64).reshape(-1, L)
    if len(committed) != values.shape[0]:
        raise ValueError(f"{len(committed)} committed wires and {values.shape[0]} values")
    if len(blind2) != 2:
        raise ValueError("the hint blinds exactly two entries")
    entries = {}
    for p, v in list(zip(committed, values)) + [(p, np.asarray(v, dtype=np.uint64).reshape(L)) for p, v in blind2]:
        pos = nb_public + int(p)
        if not 0 <= pos < lagrange_table.n:
            raise ValueError(f"position {pos} outside the {lagrange_table.n}-point Lagrange basis")
        entries[pos] = v
    idx = np.fromiter(entries.keys(), dtype=np.uint32, count=len(entries))
    sc = np.ascontiguousarray(np.stack(list(entries.values())), dtype=np.uint64)
    dense = np.zeros((lagrange_table.n, L), dtype=np.uint64)
    dense[idx] = sc
    return lagrange_table.msm_indexed(idx, sc), dense


def Prove(pk: ProvingKey, l, r, o, ch: Challenges, pi2=()) -> Proof:
    """l, r, o: (n, limbs) uint64 Lagrange/regular solution vectors (SparseR1CSSolution{L,R,O},
    constraint/bn254/system.go:208-210) on the host; pi2: one (n, limbs) Lagrange/regular vector per BSB22
    commitment of the key (the committed polynomials the solver hint produced)."""
    if len(pi2) != getattr(pk, "n_commit", 0):
        raise ValueError("one committed polynomial per Qcp selector of the key is required")
    with pk.on_stream():
        return _prove(pk, l, r, o, ch, pi2)


def _prove(pk: ProvingKey, l, r, o, ch: Challenges, pi2=()) -> Proof:
    import time
    t = pk.torch
    curve, dev, n, logn = pk.curve, pk.dev, pk.n, pk.log2n
    fr = pk.fr
    q, L = fr.q, fr.limbs
    E = fr.enc
    tm = {}
    t_start = time.perf_counter()

    def lap(name):
        _lib.sync(dev)
        nonlocal t_start
        now = time.perf_counter()
        tm[name] = tm.get(name, 0.0) + 1e3 * (now - t_start)
        t_start = now

    def commit(d_coeffs, count):
        """[sum_i c_i tau^i]: this rank's point range of the first `count` coefficients, then (sharded key) one
        all_gather of the partial digests and host-side group additions"""
        lo = min(pk.srs_off, count)
        hi = min(pk.srs_off + pk.srs_cnt, count)
        flat = d_coeffs.reshape(-1)
        part = pk.srs.msm(flat[lo * L:hi * L], n=hi - lo, on_device=True)
        if pk.world == 1:
            return part
        import torch.distributed as dist
        mine = t.from_numpy(part.view(np.int64).copy()).to(flat.device)
        parts = [t.empty_like(mine) for _ in range(pk.world)]
        dist.all_gather(parts, mine, group=pk.pg)
        acc = parts[0].cpu().numpy().view(np.uint64).copy()
        for p_ in parts[1:]:
            _lib.point_add_jac(curve, 1, acc, p_.cpu().numpy().view(np.uint64))
        return acc

    def canonical_blinded(d_lagrange, b):
        """Lagrange/regular -> (canonical bit-reversed copy for the coset NTTs, blinded canonical regular [n+len(b)])"""
        cb = d_lagrange.clone()
        pk.dom0[0].ntt_async(cb, inverse=True, decimation=_lib.DIF)
        reg = t.zeros((n + len(b)) * L, dtype=t.int64, device=cb.device)
        reg[:n * L] = cb.reshape(-1)
        _lib.vec_bit_reverse(dev, curve, reg, logn)
        # p + b (X^n - 1): low coefficients minus b, then b on top (getBlindedCoefficients :1211-1220)
        low = reg[:len(b) * L].cpu().numpy().view(np.uint64).reshape(len(b), L)
        patched = fr.enc_many([(fr.dec(low[i]) - b[i]) % q for i in range(len(b))])
        reg[:len(b) * L] = t.from_numpy(patched.view(np.int64)).to(reg.device)
        reg[n * L:] = t.from_numpy(fr.enc_many(b).view(np.int64)).to(reg.device)
        return cb, reg

    # ---- commitToLRO ----------------------------------------------------------------------------
    d_l, d_r, d_o = (pk._dev(v) for v in (l, r, o))
    cb, blinded = {}, {}
    for name, d, b in (("l", d_l, ch.bl), ("r", d_r, ch.br), ("o", d_o, ch.bo)):
        cb[name], blinded[name] = canonical_blinded(d, b)
    lro = [commit(blinded[k], n + 2) for k in ("l", "r", "o")]
    # BSB22: committed polynomials, canonical (bit-reversed for the coset NTTs, regular for [PI2_j] and the rest)
    pi2_br, pi2_canon, bsb22 = [], [], []
    for v in pi2:
        d = pk._dev(v).reshape(-1)
        pk.dom0[0].ntt_async(d, inverse=True, decimation=_lib.DIF)
        c_ = d.clone()
        _lib.vec_bit_reverse(dev, curve, c_, logn)
        pi2_br.append(d); pi2_canon.append(c_)
        bsb22.append(commit(c_, n))
    lap("commit LRO")

    # ---- buildRatioCopyConstraint + commit Z ------------------------------------------------------
    d_z = t.zeros(n * L, dtype=t.int64, device=d_l.device)
    _lib.plonk_build_z(pk.dom0[0], d_l, d_r, d_o, pk.perm, E(ch.beta), E(ch.gamma), d_z)
    cb["z"], blinded["z"] = canonical_blinded(d_z, ch.bz)
    z_digest = commit(blinded["z"], n + 3)
    lap("build + commit Z")

    # ---- computeQuotient: numerator on the 4 cosets, divide by Z_H, commit h1, h2, h3 --------------
    cres = t.zeros(4 * n * L, dtype=t.int64, device=d_l.device)
    names = ("l", "r", "o", "z", "s1", "s2", "s3", "ql", "qr", "qm", "qo", "qk")
    blind = {"l": fr.enc_many(ch.bl), "r": fr.enc_many(ch.br), "o": fr.enc_many(ch.bo), "z": fr.enc_many(ch.bz)}
    g_m, w4_m = E(pk.g), E(pk.w4)
    a_m, b_m, c_m = E(ch.alpha), E(ch.beta), E(ch.gamma)
    for i in range(4):
        if i % pk.world != pk.rank:          # this coset belongs to another rank
            continue
        on_coset = {}
        for name in names:
            if (i, name) in pk.key_cos:
                on_coset[name] = pk.key_cos[(i, name)]
                continue
            src = cb[name] if name in cb else pk.polys[name]
            d = src.clone()
            pk.dom0[i].ntt_async(d, inverse=False, decimation=_lib.DIT, on_coset=True)   # canonical/bit-rev -> coset i, regular
            on_coset[name] = d
        _lib.plonk_constraints_coset(pk.dom0[i], g_m, w4_m, on_coset, a_m, b_m, c_m, blind, i, 4, cres)
        for j in range(len(pi2)):           # + Qcp_j * PI2_j on this coset (gateConstraint :881-884)
            dp = pi2_br[j].clone()
            pk.dom0[i].ntt_async(dp, inverse=False, decimation=_lib.DIT, on_coset=True)
            dq = pk.key_cos.get((i, f"qcp{j}"))
            if dq is None:
                dq = pk.polys[f"qcp{j}"].clone()
                pk.dom0[i].ntt_async(dq, inverse=False, decimation=_lib.DIT, on_coset=True)
            _lib.plonk_bsb22_coset(pk.dom0[i], dq, dp, i, 4, cres)
        _lib.sync(dev)
        del on_coset
    if pk.world > 1:
        # every slot of cres was written by exactly one rank and is zero elsewhere: an integer SUM merges the quarters
        import torch.distributed as dist
        dist.all_reduce(cres, op=dist.ReduceOp.SUM, group=pk.pg)
    _lib.plonk_divide_by_zh(pk.dom1, logn, cres)       # -> h canonical regular (4n)
    h = cres
    H = [commit(h[k * (n + 2) * L:(k + 1) * (n + 2) * L], n + 2) for k in range(3)]
    lap("quotient + commit H")

    # ---- openZ, evaluations at zeta ------------------------------------------------------------
    zeta = ch.zeta % q
    wz = zeta * pk.w % q
    ev = lambda d, cnt, x: fr.dec(_lib.poly_eval(dev, curve, d, cnt, E(x)))
    zu = ev(blinded["z"], n + 3, wz)
    lz, rz, oz = (ev(blinded[k], n + 2, zeta) for k in ("l", "r", "o"))
    s1z, s2z = ev(pk.canon["s1"], n, zeta), ev(pk.canon["s2"], n, zeta)

    # ---- innerComputeLinearizedPoly :1366-1487 ------------------------------------------------------
    alpha, beta, gamma = ch.alpha % q, ch.beta % q, ch.gamma % q
    rl = rz * lz % q
    c1 = (lz + beta * s1z + gamma) % q * ((rz + beta * s2z + gamma) % q) % q * zu % q * beta % q * alpha % q
    uz, uuz = zeta * pk.g % q, zeta * pk.g % q * pk.g % q
    c2 = (-(lz + beta * zeta + gamma) % q * ((rz + beta * uz + gamma) % q) % q * ((oz + beta * uuz + gamma) % q) % q * alpha) % q
    zn = pow(zeta, n, q)
    zn2 = zn * zeta % q * zeta % q
    zh = (zn - 1) % q
    a2l1 = zh * pow((zeta - 1) % q, -1, q) % q * alpha % q * alpha % q * pow(n, -1, q) % q
    lin = t.zeros((n + 3) * L, dtype=t.int64, device=d_l.device)
    axpy = lambda y, a, x, cnt: _lib.vec_axpy(dev, curve, y, E(a), x, cnt)
    axpy(lin, (c2 + a2l1) % q, blinded["z"], n + 3)
    for coef, name in ((c1, "s3"), (rl, "qm"), (lz, "ql"), (rz, "qr"), (oz, "qo"), (1, "qk")):
        axpy(lin, coef, pk.canon[name], n)
    qcpz = [ev(pk.canon[f"qcp{j}"], n, zeta) for j in range(len(pi2))]
    for j in range(len(pi2)):               # + sum_j Qcp_j(zeta) PI2_j(X)   (:1457-1460)
        axpy(lin, qcpz[j], pi2_canon[j], n)
    for k, coef in enumerate((zh, zh * zn2 % q, zh * zn2 % q * zn2 % q)):
        axpy(lin, (-coef) % q, h[k * (n + 2) * L:(k + 1) * (n + 2) * L], n + 2)
    lin_digest = commit(lin, n + 3)
    lap("linearised polynomial")

    # ---- batchOpening :796-837 (fold with powers of v, divide by X - zeta) and the Z opening ---------
    to_open = [(lin, n + 3), (blinded["l"], n + 2), (blinded["r"], n + 2), (blinded["o"], n + 2),
               (pk.canon["s1"], n), (pk.canon["s2"], n)] + [(pk.canon[f"qcp{j}"], n) for j in range(len(pi2))]
    claimed = [ev(d, cnt, zeta) for d, cnt in to_open]
    fold = t.zeros((n + 3) * L, dtype=t.int64, device=d_l.device)
    vp = 1
    for d, cnt in to_open:
        axpy(fold, vp, d, cnt)
        vp = vp * ch.v % q
    _lib.poly_div_by_linear(dev, curve, fold, n + 3, E(zeta))
    batch_h = commit(fold, n + 2)
    zq = blinded["z"].clone()
    zu_check = fr.dec(_lib.poly_div_by_linear(dev, curve, zq, n + 3, E(wz)))
    assert zu_check == zu
    z_open_h = commit(zq, n + 2)
    lap("openings")
    return Proof(LRO=lro, Z=z_digest, H=H, LinearizedDigest=lin_digest, BatchedProofH=batch_h,
                 BatchedClaimedValues=claimed, ZShiftedOpeningH=z_open_h, ZShiftedClaimedValue=zu, Bsb22Commitments=bsb22,
                 timings_ms=tm)
