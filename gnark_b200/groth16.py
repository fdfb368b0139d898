"""Host-side mirror of the reference's accelerated Groth16 package
(backend/accelerated/icicle/groth16/groth16_icicle.go:79-194 and
backend/accelerated/icicle/opts.go:10-124): same function set and option names,
on top of libgnark_b200.so.  Python stands in for the Go shim of INTEGRATION.md
because this image has no Go toolchain; the arithmetic all happens in the C ABI.

    pk = NewProvingKey(ecc_id); pk.load(...)           # or ProvingKey.from_arrays
    proof = Prove(r1cs, pk, full_witness, WithDeviceID(0), WithPinToGPU(True))

Out of scope here, as in the reference's accelerated package: the R1CS solver
(`r1cs.Solve`, constraint/bn254/solver.go) - any object with a
``Solve(witness) -> R1CSSolution`` method plugs in - Setup / Verify (CPU, pairing).
"""

import ctypes
import os
import secrets
from dataclasses import dataclass, field
from typing import Callable, List, Optional

import numpy as np

from . import lib as _lib

# ecc.ID values used across the ABI
BN254, BLS12_381, BLS12_377, BW6_761 = _lib.BN254, _lib.BLS12_381, _lib.BLS12_377, _lib.BW6_761

_FR_MODULUS = {
    BN254: 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001,
    BLS12_381: 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001,
    BLS12_377: 0x12ab655e9a2ca55660b44d1e5c37b00159aa76fed00000010a11800000000001,
    BW6_761: 0x1ae3a4617c510eac63b05c06ca1493b1a22d9f300f5138f1ef3622fba094800170b5d44300000008508c00000000001,
}


# ---- options (backend/accelerated/icicle/opts.go) -----------------------------------
@dataclass
class Config:
    DeviceID: int = 0
    PinToGPU: bool = True        # tables are always device resident here; kept for API parity
    Precompute: bool = True      # build the per-window table slabs (B200_TABLE_PRECOMP)
    ProverOpts: list = field(default_factory=list)
    Randomness: Optional[Callable[[int], int]] = None   # test hook: r,s injection (SURVEY.md §0.4)
    ShardRank: int = 0           # multi-GPU (one process per GPU): this process's point-range shard
    ShardWorld: int = 1
    ProcessGroup: object = None  # torch.distributed group used to gather the partial MSM results
    Devices: tuple = ()          # multi-GPU inside ONE process (WithDevices): one point-range shard per listed device


Option = Callable[[Config], None]


def NewConfig(*opts: Option) -> Config:
    cfg = Config()
    for o in opts:
        if o is not None:
            o(cfg)
    return cfg


def WithDeviceID(dev: int) -> Option:
    def f(c: Config):
        if dev < 0:
            raise ValueError(f"invalid device id {dev}")
        c.DeviceID = dev
    return f


def WithPinToGPU(pin: bool) -> Option:
    def f(c: Config):
        c.PinToGPU = pin
    return f


def WithPrecompute(on: bool) -> Option:
    def f(c: Config):
        c.Precompute = on
    return f


def WithProverOptions(*opts) -> Option:
    def f(c: Config):
        if not opts:
            raise ValueError("no prover options provided")
        c.ProverOpts = list(opts)
    return f


def WithSharding(rank: int, world: int, process_group=None) -> Option:
    """One process per GPU: every MSM table is cut into `world` contiguous point ranges
    (SURVEY.md §8e); partial results are all-gathered over `process_group` and summed on the host
    (the shape of the reference's chunk loop, icicle.go:383-411)."""
    def f(c: Config):
        if world < 1 or not (0 <= rank < world):
            raise ValueError(f"invalid shard {rank}/{world}")
        c.ShardRank, c.ShardWorld, c.ProcessGroup = rank, world, process_group
    return f


def WithDevices(*devs: int) -> Option:
    """Several GPUs driven from ONE process - the shape a Go caller uses (a goroutine per device, no process group):
    device devs[i] holds point-range shard i of every MSM table; the device parts run concurrently (the C ABI
    serialises per device, not per process), the partial points are summed on the host and the proof is assembled
    once.  The reference has one device per proof (`WithDeviceID`, opts.go:68-77); this is its multi-GPU extension."""
    def f(c: Config):
        if not devs or any(d < 0 for d in devs) or len(set(devs)) != len(devs):
            raise ValueError(f"invalid device list {devs}")
        c.Devices = tuple(devs)
        c.DeviceID = devs[0]
    return f


def WithRandomness(fn: Callable[[int], int]) -> Option:
    """Deterministic r, s for parity tests (the reference samples crypto/rand, prove.go:170-182)."""
    def f(c: Config):
        c.Randomness = fn
    return f


# ---- data carried across the boundary ------------------------------------------------
@dataclass
class R1CSSolution:
    """constraint/bn254/system.go:162-165: fr.Vectors in gnark memory layout (uint64, Montgomery)."""
    W: np.ndarray
    A: np.ndarray
    B: np.ndarray
    C: np.ndarray


@dataclass
class Proof:
    """backend/groth16/bn254/prove.go:38-43: Ar, Krs in G1, Bs in G2 (affine, gnark layout)."""
    Ar: np.ndarray
    Bs: np.ndarray
    Krs: np.ndarray
    msm: Optional[np.ndarray] = None   # the five raw MSM results (A, B1, Z, K | B2), for parity tests


class ProvingKey:
    """Accelerated proving key: the native key's fields (backend/groth16/bn254/setup.go:25-48)
    plus the device handle, as backend/accelerated/icicle/groth16/bn254/provingkey.go:37-42."""

    def __init__(self, curve: int):
        self.curve = curve
        self.domain_size = 0
        self.domain_gen = None       # fr.Element or None (defaults as fft.NewDomain)
        self.coset_gen = None
        self.G1_Alpha = self.G1_Beta = self.G1_Delta = None
        self.G1_A = self.G1_B = self.G1_Z = self.G1_K = None
        self.G2_Beta = self.G2_Delta = self.G2_B = None
        self.InfinityA = self.InfinityB = None
        self.nb_wires = 0
        self.nb_public = 0
        self._handle = None
        self._dev = None
        self._handles = {}           # (device, shard rank, shard world, precompute) -> C handle

    @classmethod
    def from_arrays(cls, curve, domain_size, alpha, beta, delta, A, B, Z, K, beta2, delta2, B2, inf_a, inf_b,
                    nb_public, domain_gen=None, coset_gen=None, committed_private_wires=()):
        """committed_private_wires: sorted absolute indices of the private wires committed by BSB22 / Pedersen
        commitments (internal.ConcatAll(commitmentInfo.PrivateCommitted...), prove.go:231-235): K has no base for them"""
        pk = cls(curve)
        pk.k_removed = np.ascontiguousarray(sorted(int(x) for x in committed_private_wires), dtype=np.uint32)
        pk.domain_size = int(domain_size)
        pk.domain_gen, pk.coset_gen = domain_gen, coset_gen
        c = np.ascontiguousarray
        pk.G1_Alpha, pk.G1_Beta, pk.G1_Delta = c(alpha), c(beta), c(delta)
        pk.G1_A, pk.G1_B, pk.G1_Z, pk.G1_K = c(A), c(B), c(Z), c(K)
        pk.G2_Beta, pk.G2_Delta, pk.G2_B = c(beta2), c(delta2), c(B2)
        pk.InfinityA = np.ascontiguousarray(inf_a, dtype=np.uint8)
        pk.InfinityB = np.ascontiguousarray(inf_b, dtype=np.uint8)
        pk.nb_wires = len(pk.InfinityA)
        pk.nb_public = int(nb_public)
        return pk

    def use_dump_file(self, path: str, off_a: int, off_b: int, off_z: int, off_k: int, off_b2: int):
        """Load the five MSM tables from a ProvingKey dump file instead of the in-memory slices: byte offsets of the
        payloads of G1.A, G1.B, G1.Z, G1.K and G2.B (element 0 of each slice); the slice lengths are taken from the
        arrays this key was built with, which may then be dropped (set to None) by the caller."""
        self.dump = {"path": path, "off_a": off_a, "off_b": off_b, "off_z": off_z, "off_k": off_k, "off_b2": off_b2,
                     "n_a": self._count(self.G1_A, 1), "n_b": self._count(self.G1_B, 1), "n_z": self._count(self.G1_Z, 1),
                     "n_k": self._count(self.G1_K, 1)}
        for key in list(self._handles):
            _lib.check(_lib.load().b200_groth16_pk_free(self._handles.pop(key)))

    def _count(self, arr, group):
        frl, fpl, deg = _lib.CURVE_SHAPES[self.curve]
        per = 2 * fpl * (deg if group == 2 else 1)
        return arr.size // per

    def _load(self, dev: int, rank: int, world: int, precompute: bool):
        """b200_groth16_pk_load of shard rank/world on device dev (cached per key)."""
        key = (dev, rank, world, bool(precompute))
        if key in self._handles:
            return self._handles[key]
        d = _lib.Groth16PkDesc()
        d.curve = self.curve
        d.domain_size = self.domain_size
        p = _lib.ptr
        d.domain_gen, d.coset_gen = p(self.domain_gen), p(self.coset_gen)
        d.g1_alpha, d.g1_beta, d.g1_delta = p(self.G1_Alpha), p(self.G1_Beta), p(self.G1_Delta)
        d.g2_beta, d.g2_delta = p(self.G2_Beta), p(self.G2_Delta)
        dump = getattr(self, "dump", None)
        if dump is not None:
            # tables straight from gnark's ProvingKey dump file (marshal.go:375-539): payload offsets and lengths of
            # the five point slices, as the Go shim reads them from the dump's header
            d.dump_path = os.fsencode(dump["path"])
            d.dump_off_a, d.dump_off_b, d.dump_off_z = dump["off_a"], dump["off_b"], dump["off_z"]
            d.dump_off_k, d.dump_off_b2 = dump["off_k"], dump["off_b2"]
            d.n_a, d.n_b, d.n_z, d.n_k, d.n_b2 = dump["n_a"], dump["n_b"], dump["n_z"], dump["n_k"], dump["n_b"]
        else:
            d.g1_a, d.n_a = p(self.G1_A), self._count(self.G1_A, 1)
            d.g1_b, d.n_b = p(self.G1_B), self._count(self.G1_B, 1)
            d.g1_z, d.n_z = p(self.G1_Z), self._count(self.G1_Z, 1)
            d.g1_k, d.n_k = p(self.G1_K), self._count(self.G1_K, 1)
            d.g2_b, d.n_b2 = p(self.G2_B), self._count(self.G2_B, 2)
        d.infinity_a, d.infinity_b = p(self.InfinityA), p(self.InfinityB)
        d.nb_wires, d.nb_public = self.nb_wires, self.nb_public
        kr = getattr(self, "k_removed", None)
        if kr is not None and kr.size:
            d.k_removed, d.n_k_removed = p(kr), kr.size
        d.flags = _lib.TABLE_PRECOMP if precompute else 0
        d.shard_rank, d.shard_world = rank, world
        h = ctypes.c_void_p(0)
        _lib.check(_lib.load().b200_groth16_pk_load(dev, ctypes.byref(d), ctypes.byref(h)))
        self._handles[key] = h
        return h

    def setup_device_pointers(self, cfg: Config):
        """icicle.go:88-264 setupDevicePointers: once per key and device (per device AND shard with WithDevices)."""
        if len(cfg.Devices) > 1:
            want = {(dev, i, len(cfg.Devices), bool(cfg.Precompute)) for i, dev in enumerate(cfg.Devices)}
        else:
            want = {(cfg.DeviceID, cfg.ShardRank, cfg.ShardWorld, bool(cfg.Precompute))}
        for key in [k for k in self._handles if k not in want]:      # another placement: release it first
            _lib.check(_lib.load().b200_groth16_pk_free(self._handles.pop(key)))
        for key in sorted(want):
            self._load(*key)
        first = min(want, key=lambda k: k[1])
        self._handle, self._dev = self._handles[first], first

    def free_gpu_resources(self):
        """icicle.go:1493-1549 FreeGPUResources; safe to call repeatedly."""
        for key in list(self._handles):
            _lib.check(_lib.load().b200_groth16_pk_free(self._handles.pop(key)))
        self._handle = None

    def __del__(self):
        try:
            self.free_gpu_resources()
        except Exception:
            pass


def NewProvingKey(curve_id: int) -> ProvingKey:
    """groth16_icicle.go:179-194."""
    if curve_id not in _lib.CURVE_SHAPES:
        raise ValueError("b200 backend requested but curve is not supported")
    return ProvingKey(curve_id)


def _fr_to_mont_limbs(x: int, curve: int) -> np.ndarray:
    frl = _lib.CURVE_SHAPES[curve][0]
    q = _FR_MODULUS[curve]
    v = (x % q) * (1 << (64 * frl)) % q
    return np.frombuffer(v.to_bytes(8 * frl, "little"), dtype=np.uint64).copy()


def ProveSolution(pk: ProvingKey, sol: R1CSSolution, *opts: Option, keep_msm: bool = False) -> Proof:
    """The hot path proper: from the solver's output to the three proof points
    (backend/groth16/bn254/prove.go:131-315; icicle.go:981-1360)."""
    cfg = NewConfig(*opts)
    pk.setup_device_pointers(cfg)
    frl, fpl, deg = _lib.CURVE_SHAPES[pk.curve]
    q = _FR_MODULUS[pk.curve]
    rnd = cfg.Randomness or (lambda modulus: secrets.randbelow(modulus))
    r = _fr_to_mont_limbs(rnd(q), pk.curve)
    s = _fr_to_mont_limbs(rnd(q), pk.curve)
    n_constraints = sol.A.size // frl
    if sol.W.size // frl != pk.nb_wires:
        raise ValueError("witness size does not match the proving key")
    ar = np.zeros(2 * fpl, dtype=np.uint64)
    krs = np.zeros(2 * fpl, dtype=np.uint64)
    bs = np.zeros(2 * fpl * deg, dtype=np.uint64)
    p = _lib.ptr
    L = _lib.load()
    j1 = 3 * fpl
    spans = [(k * j1, (k + 1) * j1, 1) for k in range(4)] + [(4 * j1, 4 * j1 + 3 * fpl * deg, 2)]

    def fold(parts):
        """five partial MSM results per shard -> their sums (host-side group additions, icicle.go:383-411)"""
        acc = parts[0].copy()
        for q in parts[1:]:
            for lo, hi, grp in spans:
                seg = np.ascontiguousarray(acc[lo:hi])
                _lib.point_add_jac(pk.curve, grp, seg, np.ascontiguousarray(q[lo:hi]))
                acc[lo:hi] = seg
        return acc

    if len(cfg.Devices) > 1:
        # one process, several GPUs: the device parts of all shards run concurrently (ctypes releases the GIL,
        # the C ABI locks per device); what a Go shim does with one goroutine per device
        import threading
        nd = len(cfg.Devices)
        parts = [np.zeros(4 * 3 * fpl + 3 * fpl * deg, dtype=np.uint64) for _ in range(nd)]
        errs = [None] * nd

        def run(i, dev):
            try:
                h = pk._handles[(dev, i, nd, bool(cfg.Precompute))]
                _lib.check(L.b200_groth16_msms(h, p(sol.W), p(sol.A), p(sol.B), p(sol.C), n_constraints, p(parts[i])))
            except Exception as e:      # re-raised on the calling thread
                errs[i] = e
        ts = [threading.Thread(target=run, args=(i, dev)) for i, dev in enumerate(cfg.Devices)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        for e in errs:
            if e is not None:
                raise e
        msm = fold(parts)
        _lib.check(L.b200_groth16_assemble(pk._handle, p(msm), p(r), p(s), p(ar), p(bs), p(krs)))
        return Proof(Ar=ar, Bs=bs, Krs=krs, msm=msm if keep_msm else None)
    comm_world = _lib.comm_info(cfg.DeviceID)[0] if cfg.ShardWorld > 1 else 1
    if cfg.ShardWorld <= 1 or comm_world == cfg.ShardWorld:
        # single device, or sharded with the library's communicator (b200_comm_init): the five partial sums are
        # gathered and added on the device inside the call, every rank assembles the same proof
        msm = np.zeros(4 * 3 * fpl + 3 * fpl * deg, dtype=np.uint64) if keep_msm else None
        _lib.check(L.b200_groth16_prove(pk._handle, p(sol.W), p(sol.A), p(sol.B), p(sol.C), n_constraints,
                                        p(r), p(s), p(ar), p(bs), p(krs), p(msm)))
        return Proof(Ar=ar, Bs=bs, Krs=krs, msm=msm)
    # sharded: device part on every rank, one all_gather of 5 partial points, host-side sums
    import torch
    import torch.distributed as dist
    part = np.zeros(4 * 3 * fpl + 3 * fpl * deg, dtype=np.uint64)
    _lib.check(L.b200_groth16_msms(pk._handle, p(sol.W), p(sol.A), p(sol.B), p(sol.C), n_constraints, p(part)))
    t = torch.from_numpy(part.view(np.int64))
    if dist.get_backend(cfg.ProcessGroup) == "nccl":
        t = t.cuda(cfg.DeviceID)
    parts = [torch.empty_like(t) for _ in range(cfg.ShardWorld)]
    dist.all_gather(parts, t, group=cfg.ProcessGroup)
    parts = [x.cpu().numpy().view(np.uint64) for x in parts]
    msm = fold(parts)
    _lib.check(L.b200_groth16_assemble(pk._handle, p(msm), p(r), p(s), p(ar), p(bs), p(krs)))
    return Proof(Ar=ar, Bs=bs, Krs=krs, msm=msm if keep_msm else None)


def ProveSolutionBatch(pk: ProvingKey, sols, *opts: Option, keep_msm: bool = False) -> List[Proof]:
    """Several proofs of one circuit in one call (b200_groth16_prove_batch): the device work of all of them runs as one
    launch sequence, so small proofs stop paying the fixed cost of an MSM and an NTT pipeline each.  Proof k equals
    ProveSolution(pk, sols[k]) with the same r, s; the randomness is drawn r0, s0, r1, s1, ...  One device only."""
    cfg = NewConfig(*opts)
    if len(cfg.Devices) > 1 or cfg.ShardWorld > 1:
        raise ValueError("ProveSolutionBatch: one device and an unsharded key only (WithDevices / WithSharding)")
    sols = list(sols)
    frl, fpl, deg = _lib.CURVE_SHAPES[pk.curve]
    for sol in sols:
        if sol.W.size // frl != pk.nb_wires:
            raise ValueError("witness size does not match the proving key")
    n_constraints = sols[0].A.size // frl if sols else 0
    if any(x.size // frl != n_constraints for sol in sols for x in (sol.A, sol.B, sol.C)):
        raise ValueError("ProveSolutionBatch: the solutions have different constraint counts (one circuit per batch)")
    if not sols:
        return []
    pk.setup_device_pointers(cfg)
    q = _FR_MODULUS[pk.curve]
    rnd = cfg.Randomness or (lambda modulus: secrets.randbelow(modulus))
    rs = np.stack([_fr_to_mont_limbs(rnd(q), pk.curve) for _ in range(2 * len(sols))])
    r, s = np.ascontiguousarray(rs[0::2]), np.ascontiguousarray(rs[1::2])
    k = len(sols)
    vecs = {name: [np.ascontiguousarray(getattr(sol, name), dtype=np.uint64) for sol in sols] for name in "WABC"}
    arrays = {name: (ctypes.c_void_p * k)(*[v.ctypes.data for v in vs]) for name, vs in vecs.items()}
    ar = np.zeros((k, 2 * fpl), dtype=np.uint64)
    krs = np.zeros((k, 2 * fpl), dtype=np.uint64)
    bs = np.zeros((k, 2 * fpl * deg), dtype=np.uint64)
    msm = np.zeros((k, 4 * 3 * fpl + 3 * fpl * deg), dtype=np.uint64) if keep_msm else None
    p = _lib.ptr
    _lib.check(_lib.load().b200_groth16_prove_batch(pk._handle, k, arrays["W"], arrays["A"], arrays["B"], arrays["C"],
                                                    n_constraints, p(r), p(s), p(ar), p(bs), p(krs), p(msm)))
    return [Proof(Ar=ar[i], Bs=bs[i], Krs=krs[i], msm=msm[i] if keep_msm else None) for i in range(k)]


def ProveBatch(r1cs, pk: ProvingKey, full_witnesses, *opts: Option) -> List[Proof]:
    """Prove for several witnesses of one circuit: each is solved, then all are proven in one ProveSolutionBatch call."""
    return ProveSolutionBatch(pk, [r1cs.Solve(w) for w in full_witnesses], *opts)


def Prove(r1cs, pk: ProvingKey, full_witness, *opts: Option) -> Proof:
    """groth16_icicle.go:79-98.  `r1cs.Solve(full_witness)` must return an R1CSSolution
    (the solver itself is CPU code outside this backend, as in the reference)."""
    sol = r1cs.Solve(full_witness)
    return ProveSolution(pk, sol, *opts)
