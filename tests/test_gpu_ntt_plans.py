"""The radix-2 Fr NTT (k_ntt_pass, gnark_b200/csrc/ntt_impl.cuh) on all four curves, limb for limb against the C++ oracle
(oracle/corelib.py) with the same generator and coset:

- every pass plan of the tile overrides GB200_NTT_TILE_LOG = 6..11 at 2^0..2^17 (and 2^19, where the 2^6 tile needs
  five passes), on uniform residues and on the structured vectors of tests/ntt_cases.py;
- production sizes: 2^22 and 2^24 on BLS12-377, 2^20..2^24 on BW6-761, 2^26 (the quotient domain of a 2^24 PLONK
  circuit) on BN254 and BLS12-381;
- the batched kernel (b200_ntt_batch) at one, two and three passes of three tiles, from host and device memory;
- custom generators (another primitive root of unity) and cosets (w_2n as ICICLE passes it, a random element);
- computeH at 2^20 and 2^22 with padded and full inputs, host and device outputs;
- the domain sizes b200_ntt_domain_new refuses."""
import random

import numpy as np
import pytest

import ntt_cases as nc
from oracle import corelib, ff
from oracle.params import CURVES

pytestmark = pytest.mark.gpu
ALL = list(CURVES.values())
IDS = lambda c: c.name
TILE_ENV = "GB200_NTT_TILE_LOG"
TILES = tuple(range(6, 12))
SWEEP_LOGN = tuple(range(18)) + (19,)
DIF, DIT = 0, 1
MODES = [(inv, dec, cos) for inv in (False, True) for dec in (DIF, DIT) for cos in (False, True)]
MIXED = [(False, DIF, False), (False, DIT, True), (True, DIF, True), (True, DIT, False)]


def _gen(*key):
    return np.random.default_rng(random.Random("/".join(map(str, key))).randrange(1 << 63))


def _domain(gpu, monkeypatch, c, logn, tile=None, **kw):
    """a device domain planned with tile 2^tile (None: the variable unset, i.e. the default tile); the variable is read
    when the domain is created"""
    if tile is None:
        monkeypatch.delenv(TILE_ENV, raising=False)
    else:
        monkeypatch.setenv(TILE_ENV, str(tile))
    return gpu.Domain(c.curve_id, logn, **kw)


def _root(c, logn):
    return pow(c.root_of_unity, 1 << (c.two_adicity - logn), c.r)


def _bitrev(k, logn):
    return int(format(k, f"0{logn}b")[::-1], 2) if logn else 0


def _to_device(a):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a).view(np.int64).reshape(-1)).cuda()
    torch.cuda.synchronize()          # the library runs on its own stream: the upload must be done before it reads t
    return t


def _from_device(t, shape):
    return t.cpu().numpy().view(np.uint64).reshape(shape)


# ---- plan sweep ----------------------------------------------------------------------------------------------------
def test_sweep_reaches_every_plan_shape():
    """what the sweep below covers, by the planner's restatement (pinned to the C++ in test_ntt_plans_emulation.py):
    every pass count from 1 to 5, and a first pass shorter than the tile.  The clamp of a later pass's contiguous bits
    to its lo_bit never binds: the first pass spans the whole tile whenever another pass follows, so every later pass
    has lo_bit >= tile > tile - S.  Should a planner change make it bind, this test says so."""
    plans = {(logn, t): nc.make_plan(logn, t) for logn in SWEEP_LOGN for t in TILES}
    assert {len(p) for p in plans.values()} == {1, 2, 3, 4, 5}
    assert any(0 < p[0][1] < t for (logn, t), p in plans.items())
    assert not any(nc.cb_clamped(logn, t) for logn, t in plans)
    assert not any(nc.cb_clamped(logn, t) for logn in range(31) for t in range(3, 12))


@pytest.mark.parametrize("logn", SWEEP_LOGN, ids=lambda l: f"log{l}")
@pytest.mark.parametrize("c", ALL, ids=IDS)
def test_plan_sweep(gpu, monkeypatch, c, logn):
    """every family, at every tile 2^6..2^11: all eight modes up to 2^12, the four mixed modes above"""
    n = 1 << logn
    modes = MODES if logn <= 12 else MIXED
    g = _gen("sweep", c.name, logn)
    inputs = {f: nc.family(c, f, n, g) for f in nc.FAMILIES}
    want = {(f, m): corelib.ntt(c, a.copy(), logn, *m) for f, a in inputs.items() for m in modes}
    for tile in TILES:
        d = _domain(gpu, monkeypatch, c, logn, tile)
        try:
            for (f, (inv, dec, cos)), w in want.items():
                got = d.ntt(inputs[f].copy(), inverse=inv, decimation=dec, on_coset=cos)
                assert np.array_equal(got, w), (c.name, logn, tile, nc.make_plan(logn, tile), f, inv, dec, cos)
        finally:
            d.free()


@pytest.mark.parametrize("c", ALL, ids=IDS)
def test_tile_override_fallback(gpu, monkeypatch, c):
    """values outside 6..11, a non-number and an empty value plan with the default tile, as the variable unset does:
    the output is byte-identical to tile 8's, which equals the oracle's"""
    logn = 14
    n = 1 << logn
    x = nc.uniform(c, n, _gen("fallback", c.name))

    def run(tile):
        d = _domain(gpu, monkeypatch, c, logn, tile)
        try:
            return [d.ntt(x.copy(), inverse=inv, decimation=dec, on_coset=cos) for inv, dec, cos in MIXED]
        finally:
            d.free()

    ref = run(8)
    for (inv, dec, cos), r in zip(MIXED, ref):
        assert np.array_equal(r, corelib.ntt(c, x.copy(), logn, inv, dec, cos)), (c.name, inv, dec, cos)
    for tile in (None, 5, 12, "abc", ""):
        assert all(np.array_equal(a, b) for a, b in zip(run(tile), ref)), (c.name, tile)


# ---- production sizes ------------------------------------------------------------------------------------------------
PRODUCTION = [("bls12-377", 22), ("bls12-377", 24), ("bw6-761", 20), ("bw6-761", 22), ("bw6-761", 24)]


@pytest.mark.parametrize("cname,logn", PRODUCTION)
def test_production_size_vs_oracle(gpu, monkeypatch, cname, logn):
    """forward DIF plain and inverse DIT on the coset through host buffers; at the curve's smallest size also through
    a device tensor"""
    c = CURVES[cname]
    n = 1 << logn
    a = nc.uniform(c, n, _gen("production", cname, logn))
    device = logn == min(l for cn, l in PRODUCTION if cn == cname)
    d = _domain(gpu, monkeypatch, c, logn)
    try:
        for inv, dec, cos in ((False, DIF, False), (True, DIT, True)):
            want = corelib.ntt(c, a.copy(), logn, inv, dec, cos)
            got = d.ntt(a.copy(), inverse=inv, decimation=dec, on_coset=cos)
            assert np.array_equal(got, want), (cname, logn, inv, dec, cos)
            del got
            if device:
                t = _to_device(a)
                d.ntt(t, inverse=inv, decimation=dec, on_coset=cos, on_device=True)
                assert np.array_equal(_from_device(t, a.shape), want), (cname, logn, inv, dec, cos, "device")
                del t
    finally:
        d.free()


def _poly_eval(c, a, x, block=1 << 13):
    """p(x) = sum a_j x^j (a: Montgomery coefficients) by the oracle: the dot product of every block of coefficients
    with [x^l, l < block], then Horner in x^block over the blocks"""
    rows = a.reshape(-1, block, c.fr_limbs)
    pw = corelib.fr_geometric(c, 1, x, block)
    acc, xb = 0, pow(x, block, c.r)
    for h in range(rows.shape[0] - 1, -1, -1):
        acc = (acc * xb + corelib.fr_dot(c, rows[h], pw)) % c.r
    return acc


@pytest.mark.parametrize("cname", ("bn254", "bls12-381"))
def test_quotient_domain_size(gpu, monkeypatch, cname):
    """2^26 (PLONK's quotient domain of a 2^24 circuit), where a full oracle transform costs minutes: forward DIF plain
    and on the coset, X at position bitrev(k) equals p(w^k) (p(g w^k) on the coset) at k = 0, n/2, n - 1, evaluated by
    the oracle's dot products with the powers; the inverse DIT undoes it bit for bit.  The coset transform is repeated
    on a device tensor and must give the same bytes."""
    from concurrent.futures import ThreadPoolExecutor

    import torch
    c = CURVES[cname]
    logn = 26
    n, r, L = 1 << logn, c.r, c.fr_limbs
    a = nc.uniform(c, n, _gen("quotient", cname))
    w = _root(c, logn)
    ks = (0, n // 2, n - 1)
    d = _domain(gpu, monkeypatch, c, logn)
    try:
        for cos in (False, True):
            points = [pow(w, k, r) * (c.mult_gen if cos else 1) % r for k in ks]
            with ThreadPoolExecutor(len(points)) as ex:          # the oracle calls release the GIL
                evals = ex.map(lambda x: _poly_eval(c, a, x), points)
                y = d.ntt(a.copy(), inverse=False, decimation=DIF, on_coset=cos)
                for k, want in zip(ks, evals):
                    assert ff.unpack_elements(y[_bitrev(k, logn)], r, L)[0] == want, (cname, cos, k)
            if cos:
                t = _to_device(a)
                d.ntt(t, inverse=False, decimation=DIF, on_coset=True, on_device=True)
                assert torch.equal(t, _to_device(y)), (cname, "device")
                del t
                torch.cuda.empty_cache()
            d.ntt(y, inverse=True, decimation=DIT, on_coset=cos)
            assert np.array_equal(y, a), (cname, cos, "round trip")
            del y
    finally:
        d.free()


# ---- batched NTT -----------------------------------------------------------------------------------------------------
BATCH_TILES = (6, 8, 11)
# tile 6: 1, 2, 3, 4 passes; tile 8: 1, 1, 2, 2, 3; tile 11: 1, 1, 2, 2 (and 3 at 2^21, on BN254)
BATCH_CASES = [(c, logn) for c in ALL for logn in (6, 10, 13, 16)] + [(CURVES["bn254"], 21)]


@pytest.mark.parametrize("c,logn", BATCH_CASES, ids=[f"{c.name}-log{l}" for c, l in BATCH_CASES])
def test_batch_vs_oracle(gpu, monkeypatch, c, logn):
    """batches of 3 and 5 distinct vectors, all eight modes, each item against the oracle; at tile 8 the batch of 5
    also from device memory"""
    n, L = 1 << logn, c.fr_limbs
    x = nc.uniform(c, 5 * n, _gen("batch", c.name, logn))
    want = {m: np.stack([corelib.ntt(c, x[b * n:(b + 1) * n].copy(), logn, *m) for b in range(5)]) for m in MODES}
    for tile in BATCH_TILES:
        d = _domain(gpu, monkeypatch, c, logn, tile)
        plan = nc.make_plan(logn, tile)
        try:
            for batch in (3, 5):
                for m in MODES:
                    inv, dec, cos = m
                    got = d.ntt_batch(x[:batch * n].copy(), inverse=inv, decimation=dec, on_coset=cos)
                    got = got.reshape(batch, n, L)
                    for b in range(batch):
                        assert np.array_equal(got[b], want[m][b]), (c.name, logn, tile, plan, batch, b, m)
            if tile == 8:
                for m in MODES:
                    inv, dec, cos = m
                    t = _to_device(x)
                    d.ntt_batch(t, inverse=inv, decimation=dec, on_coset=cos, on_device=True)
                    got = _from_device(t, (5, n, L))
                    for b in range(5):
                        assert np.array_equal(got[b], want[m][b]), (c.name, logn, "device", b, m)
        finally:
            d.free()


# ---- custom domains --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("logn", (1, 5, 12, 16), ids=lambda l: f"log{l}")
@pytest.mark.parametrize("c", ALL, ids=IDS)
def test_custom_generator_and_coset(gpu, monkeypatch, c, logn):
    """generator w_n^k for an odd k (another primitive n-th root of unity), coset w_2n (ICICLE's convention) and a
    random element outside the subgroup: a batch of 3 and a single transform, all eight modes"""
    n, r, L = 1 << logn, c.r, c.fr_limbs
    rng = random.Random(f"custom/{c.name}/{logn}")
    k = rng.randrange(3, n, 2) if n > 4 else 3
    gen = pow(_root(c, logn), k, r)
    assert pow(gen, n // 2, r) == r - 1                       # primitive: order exactly n
    w2n = _root(c, logn + 1)
    outside = rng.randrange(2, r)
    while pow(outside, n, r) == 1:
        outside = rng.randrange(2, r)
    pk = lambda v: ff.pack_elements([v], r, L)
    for cname, coset in (("w2n", w2n), ("random", outside)):
        x = nc.uniform(c, 3 * n, _gen("custom", c.name, logn, cname))
        d = _domain(gpu, monkeypatch, c, logn, generator=pk(gen), coset_gen=pk(coset))
        try:
            for inv, dec, cos in MODES:
                want = [corelib.ntt(c, x[b * n:(b + 1) * n].copy(), logn, inv, dec, cos, generator=gen, coset_gen=coset)
                        for b in range(3)]
                got = d.ntt_batch(x.copy(), inverse=inv, decimation=dec, on_coset=cos).reshape(3, n, L)
                for b in range(3):
                    assert np.array_equal(got[b], want[b]), (c.name, logn, k, cname, b, inv, dec, cos)
                one = d.ntt(np.ascontiguousarray(x[:n]), inverse=inv, decimation=dec, on_coset=cos)
                assert np.array_equal(one, want[0]), (c.name, logn, k, cname, "single", inv, dec, cos)
        finally:
            d.free()


# ---- computeH ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cname,logn", [("bls12-377", 20), ("bw6-761", 20), ("bls12-377", 22)])
def test_compute_h_vs_oracle(gpu, monkeypatch, cname, logn):
    """a padded length (n - 12345) and a full one; host inputs and output, then device inputs and output"""
    c = CURVES[cname]
    n, L = 1 << logn, c.fr_limbs
    g = _gen("compute_h", cname, logn)
    d = _domain(gpu, monkeypatch, c, logn)
    try:
        for length in (n - 12345, n):
            abc = [nc.uniform(c, length, g) for _ in range(3)]
            padded = [np.concatenate([v, np.zeros((n - length, L), dtype=np.uint64)]) for v in abc]
            want = corelib.compute_h(c, *padded, logn)
            del padded
            got = d.compute_h(*abc, length=length)
            assert np.array_equal(got, want), (cname, logn, length, "host")
            import torch
            dev = [_to_device(v) for v in abc]
            out = torch.zeros(n * L, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            d.compute_h(*dev, length=length, on_device=True, out=out, out_on_device=True)
            assert np.array_equal(_from_device(out, (n, L)), want), (cname, logn, length, "device")
            del dev, out
    finally:
        d.free()


# ---- refusals ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", ALL, ids=IDS)
def test_domain_size_refusals(gpu, monkeypatch, c):
    """log n past the field's 2-adicity, and log n = 31, are refused with the reason; a valid domain created afterwards
    transforms correctly"""
    for logn in (c.two_adicity + 1, 31):
        with pytest.raises(gpu.B200Error, match="log2n exceeds the field's 2-adicity"):
            gpu.Domain(c.curve_id, logn)
    logn = 9
    x = nc.uniform(c, 1 << logn, _gen("after-refusal", c.name))
    d = _domain(gpu, monkeypatch, c, logn)
    try:
        for inv, dec, cos in MODES:
            got = d.ntt(x.copy(), inverse=inv, decimation=dec, on_coset=cos)
            assert np.array_equal(got, corelib.ntt(c, x.copy(), logn, inv, dec, cos)), (c.name, inv, dec, cos)
    finally:
        d.free()
