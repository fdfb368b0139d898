"""b200_msm_batch on the device: out[b] = sum_i s_bi * bases[off + i] for every row b, several MSMs over one base range
in one pipeline.

Known discrete logs (bases P_i = k_i B from the fixed-base batch, a sample checked against the big-int oracle by
test_gpu_msm_plans.build_bases): item b is expected to be (sum_i k_(off+i) s_bi mod r) B, on every curve and group,
plain and precomputed tables, at several batch sizes and base ranges.  Also: the structure of the rows (zero, equal,
negated, a lone scalar at either end), equality with b200_msm item by item, per-item sizes on both sides of every window
change, more bucket sets than a grid's y dimension holds, full-size tables, the Ethereum ceremony's Lagrange basis,
host and device scalars, a batch right after pipelined MSMs that were not joined, and the argument errors and limits."""
import ctypes
import random

import numpy as np
import pytest

from msm_families import pack, seeded
from oracle import corelib, ec, ff, kzg_srs
from oracle.params import BLS12_381, BN254
from points_ntt_cases import fr_transform
from test_gpu_msm_indexed import canonical_affine, to_dev
from test_gpu_msm_plans import BY_NAME, PAIR_IDS, default_window, expected, make_table, need_free
from util import jac_to_affine

pytestmark = pytest.mark.gpu
N_TABLE = 3000


def check_batch(t, curve, group, ks, sc, what, off=0):
    """msm_batch of the (batch, n, limbs) rows sc against bases [off, off + n) of t, every item against its dlog sum"""
    n = sc.shape[1]
    out = t.msm_batch(sc, off=off)
    assert out.shape == (sc.shape[0], 3 * t.coord_limbs)
    got = [jac_to_affine(curve, group, o) for o in out]
    for b in range(sc.shape[0]):
        assert got[b] == expected(curve, group, ks[off:off + n], sc[b]), f"{what} item {b}"
    return out, got


def rows(curve, c, fam, batch, n, rng):
    return np.ascontiguousarray(np.stack([pack(curve, c, fam, n, rng) for _ in range(batch)]))


# ---- 1. every pair, plain and precomputed, several batches and ranges ----------------------------------------------------
@pytest.mark.parametrize("precomp", (False, True), ids=("plain", "precomp"))
@pytest.mark.parametrize("pair", PAIR_IDS)
def test_batches(gpu, monkeypatch, pair, precomp):
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    t, ks = make_table(gpu, curve, group, N_TABLE, precomp)
    rng = seeded("batch", pair, precomp)
    for batch in (1, 2, 5, 33):
        for off in (0, 1000):             # the whole table, and a range that ends at the table's end
            n = N_TABLE - off
            for fam in ("mixed", "uniform"):
                sc = rows(curve, default_window(curve, n), fam, batch, n, rng)
                check_batch(t, curve, group, ks, sc, f"{pair} precomp={precomp} batch={batch} off={off} {fam}", off)
    t.free()


# ---- 2. row structure ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precomp", (False, True), ids=("plain", "precomp"))
@pytest.mark.parametrize("pair", ["bn254-g1", "bls12-381-g2", "bls12-377-g1", "bw6-761-g1"])
def test_row_structure(gpu, monkeypatch, pair, precomp):
    """a zero row is infinity, equal rows give equal canonical points, a negated row the negated point, a lone
    non-zero scalar on the first or the last base that scalar times that base"""
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    t, ks = make_table(gpu, curve, group, N_TABLE, precomp)
    F = ff.base_field(curve, group)
    rng = seeded("rows", pair, precomp)
    sc = rows(curve, default_window(curve, N_TABLE), "mixed", 6, N_TABLE, rng)
    sc[1] = 0
    sc[2] = sc[0]
    sc[3] = ff.pack_elements([(curve.r - s) % curve.r for s in ff.unpack_elements(sc[0], curve.r, curve.fr_limbs)],
                             curve.r, curve.fr_limbs)
    sc[4] = 0
    sc[4, 0] = pack(curve, 4, "uniform", 1, rng)[0]
    sc[5] = 0
    sc[5, -1] = pack(curve, 4, "uniform", 1, rng)[0]
    out, got = check_batch(t, curve, group, ks, sc, f"{pair} precomp={precomp}")
    assert got[1] is ec.INF
    assert canonical_affine(gpu, curve, group, out[2]) == canonical_affine(gpu, curve, group, out[0])
    assert got[3] == ec.affine_neg(F, got[0])
    t.free()


# ---- 3. equal to b200_msm ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precomp", (False, True), ids=("plain", "precomp"))
@pytest.mark.parametrize("pair", ["bn254-g1", "bn254-g2", "bls12-381-g1", "bls12-377-g2", "bw6-761-g1"])
def test_equals_single_msm(gpu, monkeypatch, pair, precomp):
    """canonical affine bytes: batch = 1 equals b200_msm, and every item of a batch of 7 equals its own b200_msm"""
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    t, ks = make_table(gpu, curve, group, N_TABLE, precomp)
    rng = seeded("single", pair, precomp)
    for batch in (1, 7):
        sc = rows(curve, 7, "mixed", batch, N_TABLE - 17, rng)
        out = t.msm_batch(sc, off=17)
        for b in range(batch):
            want = canonical_affine(gpu, curve, group, t.msm(sc[b], off=17))
            assert canonical_affine(gpu, curve, group, out[b]) == want, f"{pair} batch={batch} item {b}"
    t.free()


# ---- 4. window edges -----------------------------------------------------------------------------------------------------
WINDOW_EDGES = sorted({(1 << k) + d for k in range(9, 17) for d in (-1, 0)})


@pytest.mark.parametrize("n", WINDOW_EDGES)
@pytest.mark.parametrize("pair", ["bn254-g1", "bls12-381-g2", "bw6-761-g1"])
def test_window_edges(gpu, monkeypatch, pair, n):
    """per-item n on both sides of every size where msm_window_for changes, batch 3, on a plain 2^16-point table (the
    window follows n, not the table)"""
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    t, ks = make_table(gpu, curve, group, 1 << 16, False)
    sc = rows(curve, default_window(curve, n), "mixed", 3, n, seeded("edges", pair, n))
    check_batch(t, curve, group, ks, sc, f"{pair} n={n}", off=(1 << 16) - n)
    t.free()


# ---- 5. more bucket sets than a grid's y dimension -----------------------------------------------------------------------
def test_more_than_65535_sets(gpu, monkeypatch):
    """BN254 G1, plain, n = 20 (c = 4, 64 windows), batch 1100: 70 400 bucket sets.  The rows repeat 5 distinct vectors
    in a shuffled order, so 5 oracle values check all 1100 outputs"""
    curve, group = BN254, 1
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    n, batch = 20, 1100
    assert default_window(curve, n) == 4 and (curve.r.bit_length() // 4 + 1) * batch == 70400
    t, ks = make_table(gpu, curve, group, N_TABLE, False)
    rng = seeded("many-sets")
    distinct = rows(curve, 4, "mixed", 5, n, rng)
    which = np.array([b % 5 for b in range(batch)])
    random.Random(5).shuffle(which)
    sc = np.ascontiguousarray(distinct[which])
    want = [expected(curve, group, ks[:n], distinct[k]) for k in range(5)]
    out = t.msm_batch(sc)
    for b in range(batch):
        assert jac_to_affine(curve, group, out[b]) == want[which[b]], f"item {b} (vector {which[b]})"
    t.free()


# ---- 6. full size --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("curve,n,precomp,batch", [(BN254, 1 << 20, False, 4), (BLS12_381, 1 << 16, True, 64)],
                         ids=["bn254-plain-2^20-x4", "bls12-381-precomp-2^16-x64"])
def test_full_size(gpu, monkeypatch, curve, n, precomp, batch):
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    need_free(8, "a full-size batch")
    t, ks = make_table(gpu, curve, 1, n, precomp)
    g = np.random.default_rng(seeded("full", curve.name).randrange(1 << 63))
    sc = np.ascontiguousarray(np.stack([pack(curve, default_window(curve, n), "mixed", n, seeded("full", curve.name, b))
                                        for b in range(batch)]))
    sc[g.integers(batch)] = 0
    check_batch(t, curve, 1, ks, sc, f"{curve.name} n={n} precomp={precomp} batch={batch}")
    t.free()


# ---- 7. the Ethereum ceremony --------------------------------------------------------------------------------------------
def test_ethereum_ceremony_blobs(gpu):
    """8 random blobs committed to the ceremony's 4096 Lagrange points (natural order): every item equals b200_msm of
    its blob, and two items equal the MSM of the monomial points with the oracle's inverse NTT of the blob"""
    mono, lag, _ = kzg_srs.load()
    C, logn = BLS12_381, 12
    F = ff.Fp(C.p)
    t = gpu.Table(C.curve_id, 1, ec.pack_points(C, 1, lag), precomp=False)
    rng = random.Random(4844)
    blobs = np.ascontiguousarray(np.stack([ff.pack_elements([rng.randrange(C.r) for _ in range(kzg_srs.N)], C.r, C.fr_limbs)
                                           for _ in range(8)]))
    out = t.msm_batch(blobs)
    for b in range(8):
        assert canonical_affine(gpu, C, 1, out[b]) == canonical_affine(gpu, C, 1, t.msm(blobs[b])), f"blob {b}"
    for b in (0, 7):
        coeffs = fr_transform(C, blobs[b].copy(), logn, True)
        want = ec.from_jac(F, ec.unpack_points(C, 1, corelib.msm(C, 1, ec.pack_points(C, 1, mono), coeffs), ncoords=3)[0])
        assert jac_to_affine(C, 1, out[b]) == want, f"blob {b} by the monomial route"
    t.free()


# ---- 8. placements -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precomp", (False, True), ids=("plain", "precomp"))
@pytest.mark.parametrize("pair", ["bn254-g1", "bls12-381-g2"])
def test_placements(gpu, monkeypatch, pair, precomp):
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    t, ks = make_table(gpu, curve, group, N_TABLE, precomp)
    sc = rows(curve, 6, "uniform", 5, 1234, seeded("placement", pair, precomp))
    host, _ = check_batch(t, curve, group, ks, sc, f"{pair} host scalars", off=100)
    dev = t.msm_batch(to_dev(sc.reshape(5, -1)).reshape(5, 1234, -1), off=100)
    for b in range(5):
        assert canonical_affine(gpu, curve, group, dev[b]) == canonical_affine(gpu, curve, group, host[b]), \
            f"{pair} device scalars item {b}"
    t.free()


# ---- 9. after pipelined MSMs that were not joined ------------------------------------------------------------------------
def test_after_pipelined_msms(gpu, monkeypatch):
    import torch
    curve, group = BN254, 1
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    n = 1 << 16
    t, ks = make_table(gpu, curve, group, n, False)
    rng = seeded("interplay")
    sc = [pack(curve, 12, "uniform", n, rng) for _ in range(2)]
    d_sc = [to_dev(s) for s in sc]
    d_out = [torch.zeros(3 * t.coord_limbs, dtype=torch.int64, device="cuda") for _ in range(2)]
    for k in range(2):
        t.msm_pipelined(d_sc[k], d_out[k], n=n)
    batch = rows(curve, 12, "mixed", 3, n, rng)
    check_batch(t, curve, group, ks, batch, "batch after two pipelined MSMs")
    t.join()
    torch.cuda.synchronize()
    for k in range(2):
        got = jac_to_affine(curve, group, d_out[k].cpu().numpy().view(np.uint64))
        assert got == expected(curve, group, ks, sc[k]), f"pipelined MSM {k}"
    t.free()


# ---- 10. errors and limits -----------------------------------------------------------------------------------------------
def test_errors(gpu, monkeypatch):
    import torch
    c = BN254
    L = gpu.load()
    null = ctypes.c_void_p(0)
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    t, ks = make_table(gpu, c, 1, N_TABLE, False)
    rng = seeded("batch-errors")
    sc = rows(c, 4, "uniform", 3, 100, rng)
    want, _ = check_batch(t, c, 1, ks, sc, "valid call")
    jac = 3 * c.fp_limbs
    out = np.full(3 * jac, 7, dtype=np.uint64)

    def fails(match, rc, buf=out):
        assert rc != 0
        assert match in L.b200_last_error().decode(), L.b200_last_error()
        assert (buf == 7).all(), "the output was written"

    def valid_call_after():
        got = np.zeros_like(out)
        gpu.check(L.b200_msm_batch(t.handle, 0, 100, 3, gpu.ptr(sc), 0, gpu.ptr(got)))
        assert np.array_equal(got.reshape(3, jac), want)

    fails("msm_batch: null table", L.b200_msm_batch(null, 0, 100, 3, gpu.ptr(sc), 0, gpu.ptr(out)))
    fails("msm_batch: null argument", L.b200_msm_batch(t.handle, 0, 100, 3, null, 0, gpu.ptr(out)))
    with pytest.raises(gpu.B200Error, match="msm_batch: null argument"):
        gpu.check(L.b200_msm_batch(t.handle, 0, 100, 3, gpu.ptr(sc), 0, null))
    fails("msm_batch: range [off, off+n) exceeds the table",
          L.b200_msm_batch(t.handle, N_TABLE - 99, 100, 3, gpu.ptr(sc), 0, gpu.ptr(out)))
    fails("msm_batch: range [off, off+n) exceeds the table",
          L.b200_msm_batch(t.handle, 2 ** 63, 100, 3, gpu.ptr(sc), 0, gpu.ptr(out)))
    valid_call_after()
    # batch = 0 writes nothing; n = 0 writes `batch` points at infinity (null scalars accepted for both)
    gpu.check(L.b200_msm_batch(t.handle, 0, 100, 0, null, 0, gpu.ptr(out)))
    assert (out == 7).all()
    gpu.check(L.b200_msm_batch(t.handle, 0, 0, 3, null, 0, gpu.ptr(out)))
    assert all(jac_to_affine(c, 1, o) is ec.INF for o in out.reshape(3, jac))
    out[:] = 7
    # 2^31 entries: n = 16 (c = 4, 64 windows), batch 2^21 - a real device buffer of all 2^21 * 16 scalars (1 GiB)
    need_free(2, "the entry-limit test")
    batch = 1 << 21
    d_big = torch.zeros((batch * 16 * c.fr_limbs,), dtype=torch.int64, device="cuda")
    big_out = np.full(batch * jac, 7, dtype=np.uint64)
    fails("msm_batch: batch * n * windows exceeds 2^31 entries",
          L.b200_msm_batch(t.handle, 0, 16, batch, gpu.ptr(d_big), 1, gpu.ptr(big_out)), big_out)
    del d_big, big_out
    valid_call_after()
    # 2^32 bucket keys: a table precomputed at c = 16 (one set of 2^15 buckets per item), n = 1, batch 2^17
    monkeypatch.setenv("GB200_MSM_WINDOW", "16")
    tp, _ = make_table(gpu, c, 1, N_TABLE, True)
    monkeypatch.delenv("GB200_MSM_WINDOW")
    assert tp.info()["window_bits"] == 16
    batch = 1 << 17
    d_keys = torch.zeros((batch * c.fr_limbs,), dtype=torch.int64, device="cuda")
    key_out = np.full(batch * jac, 7, dtype=np.uint64)
    fails("msm_batch: batch * bucket sets * 2^(c-1) exceeds",
          L.b200_msm_batch(tp.handle, 0, 1, batch, gpu.ptr(d_keys), 1, gpu.ptr(key_out)), key_out)
    del d_keys, key_out
    valid_call_after()
    tp.free()
    t.free()
