"""KZG on the device: b200_poly_eval_batch, b200_kzg_open_batch and b200_kzg_fold_open on all four curves.

Known discrete logs (SRS points P_i = k_i B from the fixed-base batch, test_gpu_msm_plans.make_table): opening b must be
(sum_i k_i q_b[i]) B with q_b the oracle's quotient of row b, and value b the oracle's Horner value.  Also: agreement with
the single-polynomial path (b200_poly_div_by_linear + b200_msm) and the PLONK-style fold (axpy loop + division + MSM),
every proof checked with the big-int BLS12-381 pairing on the Ethereum ceremony SRS (whose trapdoor nobody knows), the
refusals with every output untouched, host and device polynomials, and a call right after pipelined MSMs not joined."""
import ctypes
import random

import numpy as np
import pytest

from oracle import corelib, ec, ff, kzg_srs, ntt, plonk
from oracle.params import BLS12_381, BN254, CURVES
from test_gpu_msm_indexed import canonical_affine, to_dev
from test_gpu_msm_plans import build_bases, make_table, need_free
from util import jac_to_affine, pick_base

pytestmark = pytest.mark.gpu
CURVE_LIST = list(CURVES.values())
IDS = [c.name for c in CURVE_LIST]


def rand_rows(curve, batch, n, rng):
    rows = [[rng.randrange(curve.r) for _ in range(n)] for _ in range(batch)]
    if batch >= 3:
        rows[1] = [0] * n
        rows[2] = list(rows[0])
    return rows


def pack_rows(curve, rows, n):
    flat = [v for row in rows for v in row]
    return np.ascontiguousarray(ff.pack_elements(flat, curve.r, curve.fr_limbs).reshape(len(rows), n, curve.fr_limbs))


def make_points(curve, batch, rng):
    """a mix of 0, 1, r - 1, a root of unity and random points (one shared by two items)"""
    w = pow(curve.root_of_unity, 1 << (curve.two_adicity - 12), curve.r)
    shared = rng.randrange(curve.r)
    cycle = [rng.randrange(curve.r), 0, shared, 1, curve.r - 1, w, shared]
    return [cycle[b % len(cycle)] for b in range(batch)]


def pack_fr(curve, vals):
    return np.ascontiguousarray(ff.pack_elements(vals, curve.r, curve.fr_limbs))


def unpack_fr(curve, arr):
    return ff.unpack_elements(np.ascontiguousarray(arr).reshape(-1), curve.r, curve.fr_limbs)


def check_open(t, curve, ks, rows, n, pts, what, on_device=False):
    """kzg_open_batch of rows at pts against the oracle's values and the known discrete logs ks of the SRS"""
    F, B = pick_base(curve, 1)
    polys = pack_rows(curve, rows, n)
    vals, proofs = t.kzg_open_batch(to_dev(polys) if on_device else polys, pack_fr(curve, pts), on_device=on_device)
    got_v = unpack_fr(curve, vals)
    for b, row in enumerate(rows):
        q, y = plonk.div_by_linear(curve.r, row, pts[b])
        assert got_v[b] == y == ntt.poly_eval(curve.r, row, pts[b]), f"{what} item {b}: value"
        s = corelib.fr_dot(curve, np.ascontiguousarray(ks[:n - 1]), pack_fr(curve, q)) if n > 1 else 0
        assert jac_to_affine(curve, 1, proofs[b]) == ec.scalar_mul(F, s, B), f"{what} item {b}: proof"
    return vals, proofs


# ---- 1. known discrete logs: batches, sizes, an SRS of exactly n - 1 points -----------------------------------------------
@pytest.mark.parametrize("precomp", (False, True), ids=("plain", "precomp"))
@pytest.mark.parametrize("curve", CURVE_LIST, ids=IDS)
def test_open_known_dlogs(gpu, monkeypatch, curve, precomp):
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    T = 3000
    t, ks = make_table(gpu, curve, 1, T, precomp)
    for batch, n in ((1, 0), (1, 1), (2, 1), (1, 2), (2, 3), (5, 1025), (33, 300), (5, 2049), (2, T + 1)):
        rng = random.Random(f"kzg-open-{curve.name}-{precomp}-{batch}-{n}")
        check_open(t, curve, ks, rand_rows(curve, batch, n, rng), n, make_points(curve, batch, rng),
                   f"{curve.name} precomp={precomp} batch={batch} n={n}")
    t.free()


@pytest.mark.parametrize("curve", CURVE_LIST, ids=IDS)
def test_open_large(gpu, monkeypatch, curve):
    """n = 2^16 + 3 on an SRS of exactly n - 1 points (64 scan blocks per row, a second scan level of one block), and on
    BN254 n = 2^20 + 3 (1025 scan blocks per row: the block totals take a second level of two blocks)"""
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    n = (1 << 16) + 3
    t, ks = make_table(gpu, curve, 1, n - 1, False)
    rng = random.Random(f"kzg-large-{curve.name}")
    check_open(t, curve, ks, rand_rows(curve, 2, n, rng), n, [rng.randrange(curve.r), 0], f"{curve.name} n=2^16+3")
    t.free()
    if curve is BN254:
        need_free(4, "the 2^20 + 3 opening")
        n = (1 << 20) + 3
        F, B, ks, d_pts = build_bases(gpu, curve, 1, n - 1, ("kzg", n))
        t = gpu.Table(curve.curve_id, 1, d_pts, precomp=False, n=n - 1, on_device=True)
        check_open(t, curve, ks, rand_rows(curve, 2, n, rng), n, [rng.randrange(curve.r), 1], "bn254 n=2^20+3",
                   on_device=True)
        t.free()


@pytest.mark.parametrize("curve", CURVE_LIST, ids=IDS)
def test_more_than_65535_items(gpu, monkeypatch, curve):
    """65 537 polynomials of 3 coefficients: the launches are split at the grid's 65 535 rows; every value against the
    oracle, every proof against (k_0 q_0 + k_1 q_1) B from the fixed-base batch, and the evaluation entry point too.
    A precomputed table keeps one bucket set per item; on a plain one BW6-761's 63 sets of 2^5 buckets per item would
    take about 50 GB for this batch."""
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    batch, n = 65537, 3
    t, ks = make_table(gpu, curve, 1, n - 1, True)
    F, B = pick_base(curve, 1)
    rng = random.Random(f"kzg-many-{curve.name}")
    rows = [[rng.randrange(curve.r) for _ in range(n)] for _ in range(batch)]
    pts = [rng.randrange(curve.r) if b % 5 else 0 for b in range(batch)]
    polys = pack_rows(curve, rows, n)
    vals, proofs = t.kzg_open_batch(polys, pack_fr(curve, pts))
    k0, k1 = unpack_fr(curve, ks[:2])
    want_s, want_v = [], []
    for row, z in zip(rows, pts):
        q, y = plonk.div_by_linear(curve.r, row, z)
        want_v.append(y)
        want_s.append((k0 * q[0] + k1 * q[1]) % curve.r)
    assert unpack_fr(curve, vals) == want_v
    assert unpack_fr(curve, gpu.poly_eval_batch(0, curve.curve_id, polys, pack_fr(curve, pts))) == want_v
    want_p = gpu.fixed_base_batch(curve.curve_id, 1, ec.pack_points(curve, 1, [B]), pack_fr(curve, want_s))
    got_p = np.stack([gpu.point_to_affine(curve.curve_id, 1, np.ascontiguousarray(p)) for p in proofs])
    bad = [b for b in range(batch) if not np.array_equal(got_p[b], want_p[b])]
    assert not bad, f"{curve.name}: {len(bad)} proofs differ, first {bad[:5]}"
    t.free()


# ---- 2. agreement with the existing single-polynomial path and the PLONK-style fold -----------------------------------------
@pytest.mark.parametrize("curve", CURVE_LIST, ids=IDS)
def test_agrees_with_existing_paths(gpu, monkeypatch, curve):
    import torch
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    T, n = 3000, 3001
    t, ks = make_table(gpu, curve, 1, T, False)
    rng = random.Random(f"kzg-agree-{curve.name}")
    for z in (rng.randrange(curve.r), 0):
        row = [rng.randrange(curve.r) for _ in range(n)]
        p = pack_rows(curve, [row], n)
        vals, proofs = t.kzg_open_batch(p, pack_fr(curve, [z]))
        d = to_dev(p.reshape(-1))
        y = gpu.poly_div_by_linear(0, curve.curve_id, d, n, pack_fr(curve, [z]))
        torch.cuda.synchronize()
        want = t.msm(d, n=n - 1, on_device=True)
        assert np.array_equal(vals[0], y), f"{curve.name} z={z}: value"
        assert canonical_affine(gpu, curve, 1, proofs[0]) == canonical_affine(gpu, curve, 1, want), f"{curve.name} z={z}"
    # fold: f = sum_b v^b p_b as b200_plonk_batch_open builds it (axpy from gamma^0 = 1), then division and MSM
    batch = 6
    rows = rand_rows(curve, batch, n, rng)
    polys = pack_rows(curve, rows, n)
    z, gamma = rng.randrange(curve.r), rng.randrange(curve.r)
    got = t.kzg_fold_open(polys, pack_fr(curve, [z]), pack_fr(curve, [gamma]))
    fold = torch.zeros(n * curve.fr_limbs, dtype=torch.int64, device="cuda")
    d_rows = [to_dev(polys[b].reshape(-1)) for b in range(batch)]
    for b in range(batch):
        gpu.vec_axpy(0, curve.curve_id, fold, pack_fr(curve, [pow(gamma, b, curve.r)]), d_rows[b], n)
    gpu.poly_div_by_linear(0, curve.curve_id, fold, n, pack_fr(curve, [z]))
    torch.cuda.synchronize()
    want = t.msm(fold, n=n - 1, on_device=True)
    assert canonical_affine(gpu, curve, 1, got) == canonical_affine(gpu, curve, 1, want), f"{curve.name} fold"
    # and from device polynomials
    got_dev = t.kzg_fold_open(to_dev(polys), pack_fr(curve, [z]), pack_fr(curve, [gamma]), on_device=True)
    assert canonical_affine(gpu, curve, 1, got_dev) == canonical_affine(gpu, curve, 1, got), f"{curve.name} fold, device"
    t.free()


# ---- 3. external pin: the Ethereum ceremony SRS, checked with the pairing -------------------------------------------------
def test_ethereum_ceremony_pairing(gpu):
    """random 4096-coefficient polynomials opened on the ceremony's monomial G1 points: e(pi, [tau]G2 - z G2) =
    e(C - y G1, G2) for every opening (C from b200_msm_batch, the batch commitment), and for one folded proof against
    sum gamma^b C_b and sum gamma^b y_b"""
    from oracle import pairing_bls12_381 as pr
    C = BLS12_381
    mono, _, g2 = kzg_srs.load()
    F, F2 = ff.Fp(C.p), ff.base_field(C, 2)
    t = gpu.Table(C.curve_id, 1, ec.pack_points(C, 1, mono), precomp=False)
    rng = random.Random("kzg-eth")
    batch, n = 3, kzg_srs.N
    rows = [[rng.randrange(C.r) for _ in range(n)] for _ in range(batch)]
    polys = pack_rows(C, rows, n)
    pts = [rng.randrange(C.r), 0, rng.randrange(C.r)]
    commits = [jac_to_affine(C, 1, c) for c in t.msm_batch(polys)]
    vals, proofs = t.kzg_open_batch(polys, pack_fr(C, pts))
    ys = unpack_fr(C, vals)
    G1, G2, tauG2 = mono[0], g2[0], g2[1]

    def verifies(pi, cm, z, y):
        lhs_g2 = ec.affine_add(F2, tauG2, ec.affine_neg(F2, ec.scalar_mul(F2, z, G2)))
        rhs_g1 = ec.affine_add(F, cm, ec.affine_neg(F, ec.scalar_mul(F, y, G1)))
        return pr.pairing_product_is_one([(pi, lhs_g2), (ec.affine_neg(F, rhs_g1), G2)])

    for b in range(batch):
        assert ys[b] == ntt.poly_eval(C.r, rows[b], pts[b]), f"value {b}"
        pi = jac_to_affine(C, 1, proofs[b])
        assert verifies(pi, commits[b], pts[b], ys[b]), f"opening {b} fails the pairing check"
        if b == 0:
            assert not verifies(pi, commits[b], pts[b], (ys[b] + 1) % C.r), "the check accepts a wrong value"
    z, gamma = rng.randrange(C.r), rng.randrange(C.r)
    ys = unpack_fr(C, gpu.poly_eval_batch(0, C.curve_id, polys, pack_fr(C, [z] * batch)))
    H = jac_to_affine(C, 1, t.kzg_fold_open(polys, pack_fr(C, [z]), pack_fr(C, [gamma])))
    cf, yf = None, 0
    for b in range(batch):
        cf = ec.affine_add(F, cf, ec.scalar_mul(F, pow(gamma, b, C.r), commits[b]))
        yf = (yf + pow(gamma, b, C.r) * ys[b]) % C.r
    assert verifies(H, cf, z, yf), "the folded opening fails the pairing check"
    t.free()


# ---- 4. refusals, degenerate sizes, placements, ordering -------------------------------------------------------------------
@pytest.mark.parametrize("curve", CURVE_LIST, ids=IDS)
def test_refusals_and_degenerate_sizes(gpu, monkeypatch, curve):
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    L = gpu.load()
    P = gpu.ptr
    null = ctypes.c_void_p(0)
    T = 100
    t, ks = make_table(gpu, curve, 1, T, False)
    t2, _ = make_table(gpu, curve, 2, T, False)
    fl, jac = curve.fr_limbs, 3 * curve.fp_limbs
    rng = random.Random(f"kzg-refuse-{curve.name}")
    n, batch = 50, 3
    rows = rand_rows(curve, batch, n, rng)
    polys = pack_rows(curve, rows, n)
    pts = pack_fr(curve, make_points(curve, batch, rng))
    z, gamma = pack_fr(curve, [5]), pack_fr(curve, [7])
    vals = np.full(batch * fl, 7, dtype=np.uint64)
    proofs = np.full(batch * jac, 7, dtype=np.uint64)

    def fails(match, rc):
        assert rc != 0
        assert match in L.b200_last_error().decode(), L.b200_last_error()
        assert (vals == 7).all() and (proofs == 7).all(), f"an output was written ({match})"

    op = lambda tab, p, nn, bb: L.b200_kzg_open_batch(tab, P(p), nn, bb, 0, P(pts), P(vals), P(proofs))
    fo = lambda tab, p, nn, bb: L.b200_kzg_fold_open(tab, P(p), nn, bb, 0, P(z), P(gamma), P(proofs))
    fails("kzg_open_batch: null table", op(null, polys, n, batch))
    fails("kzg_fold_open: null table", fo(null, polys, n, batch))
    fails("kzg_open_batch: null argument", op(t.handle, None, n, batch))
    fails("kzg_open_batch: null argument", L.b200_kzg_open_batch(t.handle, P(polys), n, batch, 0, null, P(vals), P(proofs)))
    fails("kzg_open_batch: null argument", L.b200_kzg_open_batch(t.handle, P(polys), n, batch, 0, P(pts), null, P(proofs)))
    fails("kzg_fold_open: null argument", L.b200_kzg_fold_open(t.handle, P(polys), n, batch, 0, P(z), null, P(proofs)))
    fails("poly_eval_batch: null argument", L.b200_poly_eval_batch(0, curve.curve_id, P(polys), n, batch, 0, null, P(vals)))
    fails("kzg_open_batch: the SRS table holds G2 points", op(t2.handle, polys, n, batch))
    fails("kzg_fold_open: the SRS table holds G2 points", fo(t2.handle, polys, n, batch))
    fails("kzg_open_batch: n - 1 = 101 quotient coefficients exceed the SRS's 100 points", op(t.handle, polys, T + 2, batch))
    fails("kzg_fold_open: n - 1 = 101 quotient coefficients exceed", fo(t.handle, polys, T + 2, batch))
    fails("kzg_open_batch: batch * n overflows", op(t.handle, polys, T, 1 << 60))
    fails("kzg_fold_open: batch * n overflows", fo(t.handle, polys, T, 1 << 60))
    fails("poly_eval_batch: batch * n overflows", L.b200_poly_eval_batch(0, curve.curve_id, P(polys), 1 << 40, 1 << 40, 0,
                                                                          P(pts), P(vals)))
    # the quotient MSM's entry limit: n - 1 = 16 scalars at the smallest window; nothing is read before the refusal
    bits, c = curve.r.bit_length(), 4            # the window of 17 points on a plain table, raised to <= 64 windows
    while bits // c + 1 > 64:
        c += 1
    nwin = bits // c + 1
    most = min(((1 << 31) - 1) // (16 * nwin), ((1 << 31) - 2) // (nwin << (c - 1)))
    fails(f"at most {most} items of this n fit", op(t.handle, polys, 17, most + 1))
    # batch = 0 writes nothing
    gpu.check(op(t.handle, polys, n, 0))
    gpu.check(fo(t.handle, polys, n, 0))
    gpu.check(L.b200_poly_eval_batch(0, curve.curve_id, P(polys), n, 0, 0, P(pts), P(vals)))
    assert (vals == 7).all() and (proofs == 7).all()
    # n = 0: value 0 and the point at infinity; n = 1: value c_0 and the point at infinity (null polynomials accepted at 0)
    gpu.check(L.b200_kzg_open_batch(t.handle, null, 0, batch, 0, P(pts), P(vals), P(proofs)))
    assert unpack_fr(curve, vals) == [0] * batch
    assert all(jac_to_affine(curve, 1, p) is ec.INF for p in proofs.reshape(batch, jac))
    one = pack_rows(curve, [row[:1] for row in rows], 1)
    v1, p1 = t.kzg_open_batch(one, pts)
    assert unpack_fr(curve, v1) == [row[0] for row in rows]
    assert all(jac_to_affine(curve, 1, p) is ec.INF for p in p1)
    assert jac_to_affine(curve, 1, t.kzg_fold_open(one, z, gamma)) is ec.INF
    e0 = np.zeros(jac, dtype=np.uint64)
    gpu.check(L.b200_kzg_fold_open(t.handle, null, 0, batch, 0, P(z), P(gamma), P(e0)))
    assert jac_to_affine(curve, 1, e0) is ec.INF
    # host and device polynomials give the same results, and a valid call after the refusals is right
    vh, ph = check_open(t, curve, ks, rows, n, unpack_fr(curve, pts), f"{curve.name} host")
    vd, pdv = check_open(t, curve, ks, rows, n, unpack_fr(curve, pts), f"{curve.name} device", on_device=True)
    assert np.array_equal(vh, vd) and np.array_equal(ph, pdv)
    ev = gpu.poly_eval_batch(0, curve.curve_id, to_dev(polys), pts, on_device=True)
    assert np.array_equal(ev, vh)
    t.free()
    t2.free()


def test_after_pipelined_msms(gpu, monkeypatch):
    """kzg_open_batch and kzg_fold_open right after pipelined MSMs that were not joined: all results right"""
    import torch
    from msm_families import pack, seeded
    from test_gpu_msm_plans import expected
    curve = BN254
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    n = 1 << 16
    t, ks = make_table(gpu, curve, 1, n, False)
    rng = seeded("kzg-interplay")
    sc = [pack(curve, 12, "uniform", n, rng) for _ in range(2)]
    d_sc = [to_dev(s) for s in sc]
    d_out = [torch.zeros(3 * t.coord_limbs, dtype=torch.int64, device="cuda") for _ in range(2)]
    for k in range(2):
        t.msm_pipelined(d_sc[k], d_out[k], n=n)
    r = random.Random("kzg-interplay")
    rows = rand_rows(curve, 3, n + 1, r)
    check_open(t, curve, ks, rows, n + 1, make_points(curve, 3, r), "open after two pipelined MSMs")
    for k in range(2):
        t.msm_pipelined(d_sc[k], d_out[k], n=n)
    z, gamma = r.randrange(curve.r), r.randrange(curve.r)
    got = jac_to_affine(curve, 1, t.kzg_fold_open(pack_rows(curve, rows, n + 1), pack_fr(curve, [z]),
                                                  pack_fr(curve, [gamma])))
    f = [sum(pow(gamma, b, curve.r) * rows[b][j] for b in range(3)) % curve.r for j in range(n + 1)]
    q, _ = plonk.div_by_linear(curve.r, f, z)
    F, B = pick_base(curve, 1)
    assert got == ec.scalar_mul(F, corelib.fr_dot(curve, np.ascontiguousarray(ks[:n]), pack_fr(curve, q)), B), "fold"
    t.join()
    torch.cuda.synchronize()
    for k in range(2):
        assert jac_to_affine(curve, 1, d_out[k].cpu().numpy().view(np.uint64)) == expected(curve, 1, ks, sc[k]), k
    t.free()
