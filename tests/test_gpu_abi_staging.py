"""Host / device placement of the buffers of the synchronous C ABI entry points.

Every synchronous entry point stages its host inputs into device memory, runs, downloads its host outputs and
synchronises before it returns; device-resident buffers are used in place.  For each placement of each buffer the
result must equal the all-host result byte for byte (MSM results are compared in canonical affine form: a Jacobian
point has many representatives).  The all-host results themselves are checked against the oracles elsewhere
(test_gpu_msm.py, test_gpu_ntt.py, test_gpu_points_ntt.py, test_gpu_round2.py, test_gpu_zz_late.py).  Also: the
zero-size edges, and one argument error per entry point, after which the same device still answers correctly."""
import ctypes
import itertools
import random

import numpy as np
import pytest

from oracle import corelib, ec, ff
from oracle.params import CURVES
from util import jac_to_affine, pick_base

pytestmark = pytest.mark.gpu
TWO = [CURVES["bn254"], CURVES["bls12-381"]]
CURVE_IDS = lambda c: c.name


def _dev(a):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a).view(np.int64).copy()).cuda()
    torch.cuda.synchronize()
    return t


def _host(t):
    return t.cpu().numpy().view(np.uint64)


def _scalars(c, n, seed):
    rng = random.Random(seed)
    return ff.pack_elements([rng.randrange(c.r) for _ in range(n)], c.r, c.fr_limbs).reshape(n, c.fr_limbs)


def _points(gpu, c, group, n, seed):
    """n affine points k_i * B of the group (the C++ oracle's fixed-base batch: independent of the library)"""
    _, base = pick_base(c, group)
    return corelib.fixed_base(c, group, ec.pack_points(c, group, [base]), _scalars(c, n, seed))


def _affine(gpu, c, group, jac):
    return gpu.point_to_affine(c.curve_id, group, np.ascontiguousarray(jac, dtype=np.uint64))


def _is_infinity(c, group, jac):
    return jac_to_affine(c, group, np.ascontiguousarray(jac, dtype=np.uint64)) is ec.INF


# ---- placement matrix -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", TWO, ids=CURVE_IDS)
@pytest.mark.parametrize("group", (1, 2))
def test_msm_and_msm_allreduce_scalar_placement(gpu, c, group):
    n = 1500
    t = gpu.Table(c.curve_id, group, _points(gpu, c, group, n, 1), precomp=False)
    sc = _scalars(c, n, 2)
    jac = t.msm(sc)
    assert not _is_infinity(c, group, jac)
    want = _affine(gpu, c, group, jac)
    assert np.array_equal(_affine(gpu, c, group, t.msm(_dev(sc), n=n, on_device=True)), want)
    assert np.array_equal(_affine(gpu, c, group, t.msm_allreduce(sc)), want)
    assert np.array_equal(_affine(gpu, c, group, t.msm_allreduce(_dev(sc), n=n, on_device=True)), want)
    # a sub-range, both placements
    part = np.ascontiguousarray(sc[200:900])
    want_part = _affine(gpu, c, group, t.msm(part, off=200))
    assert np.array_equal(_affine(gpu, c, group, t.msm(_dev(part), off=200, n=700, on_device=True)), want_part)
    t.free()


@pytest.mark.parametrize("c", TWO, ids=CURVE_IDS)
@pytest.mark.parametrize("group", (1, 2))
def test_fixed_base_batch_placement(gpu, c, group):
    import torch
    n = 777
    _, base = pick_base(c, group)
    BA = ec.pack_points(c, group, [base])
    ks = _scalars(c, n, 3)
    want = gpu.fixed_base_batch(c.curve_id, group, BA, ks)
    for sc_dev, out_dev in itertools.product((False, True), repeat=2):
        sc = _dev(ks) if sc_dev else ks
        out = torch.zeros(want.size, dtype=torch.int64, device="cuda") if out_dev else np.zeros_like(want)
        gpu.fixed_base_batch(c.curve_id, group, BA, sc, n=n, out=out)
        got = _host(out) if out_dev else out
        assert np.array_equal(got.reshape(want.shape), want), (sc_dev, out_dev)


@pytest.mark.parametrize("c", TWO, ids=CURVE_IDS)
def test_ntt_placement(gpu, c):
    logn = 10
    d = gpu.Domain(c.curve_id, logn)
    a = _scalars(c, 1 << logn, 4)
    for inverse, decimation, coset in ((False, gpu.DIF, False), (True, gpu.DIT, True)):
        want = d.ntt(a.copy(), inverse=inverse, decimation=decimation, on_coset=coset)
        assert not np.array_equal(want, a)
        t = _dev(a)
        d.ntt(t, inverse=inverse, decimation=decimation, on_coset=coset, on_device=True)
        assert np.array_equal(_host(t).reshape(want.shape), want)
    d.free()


@pytest.mark.parametrize("c", TWO, ids=CURVE_IDS)
def test_points_ntt_placement(gpu, c):
    logn = 6
    d = gpu.Domain(c.curve_id, logn)
    pts = _points(gpu, c, 1, 1 << logn, 5)
    for inverse in (True, False):
        want = d.points_ntt(pts, inverse=inverse)
        assert not np.array_equal(want, pts)
        t = _dev(pts)
        assert d.points_ntt(t, inverse=inverse) is t
        assert np.array_equal(_host(t).reshape(want.shape), want)
    d.free()


@pytest.mark.parametrize("c", TWO, ids=CURVE_IDS)
def test_compute_h_placement(gpu, c):
    import torch
    logn, length = 10, 700                  # len < n: the inputs are zero-padded to the domain
    d = gpu.Domain(c.curve_id, logn)
    a, b, cc = (_scalars(c, length, s) for s in (6, 7, 8))
    want = d.compute_h(a, b, cc)
    assert want.shape == (1 << logn, c.fr_limbs) and want.any()
    for in_dev, out_dev in itertools.product((False, True), repeat=2):
        ins = [_dev(v) for v in (a, b, cc)] if in_dev else [v.copy() for v in (a, b, cc)]
        out = torch.zeros(want.size, dtype=torch.int64, device="cuda") if out_dev else np.zeros_like(want)
        d.compute_h(*ins, length=length, on_device=in_dev, out=out, out_on_device=out_dev)
        got = _host(out) if out_dev else out
        assert np.array_equal(got.reshape(want.shape), want), (in_dev, out_dev)
        # the transform works on copies: the inputs are unchanged
        for v, x in zip(ins, (a, b, cc)):
            assert np.array_equal((_host(v) if in_dev else v).reshape(x.shape), x)
    d.free()


@pytest.mark.parametrize("c", TWO, ids=CURVE_IDS)
def test_pedersen_commit_placement(gpu, c):
    n = 300
    key = gpu.PedersenKey(c.curve_id, _points(gpu, c, 1, n, 9), _points(gpu, c, 1, n, 10))
    v = _scalars(c, n, 11)
    cm, pok = key.commit(v)
    assert cm.any() and pok.any() and not np.array_equal(cm, pok)
    for on_dev in (False, True):
        vals = _dev(v) if on_dev else v
        got_cm, got_pok = key.commit(vals)
        assert np.array_equal(got_cm, cm) and np.array_equal(got_pok, pok), on_dev
        only_cm, none = key.commit(vals, want_pok=False)
        assert none is None and np.array_equal(only_cm, cm), on_dev
        none, only_pok = key.commit(vals, want_commitment=False)
        assert none is None and np.array_equal(only_pok, pok), on_dev
    key.free()


@pytest.mark.parametrize("c", TWO, ids=CURVE_IDS)
@pytest.mark.parametrize("group", (1, 2))
def test_msm_gather_placement(gpu, c, group):
    import torch
    n_wires, n = 2500, 1800
    rng = random.Random(12)
    idx = np.array(sorted(rng.sample(range(n_wires), n)), dtype=np.uint32)
    wires = _scalars(c, n_wires, 13)
    t = gpu.Table(c.curve_id, group, _points(gpu, c, group, n, 14), precomp=False)
    jac = t.msm_gather(idx, wires)
    assert not _is_infinity(c, group, jac)
    want = _affine(gpu, c, group, jac)
    assert np.array_equal(want, _affine(gpu, c, group, t.msm(np.ascontiguousarray(wires[idx]))))
    for idx_dev, sc_dev in itertools.product((False, True), repeat=2):
        ix = torch.from_numpy(idx.astype(np.int32)).cuda() if idx_dev else idx
        got = t.msm_gather(ix, _dev(wires) if sc_dev else wires)
        assert np.array_equal(_affine(gpu, c, group, got), want), (idx_dev, sc_dev)
    t.free()


def test_msm_submit_vs_submit_dev(gpu):
    """b200_msm_submit (result downloaded on the tail stream) and b200_msm_submit_dev + b200_d2h agree over a run of
    submissions of different ranges, empty ones included, ended by b200_sync"""
    import torch
    c = CURVES["bn254"]
    n = 3000
    t = gpu.Table(c.curve_id, 1, _points(gpu, c, 1, n, 15), precomp=True)
    sc = _scalars(c, n, 16)
    h_sc = torch.from_numpy(sc.view(np.int64).copy()).pin_memory()
    runs = [(0, n), (100, 2000), (0, 0), (n - 1, 1), (0, n)]
    h_out = torch.zeros((len(runs), 12), dtype=torch.int64).pin_memory()
    d_out = torch.zeros((len(runs), 12), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    for i, (off, m) in enumerate(runs):
        t.msm_submit(h_sc.view(n, 4)[off:], h_out[i], off=off, n=m)
        t.msm_submit_dev(h_sc.view(n, 4)[off:], d_out[i], off=off, n=m)
    gpu.sync(0)
    from_dev = np.zeros((len(runs), 12), dtype=np.uint64)
    gpu.check(gpu.load().b200_d2h(0, gpu.ptr(from_dev), gpu.ptr(d_out), from_dev.nbytes))
    for i, (off, m) in enumerate(runs):
        jac = t.msm(np.ascontiguousarray(sc[off:off + m]), off=off, n=m)
        assert _is_infinity(c, 1, jac) == (m == 0)
        want = _affine(gpu, c, 1, jac)
        assert np.array_equal(_affine(gpu, c, 1, h_out[i].numpy().view(np.uint64)), want), (off, m)
        assert np.array_equal(_affine(gpu, c, 1, from_dev[i]), want), (off, m)
    assert _is_infinity(c, 1, h_out[2].numpy().view(np.uint64))
    t.free()


# ---- zero-size edges ----------------------------------------------------------------------------------------------
def test_zero_size_edges(gpu):
    c = CURVES["bn254"]
    L = gpu.load()
    null = ctypes.c_void_p(0)
    t = gpu.Table(c.curve_id, 1, _points(gpu, c, 1, 64, 17), precomp=False)
    out = np.full(12, 7, dtype=np.uint64)
    # msm, n = 0: null scalars are accepted, the result is the point at infinity
    gpu.check(L.b200_msm(t.handle, 0, 0, null, 0, gpu.ptr(out)))
    assert _is_infinity(c, 1, out)
    out[:] = 7
    gpu.check(L.b200_msm(t.handle, 0, 0, null, 1, gpu.ptr(out)))
    assert _is_infinity(c, 1, out)
    # msm_gather, n_idx = 0
    out[:] = 7
    gpu.check(L.b200_msm_gather(t.handle, 0, null, 0, 0, null, 0, 0, gpu.ptr(out)))
    assert _is_infinity(c, 1, out)
    # fixed_base_batch, n = 0: succeeds and writes nothing
    _, base = pick_base(c, 1)
    gpu.check(L.b200_fixed_base_batch(0, c.curve_id, 1, gpu.ptr(ec.pack_points(c, 1, [base])), null, 0, 0, null, 0))
    # compute_h, len = 0: all three inputs are the zero polynomial, and so is h
    d = gpu.Domain(c.curve_id, 6)
    zero = np.zeros((64, c.fr_limbs), dtype=np.uint64)
    want = d.compute_h(zero, zero, zero)
    assert not want.any()
    h = np.full_like(want, 5)
    gpu.check(L.b200_groth16_compute_h(d.handle, null, null, null, 0, 0, gpu.ptr(h), 0))
    assert np.array_equal(h, want)
    d.free()
    # a Pedersen key of 0 points: commitment and proof of knowledge are the point at infinity (0, 0)
    empty = np.zeros((0, 2 * c.fp_limbs), dtype=np.uint64)
    key = gpu.PedersenKey(c.curve_id, empty, empty)
    cm, pok = np.full(8, 3, dtype=np.uint64), np.full(8, 3, dtype=np.uint64)
    gpu.check(L.b200_pedersen_commit(key.handle, null, 0, 0, gpu.ptr(cm), gpu.ptr(pok)))
    assert not cm.any() and not pok.any()
    key.free()
    t.free()


# ---- argument errors ----------------------------------------------------------------------------------------------
def test_argument_errors_then_a_valid_call(gpu):
    """one bad call per entry point (its message, unchanged), then a valid call on the same device"""
    import torch
    from oracle import encoding
    c = CURVES["bn254"]
    L = gpu.load()
    null = ctypes.c_void_p(0)
    n = 64
    pts = _points(gpu, c, 1, n, 18)
    sc = _scalars(c, n, 19)
    t = gpu.Table(c.curve_id, 1, pts, precomp=False)
    jac = t.msm(sc)
    assert not _is_infinity(c, 1, jac)
    want = _affine(gpu, c, 1, jac)
    out = np.zeros(12, dtype=np.uint64)

    def fails(match, rc):
        assert rc != 0
        assert match in L.b200_last_error().decode(), L.b200_last_error()

    fails("msm: null scalars", L.b200_msm(t.handle, 0, n, null, 0, gpu.ptr(out)))
    assert np.array_equal(_affine(gpu, c, 1, t.msm(sc)), want)
    fails("msm_allreduce: null argument", L.b200_msm_allreduce(t.handle, 0, n, gpu.ptr(sc), 0, null))
    assert np.array_equal(_affine(gpu, c, 1, t.msm_allreduce(sc)), want)

    _, base = pick_base(c, 1)
    BA = ec.pack_points(c, 1, [base])
    fails("fixed_base_batch: null argument", L.b200_fixed_base_batch(0, c.curve_id, 1, gpu.ptr(BA), null, 0, n, gpu.ptr(pts), 0))
    assert np.array_equal(gpu.fixed_base_batch(c.curve_id, 1, BA, _scalars(c, n, 18)), pts)

    d = gpu.Domain(c.curve_id, 6)
    a = _scalars(c, 64, 20)
    want_ntt = d.ntt(a.copy())
    fails("ntt: decimation must be DIF or DIT", L.b200_ntt(d.handle, gpu.ptr(a), 0, 0, 7, 0))
    assert np.array_equal(d.ntt(a.copy()), want_ntt)
    want_pntt = d.points_ntt(pts)
    fails("points_ntt: null points", L.b200_points_ntt(d.handle, 1, null, 0, 1))
    assert np.array_equal(d.points_ntt(pts), want_pntt)
    want_h = d.compute_h(a, a, a)
    h = np.zeros_like(want_h)
    fails("compute_h: len exceeds the domain",
          L.b200_groth16_compute_h(d.handle, gpu.ptr(h), gpu.ptr(h), gpu.ptr(h), 65, 0, gpu.ptr(h), 0))
    assert np.array_equal(d.compute_h(a, a, a), want_h)
    d.free()

    key = gpu.PedersenKey(c.curve_id, pts[:4], pts[4:8])
    cm, pok = key.commit(sc[:4])
    fails("pedersen_commit: 5 values for a basis of 4 points", L.b200_pedersen_commit(key.handle, gpu.ptr(sc), 5, 0,
                                                                                      gpu.ptr(out), null))
    got_cm, got_pok = key.commit(sc[:4])
    assert np.array_equal(got_cm, cm) and np.array_equal(got_pok, pok)
    key.free()

    idx = np.arange(n, dtype=np.uint32)
    idx[2] = 1000
    fails("msm_gather: index 1000 out of range at position 2", L.b200_msm_gather(t.handle, 0, gpu.ptr(idx), n, 0, gpu.ptr(sc),
                                                                                 n, 0, gpu.ptr(out)))
    assert np.array_equal(_affine(gpu, c, 1, t.msm_gather(np.arange(n, dtype=np.uint32), sc)), want)

    h_sc = torch.from_numpy(sc.view(np.int64).copy()).pin_memory()
    h_out = torch.zeros(12, dtype=torch.int64).pin_memory()
    d_out = torch.zeros(12, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    fails("msm_submit: null argument", L.b200_msm_submit(t.handle, 0, n, gpu.ptr(h_sc), null))
    fails("msm_submit_dev: null argument", L.b200_msm_submit_dev(t.handle, 0, n, null, gpu.ptr(d_out)))
    t.msm_submit(h_sc, h_out, n=n)
    t.msm_submit_dev(h_sc, d_out, n=n)
    gpu.sync(0)
    assert np.array_equal(_affine(gpu, c, 1, h_out.numpy().view(np.uint64)), want)
    assert np.array_equal(_affine(gpu, c, 1, _host(d_out)), want)

    P = ec.unpack_points(c, 1, pts)
    blob = b"".join(encoding.encode_g1(c, p, True) for p in P)
    h_tab = ctypes.c_void_p(0)
    buf = np.frombuffer(blob, dtype=np.uint8).copy()
    fails("table_upload_encoded: unknown encoding (1 = raw, 2 = compressed)",
          L.b200_table_upload_encoded(0, c.curve_id, 1, gpu.ptr(buf), n, 3, 0, ctypes.byref(h_tab)))
    t2 = gpu.Table.from_encoded(c.curve_id, 1, blob, n, gpu.POINTS_COMPRESSED, precomp=False)
    assert np.array_equal(_affine(gpu, c, 1, t2.msm(sc)), want)
    t2.free()
    t.free()
