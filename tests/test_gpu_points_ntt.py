"""b200_points_ntt on the device (kzg.ToLagrangeG1 and its inverse on G1 of all four curves): the Ethereum ceremony's
Lagrange basis reproduced byte for byte, known discrete logs from 2^0 to 2^20 points with every input family of
points_ntt_cases.py, the converted table used as a commitment key, and the argument errors."""
import numpy as np
import pytest

from oracle import corelib, ec, ff, kzg_srs
from oracle.params import BLS12_381, BN254, CURVES
from points_ntt_cases import FAMILIES, ceremony, ceremony_case, fr_transform, known_dlog_cases, scalar_mul_points
from util import jac_to_affine, pick_base

pytestmark = pytest.mark.gpu
CURVE_LIST = list(CURVES.values())


def device_fixed_base(curve, base, K):
    """[k_i * base] by b200_fixed_base_batch, pinned against the oracles by the fixed-base tests (the C++ oracle's batch
    costs seconds per call on BW6-761 whatever n is)"""
    from gnark_b200 import lib
    return lib.fixed_base_batch(curve.curve_id, 1, ec.pack_points(curve, 1, [base])[0], np.ascontiguousarray(K))


def to_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64).reshape(-1)).cuda()


def from_dev(t, like):
    return t.cpu().numpy().view(np.uint64).reshape(like.shape)


def check(got, want, what):
    if not np.array_equal(got, want):
        bad = np.nonzero(~np.all(got == want, axis=1))[0]
        pytest.fail(f"{what}: outputs {bad[:8].tolist()} differ ({len(bad)} of {len(want)})")


@pytest.fixture(scope="module")
def srs():
    return ceremony()


@pytest.mark.parametrize("on_device", (False, True), ids=("host", "device"))
def test_ethereum_ceremony_every_size(gpu, srs, on_device):
    """m = 2..4096: the inverse transform of monomial[(4096/m) k] is sum_t lagrange[j + m t], the forward transform
    maps it back; at 4096 the output is the fixture's Lagrange basis, byte for byte"""
    mono, sums = srs
    for s in range(1, 13):
        m = 1 << s
        x, want = ceremony_case(mono, sums, m)
        d = gpu.Domain(gpu.BLS12_381, s)
        for inverse, src, dst in ((True, x, want), (False, want, x)):
            if on_device:
                t = to_dev(src)
                assert d.points_ntt(t, inverse=inverse) is t
                got = from_dev(t, src)
            else:
                got = d.points_ntt(src, inverse=inverse)
            check(got, dst, f"ceremony m={m} inverse={inverse}")
        d.free()
    d = gpu.Domain(gpu.BLS12_381, 12)
    got = d.points_ntt(ec.pack_points(BLS12_381, 1, mono))
    d.free()
    assert got.tobytes() == ec.pack_points(BLS12_381, 1, kzg_srs.load()[1]).tobytes()


def run_cases(gpu, curve, family, logns, on_device=False):
    _, B = pick_base(curve, 1)
    for logn in logns:
        pts, want = known_dlog_cases(curve, B, family, logn, scalar_mul_points if logn <= 4 else device_fixed_base)
        d = gpu.Domain(curve.curve_id, logn)
        for inverse in (True, False):
            if on_device:
                t = to_dev(pts)
                d.points_ntt(t, inverse=inverse)
                got = from_dev(t, pts)
            else:
                got = d.points_ntt(pts, inverse=inverse)
            check(got, want[inverse], f"{curve.name} 2^{logn} {family} inverse={inverse}")
        d.free()


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("curve", CURVE_LIST, ids=[c.name for c in CURVE_LIST])
def test_known_discrete_logs_small(gpu, curve, family):
    """2^0..2^12 points, both directions, host buffers"""
    run_cases(gpu, curve, family, range(13))


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("curve", CURVE_LIST, ids=[c.name for c in CURVE_LIST])
def test_known_discrete_logs_2p16(gpu, curve, family):
    run_cases(gpu, curve, family, [16])


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("curve", [BN254, BLS12_381], ids=["bn254", "bls12-381"])
def test_known_discrete_logs_2p20(gpu, curve, family):
    """2^20 points in a device tensor, transformed in place"""
    run_cases(gpu, curve, family, [20], on_device=True)


def test_converted_table_commits_like_the_monomial_one(gpu):
    """BN254, 2^16: MSM(Lagrange table, NTT(c)) = MSM(monomial table, c) for a random polynomial c - the use of the
    converted SRS as a KZG commitment key (pk.KzgLagrange)"""
    import random
    rng = random.Random(7)
    logn, C = 16, BN254
    _, B = pick_base(C, 1)
    mono = device_fixed_base(C, B, ff.pack_elements([rng.randrange(1, C.r) for _ in range(1 << logn)], C.r, C.fr_limbs))
    c = ff.pack_elements([rng.randrange(C.r) for _ in range(1 << logn)], C.r, C.fr_limbs)
    d = gpu.Domain(gpu.BN254, logn)
    lag = d.points_ntt(mono)
    d.free()

    def commit(table, sc):
        t = gpu.Table(gpu.BN254, 1, table, precomp=False)
        out = jac_to_affine(C, 1, t.msm(sc))
        t.free()
        return out

    want = commit(mono, c)
    assert want == jac_to_affine(C, 1, corelib.msm(C, 1, mono, c))
    assert commit(lag, fr_transform(C, c, logn, False)) == want


def test_argument_errors_leave_the_buffer_untouched(gpu):
    _, B = pick_base(BN254, 1)
    pts = scalar_mul_points(BN254, B, ff.pack_elements(list(range(1, 17)), BN254.r, BN254.fr_limbs))
    keep = pts.copy()
    d = gpu.Domain(gpu.BN254, 4)
    lib = gpu.load()
    with pytest.raises(gpu.B200Error, match="G2"):
        d.points_ntt(pts, group=2)
    t = to_dev(pts)
    with pytest.raises(gpu.B200Error, match="G2"):
        d.points_ntt(t, group=2)
    assert np.array_equal(from_dev(t, pts), keep)
    with pytest.raises(gpu.B200Error, match="null points"):
        gpu.check(lib.b200_points_ntt(d.handle, 1, None, 0, 1))
    with pytest.raises(gpu.B200Error, match="null domain"):
        gpu.check(lib.b200_points_ntt(None, 1, gpu.ptr(pts), 0, 1))
    assert np.array_equal(pts, keep)
    # one-point transform: the input unchanged
    d1 = gpu.Domain(gpu.BN254, 0)
    assert np.array_equal(d1.points_ntt(pts[:1]), keep[:1])
    d1.free()
    d.free()
