"""The group-element NTT (points_ntt.cuh: kzg.ToLagrangeG1 and its inverse) walked on the CPU: the device templates
compiled for the host with the PTX carry chains emulated (tests/emu/points_ntt_emu.cpp), on G1 of all four curves, in
both directions, against known discrete logs (points_ntt_cases.py) and against the Ethereum ceremony's own Lagrange
basis."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import ec, ff, ntt
from oracle.params import BLS12_381, CURVES
from points_ntt_cases import FAMILIES, ceremony, ceremony_case, known_dlog_cases, scalar_mul_points
from util import pick_base

CURVE_LIST = list(CURVES.values())


def P(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module")
def pnttemu():
    """tests/emu/points_ntt_emu.cpp: points_ntt.cuh's per-thread logic, host build"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call(["make", "-C", os.path.join(root, "gnark_b200", "csrc"), "../../tests/_build/libgb200_pnttemu.so"])
    lib = ctypes.CDLL(os.path.join(root, "tests", "_build", "libgb200_pnttemu.so"))
    lib.emu_points_ntt.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    lib.emu_points_ntt_mul.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def emu(lib, curve, pts, logn, inverse):
    out = np.ascontiguousarray(pts, dtype=np.uint64).copy()
    assert lib.emu_points_ntt(curve.curve_id, P(out), logn, 1 if inverse else 0) == 0
    return out


@pytest.mark.parametrize("curve", CURVE_LIST, ids=[c.name for c in CURVE_LIST])
def test_twiddle_scalar_mul(pnttemu, curve):
    """the butterfly's variable-base multiplication alone against the big-int oracle: 0, 1, r - 1, roots of unity
    (twiddles and their inverses), random scalars, and the point at infinity"""
    F, B = pick_base(curve, 1)
    rng = np.random.RandomState(curve.curve_id)
    w = ntt.Domain(curve, 1 << 6).generator
    ks = [0, 1, 2, curve.r - 1, curve.r - 2, w, pow(w, -1, curve.r), curve.root_of_unity, pow(2, -6, curve.r)]
    ks += [int.from_bytes(rng.bytes(64), "little") % curve.r for _ in range(6)]
    bases = [B, ec.scalar_mul(F, 12345, B), None]
    for base in bases:
        bp = ec.pack_points(curve, 1, [base])
        for k in ks:
            out = np.zeros_like(bp)
            assert pnttemu.emu_points_ntt_mul(curve.curve_id, P(bp), P(ff.pack_elements([k], curve.r, curve.fr_limbs)),
                                              P(out)) == 0
            assert ec.unpack_points(curve, 1, out)[0] == ec.scalar_mul(F, k, base), (curve.name, k, base is None)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("curve", CURVE_LIST, ids=[c.name for c in CURVE_LIST])
def test_known_discrete_logs(pnttemu, curve, family):
    """P_k = d_k B in, (iNTT(d))_i B (forward: NTT(d)_k B) out, bit for bit as canonical affine points, 2^0..2^6,
    both directions"""
    _, B = pick_base(curve, 1)
    for logn in range(7):
        pts, want = known_dlog_cases(curve, B, family, logn, scalar_mul_points)
        for inverse in (True, False):
            got = emu(pnttemu, curve, pts, logn, inverse)
            if not np.array_equal(got, want[inverse]):
                bad = [i for i in range(1 << logn) if not np.array_equal(got[i], want[inverse][i])]
                pytest.fail(f"{curve.name} 2^{logn} {family} inverse={inverse}: outputs {bad[:8]} differ "
                            f"({len(bad)} of {1 << logn})")


@pytest.fixture(scope="module")
def srs():
    return ceremony()


@pytest.mark.parametrize("m", [1 << s for s in range(1, 9)])
def test_ethereum_ceremony(pnttemu, srs, m):
    """m-point inverse transform of monomial[(4096/m) k] = the sums of the fixture's Lagrange points; the forward
    transform maps them back"""
    mono, sums = srs
    logm = m.bit_length() - 1
    x, want = ceremony_case(mono, sums, m)
    lag = emu(pnttemu, BLS12_381, x, logm, True)
    assert np.array_equal(lag, want)
    assert np.array_equal(emu(pnttemu, BLS12_381, want, logm, False), x)
