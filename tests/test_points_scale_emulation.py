"""b200_points_scale (points_scale.cuh) walked on the CPU: the scalar construction, the per-thread signed-window
multiplication and the per-block batched affine conversion compiled for the host with the PTX carry chains emulated
(tests/emu/points_scale_emu.cpp), on G1 and G2 of all four curves, against known discrete logs and the big-int oracle."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import ec, ff
from oracle.params import CURVES
from points_scale_cases import dlogs, expected_dlogs, fr, oracle_points, scalar_edges
from util import pick_base

CASES = [(c, g) for c in CURVES.values() for g in (1, 2)]
IDS = [f"{c.name}-g{g}" for c, g in CASES]


def P(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module")
def psemu():
    """tests/emu/points_scale_emu.cpp: points_scale.cuh's per-thread logic, host build"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call(["make", "-C", os.path.join(root, "gnark_b200", "csrc"), "../../tests/_build/libgb200_pscaleemu.so"])
    lib = ctypes.CDLL(os.path.join(root, "tests", "_build", "libgb200_pscaleemu.so"))
    lib.emu_points_scale.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p,
                                     ctypes.c_void_p]
    lib.emu_points_scale_mul.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    return lib


@pytest.mark.parametrize("curve,group", CASES, ids=IDS)
def test_scalar_edges(psemu, curve, group):
    """k * B for the bit-pattern edges of scalar_edges (0, 1, r - 1, all-ones runs) and k * infinity"""
    F, B = pick_base(curve, group)
    bp = ec.pack_points(curve, group, [B])
    inf = ec.pack_points(curve, group, [None])
    for k in scalar_edges(curve):
        kp = fr(curve, k)
        out = np.zeros_like(bp)
        assert psemu.emu_points_scale_mul(curve.curve_id, group, P(bp), P(kp), P(out)) == 0
        assert ec.unpack_points(curve, group, out)[0] == ec.scalar_mul(F, k, B), (curve.name, group, hex(k))
        assert psemu.emu_points_scale_mul(curve.curve_id, group, P(inf), P(kp), P(out)) == 0
        assert not out.any()


def run(psemu, curve, group, pts, n, c, t):
    out = np.ascontiguousarray(pts[:n], dtype=np.uint64).copy()
    assert psemu.emu_points_scale(curve.curve_id, group, P(out) if n else None, n, P(fr(curve, c)),
                                  None if t is None else P(fr(curve, t))) == 0
    return out


@pytest.mark.parametrize("curve,group", CASES, ids=IDS)
def test_known_discrete_logs(psemu, curve, group):
    """P_i = k_i B (one infinity, one P, -P pair) scaled by c t^i: random (c, t) at n = 0, 1, 17 and 64 (not a multiple of
    the 64-point block at 17, one full block at 64) and (r - 1, random); c = 0 gives infinities, (1, 1) the input,
    t = 0 keeps c P_0 alone, t = None means t = 1"""
    import random
    rng = random.Random(f"pscale-emu/{curve.name}/{group}")
    F, B = pick_base(curve, group)
    n = 64
    ks = dlogs(curve, group, n, 0)
    pts = oracle_points(curve, group, B, ks)
    r = curve.r
    c, t = rng.randrange(2, r), rng.randrange(2, r)
    for m in (0, 1, 17, n):
        got = run(psemu, curve, group, pts, m, c, t)
        assert np.array_equal(got, oracle_points(curve, group, B, expected_dlogs(curve, ks[:m], c, t))), m
    got = run(psemu, curve, group, pts, 9, r - 1, t)
    assert np.array_equal(got, oracle_points(curve, group, B, expected_dlogs(curve, ks[:9], r - 1, t)))
    assert not run(psemu, curve, group, pts, n, 0, t).any()
    assert np.array_equal(run(psemu, curve, group, pts, n, 1, 1), pts)
    assert np.array_equal(run(psemu, curve, group, pts, n, 1, None), pts)
    got = run(psemu, curve, group, pts, n, c, 0)
    assert np.array_equal(got[:1], oracle_points(curve, group, B, [c * ks[0] % r])) and not got[1:].any()
    got = run(psemu, curve, group, pts, 9, c, None)
    assert np.array_equal(got, oracle_points(curve, group, B, [c * k % r for k in ks[:9]]))
