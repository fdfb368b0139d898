"""The indexed MSM (sum_j s_j * bases[idx[j]]) walked on the CPU: msm.cuh's decompose with an index list, the index
check that guards it, and the unchanged rest of the pipeline, compiled for the host with the PTX carry chains emulated
(tests/emu/msm_indexed_emu.cpp, emu_msm_table_indexed) - on every curve and group, plain and precomputed tables, against
the known discrete logs of the bases."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from msm_families import pack, seeded
from oracle import corelib, ec, ff
from oracle.params import CURVES
from test_msm_plans_emulation import P, device_table, known_dlog_bases, msmemu  # noqa: F401  (msmemu: fixture)

PAIRS = [(c, g) for c in CURVES.values() for g in (1, 2)]
WINDOWS = (4, 7)


@pytest.fixture(scope="module")
def idxemu():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call(["make", "-C", os.path.join(root, "gnark_b200", "csrc"), "../../tests/_build/libgb200_msmidxemu.so"])
    lib = ctypes.CDLL(os.path.join(root, "tests", "_build", "libgb200_msmidxemu.so"))
    lib.emu_msm_table_indexed.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.c_uint32, ctypes.c_int, ctypes.c_int, ctypes.c_uint32,
                                          ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def index_sets(T, rng):
    """the index lists every indexed test runs: name -> uint32 array"""
    return {
        "random_repeats": np.array([rng.randrange(T) for _ in range(2 * T + 5)], dtype=np.uint32),
        "ends": np.array([T - 1, 0, rng.randrange(T), T - 1, 0], dtype=np.uint32),
        "one_index": np.full(17, rng.randrange(T), dtype=np.uint32),
        "permutation": np.array(rng.sample(range(T), T), dtype=np.uint32),
    }


def run(idxemu, curve, group, table, T, idx, sc, c, precomp, task_len=3, chunk=4):
    F = ff.base_field(curve, group)
    out = np.zeros(3 * F.degree * curve.fp_limbs, dtype=np.uint64)
    bad = np.zeros(1, dtype=np.uint32)
    rc = idxemu.emu_msm_table_indexed(curve.curve_id, group, P(table), T, P(idx), P(sc), idx.size, c, precomp, task_len,
                                      chunk, P(out), P(bad))
    return rc, int(bad[0]), out


@pytest.mark.parametrize("precomp", (0, 1), ids=("plain", "precomp"))
@pytest.mark.parametrize("curve,group", PAIRS, ids=[f"{c.name}-g{g}" for c, g in PAIRS])
def test_indexed_msm_known_dlogs(hostemu, idxemu, curve, group, precomp):
    """every index set at windows 4 and 7; the expected sum is (sum_j k_{idx[j]} s_j) B"""
    F, B, ks, _ = known_dlog_bases(curve, group)
    T = len(ks)
    KS = ff.pack_elements(ks, curve.r, curve.fr_limbs)
    for c in WINDOWS:
        table = device_table(hostemu, curve, group, c, precomp)
        rng = seeded("idx-emu", curve.name, group, c, precomp)
        for name, idx in index_sets(T, rng).items():
            sc = pack(curve, c, "mixed", idx.size, rng)
            rc, _, out = run(idxemu, curve, group, table, T, idx, sc, c, precomp)
            assert rc == 0
            got = ec.from_jac(F, ec.unpack_points(curve, group, out, ncoords=3)[0])
            want = ec.scalar_mul(F, corelib.fr_dot(curve, np.ascontiguousarray(KS[idx]), sc), B)
            assert got == want, f"{curve.name} G{group} c={c} precomp={precomp} index set {name}"


@pytest.mark.parametrize("curve", list(CURVES.values()), ids=[c.name for c in CURVES.values()])
def test_indexed_equals_dense_msm(hostemu, idxemu, msmemu, curve):
    """the indexed MSM equals the MSM over the dense vector that scatters and sums the same entries (emu_msm_table of
    tests/emu/msm_table_emu.cpp: the decompose without an index list), byte for byte in canonical affine form"""
    F, B, ks, PTS = known_dlog_bases(curve, 1)
    T, c = len(ks), 5
    rng = seeded("idx-dense", curve.name)
    idx = index_sets(T, rng)["random_repeats"]
    sc = pack(curve, c, "uniform", idx.size, rng)
    dense = [0] * T
    for i, s in zip(idx, ff.unpack_elements(sc, curve.r, curve.fr_limbs)):
        dense[i] = (dense[i] + s) % curve.r
    D = ff.pack_elements(dense, curve.r, curve.fr_limbs)
    rc, _, got = run(idxemu, curve, 1, PTS, T, idx, sc, c, 0)
    assert rc == 0
    want = np.zeros_like(got)
    assert msmemu.emu_msm_table(curve.curve_id, 1, P(PTS), T, 0, P(D), T, c, 0, 3, 4, P(want)) == 0
    aff = lambda j: ec.pack_points(curve, 1, [ec.from_jac(F, ec.unpack_points(curve, 1, j, ncoords=3)[0])]).tobytes()
    assert aff(got) == aff(want)


@pytest.mark.parametrize("precomp", (0, 1), ids=("plain", "precomp"))
@pytest.mark.parametrize("curve", list(CURVES.values()), ids=[c.name for c in CURVES.values()])
def test_out_of_range_index_is_refused(hostemu, idxemu, curve, precomp):
    """an index equal to the point count (a valid slab entry of a precomputed table, but not a point) and the largest
    uint32 are refused before any point is read, with the lowest bad position; a valid call afterwards is right"""
    F, B, ks, _ = known_dlog_bases(curve, 1)
    T, c = len(ks), 4
    table = device_table(hostemu, curve, 1, c, precomp)
    rng = seeded("idx-bad", curve.name, precomp)
    sc = pack(curve, c, "uniform", 9, rng)
    for bad_pos, bad_val in ((6, T), (0, 0xFFFFFFFF), (8, T + 1)):
        idx = np.array([rng.randrange(T) for _ in range(9)], dtype=np.uint32)
        idx[bad_pos] = bad_val
        if bad_pos < 8:
            idx[8] = T
        rc, bad, out = run(idxemu, curve, 1, table, T, idx, sc, c, precomp)
        assert (rc, bad) == (1, bad_pos)
        assert not out.any(), "the output was written"
    idx = np.array([rng.randrange(T) for _ in range(9)], dtype=np.uint32)
    rc, _, out = run(idxemu, curve, 1, table, T, idx, sc, c, precomp)
    KS = ff.pack_elements(ks, curve.r, curve.fr_limbs)
    assert rc == 0
    assert ec.from_jac(F, ec.unpack_points(curve, 1, out, ncoords=3)[0]) == \
        ec.scalar_mul(F, corelib.fr_dot(curve, np.ascontiguousarray(KS[idx]), sc), B)
