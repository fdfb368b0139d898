"""The NTT pass planner restated in tests/ntt_cases.py, pinned to ntt_make_plan (ntt.cuh) compiled for the host: every
size 2^0..2^30 at every tile 2^3..2^11, including the tiles widened to keep a plan within NTT_MAX_PASSES passes.  The
GPU plan sweep (test_gpu_ntt_plans.py) relies on the restatement to say which plans it reached."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import ntt_cases as nc


@pytest.fixture(scope="module")
def planemu():
    """tests/emu/ntt_plan_emu.cpp: ntt_make_plan, host build"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call(["make", "-C", os.path.join(root, "gnark_b200", "csrc"), "../../tests/_build/libgb200_nttplanemu.so"])
    lib = ctypes.CDLL(os.path.join(root, "tests", "_build", "libgb200_nttplanemu.so"))
    lib.emu_ntt_plan.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    return lib


def _cpp_plan(planemu, logn, tile_log):
    out = np.full(1 + 3 * nc.MAX_PASSES, -1, dtype=np.int32)
    assert planemu.emu_ntt_plan(logn, tile_log, out.ctypes.data) == 0
    k = int(out[0])
    assert 1 <= k <= nc.MAX_PASSES, (logn, tile_log, k)
    return [tuple(int(v) for v in out[1 + 3 * p:4 + 3 * p]) for p in range(k)]


@pytest.mark.parametrize("tile_log", range(3, 12), ids=lambda t: f"tile{t}")
def test_plan_mirror_matches_cpp(planemu, tile_log):
    for logn in range(31):
        want = _cpp_plan(planemu, logn, tile_log)
        assert nc.make_plan(logn, tile_log) == want, (logn, tile_log)


@pytest.mark.parametrize("tile_log", range(3, 12), ids=lambda t: f"tile{t}")
def test_plan_shape(tile_log):
    """the passes cover the index bits once, in order; every tile fits the widened tile size and the kernel's launch
    bound; cb never exceeds lo_bit; the first pass is contiguous"""
    for logn in range(31):
        plan = nc.make_plan(logn, tile_log)
        eff = tile_log
        while eff < nc.MAX_TILE_LOG and nc.passes_needed(logn, eff) > nc.MAX_PASSES:
            eff += 1
        assert len(plan) == nc.passes_needed(logn, max(eff, 3)) <= nc.MAX_PASSES, (logn, tile_log)
        assert plan[0] == (0, min(logn, max(eff, 3)), 0)
        bit = 0
        for lo, s, cb in plan:
            assert lo == bit and (s >= 1 or logn == 0) and 0 <= cb <= lo
            assert s + cb <= max(eff, 3) <= nc.MAX_TILE_LOG
            bit += s
        assert bit == logn


def test_tile_widening_cases():
    """the widening rule is exercised: 2^3 tiles at 2^11 need nine passes and are widened to 2^4 (five passes)"""
    assert nc.passes_needed(11, 3) == 9
    assert nc.make_plan(11, 3) == [(0, 4, 0), (4, 2, 2), (6, 2, 2), (8, 2, 2), (10, 1, 3)]
    assert nc.make_plan(10, 3)[0] == (0, 3, 0) and len(nc.make_plan(10, 3)) == 8


def test_families():
    """every family is a vector of residues below r with the promised shape"""
    import random
    from oracle.params import CURVES
    for c in CURVES.values():
        g = np.random.default_rng(random.Random(c.name).randrange(1 << 32))
        for f in nc.FAMILIES:
            a = nc.family(c, f, 64, g)
            assert a.shape == (64, c.fr_limbs) and a.dtype == np.uint64
            vals = [int.from_bytes(row.tobytes(), "little") for row in a]
            assert all(v < c.r for v in vals), (c.name, f)
        u = [int.from_bytes(row.tobytes(), "little") for row in nc.uniform(c, 4096, g)]
        # uniform over [0, r): both halves of the range are hit about equally
        upper = sum(v >= c.r // 2 for v in u)
        assert 1800 < upper < 2300, (c.name, upper)
        assert nc.family(c, "one_hot_last", 8, g)[:7].sum() == 0
