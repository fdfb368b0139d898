"""The MSM's plan space walked on the CPU: msm.cuh's per-thread logic (signed-digit decomposition, tasks, chunked
bucket reduction, Horner over the windows), compiled for the host with the PTX carry chains emulated, for every window
c from 4 to 16, forced task lengths and reduction chunks, all curves and groups, plain and precomputed tables, and
every scalar family of msm_families.py - against the known discrete logs of the bases."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from msm_families import FAMILIES, pack, seeded
from oracle import corelib, ec, ff
from oracle.params import CURVES
from util import pick_base

PAIRS = [(c, g) for c in CURVES.values() for g in (1, 2)]
TASK_LENS = (1, 2, 5, 64)
PER_FAMILY = 4
N = PER_FAMILY * (len(FAMILIES) + 1)


def _chunks(c, precomp):
    """reduction chunks; a plain table at c >= 13 leaves out the single chunk per set, whose running sum makes every
    one of the nwin * 2^(c-1) buckets a full addition (minutes of emulated arithmetic; the GPU tests run it)"""
    if not precomp and c >= 13:
        return (1, 3, 8)
    return (1, 3, 8, 1 << (c - 1))


def P(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module")
def msmemu():
    """tests/emu/msm_table_emu.cpp: msm.cuh's MSM, host build, on a caller-built table with a stride and an offset"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call(["make", "-C", os.path.join(root, "gnark_b200", "csrc"), "../../tests/_build/libgb200_msmemu.so"])
    lib = ctypes.CDLL(os.path.join(root, "tests", "_build", "libgb200_msmemu.so"))
    lib.emu_msm_table.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32,
                                  ctypes.c_void_p, ctypes.c_uint32, ctypes.c_int, ctypes.c_int, ctypes.c_uint32,
                                  ctypes.c_uint32, ctypes.c_void_p]
    return lib


_BASES = {}


def known_dlog_bases(curve, group):
    """T = N + 3 discrete logs k_i, with a zero (the point at infinity), a repeated base and a base next to its
    negation; slab 0 of the bases (C++ oracle fixed-base) checked against the Python oracle"""
    key = (curve.name, group)
    if key not in _BASES:
        rng = seeded("emu-bases", *key)
        F, B = pick_base(curve, group)
        ks = [rng.randrange(1, curve.r) for _ in range(N + 3)]
        ks[3], ks[5], ks[7] = 0, ks[4], curve.r - ks[6]
        PTS = corelib.fixed_base(curve, group, ec.pack_points(curve, group, [B]), ff.pack_elements(ks, curve.r, curve.fr_limbs))
        assert ec.unpack_points(curve, group, PTS) == [ec.scalar_mul(F, k, B) for k in ks]
        _BASES[key] = (F, B, ks, PTS)
    return _BASES[key]


_TABLES = {}


def device_table(hostemu, curve, group, c, precomp):
    """the table as b200_table_upload lays it out ([w][i], stride T): slab w holds 2^(c*w) * P_i, built point by point
    by the emulated table precompute (emu_precompute, checked against the big-int oracle in test_emulation.py) and
    spot-checked here on a few slab points"""
    F, B, ks, PTS = known_dlog_bases(curve, group)
    if not precomp:
        return PTS
    key = (curve.name, group, c)
    if key not in _TABLES:
        T, nwin = len(ks), curve.r.bit_length() // c + 1
        per = np.zeros((T, nwin, PTS.shape[1]), dtype=np.uint64)
        for i in range(T):
            assert hostemu.emu_precompute(curve.curve_id, group, P(np.ascontiguousarray(PTS[i])), nwin, c, P(per[i])) == 0
        table = np.ascontiguousarray(per.transpose(1, 0, 2)).reshape(nwin * T, -1)
        rng = seeded("emu-table", *key)
        for _ in range(3):
            w, i = rng.randrange(nwin), rng.randrange(T)
            assert ec.unpack_points(curve, group, table[w * T + i])[0] == ec.scalar_mul(F, (ks[i] << (c * w)) % curve.r, B)
        _TABLES[key] = table
    return _TABLES[key]


@pytest.mark.parametrize("precomp", (0, 1), ids=("plain", "precomp"))
@pytest.mark.parametrize("c", range(4, 17), ids=lambda c: f"c{c}")
@pytest.mark.parametrize("curve,group", PAIRS, ids=[f"{c.name}-g{g}" for c, g in PAIRS])
def test_msm_plan_families(hostemu, msmemu, curve, group, c, precomp):
    """one emulated MSM per plan over PER_FAMILY scalars of every family, on the bases [off, off + N) of a table of
    N + 3 (off = 0 or 3: the slab index w * stride + off + i); the (task length, chunk) pair walks all 16 combinations
    over the 26 plans of a curve and group.  A mismatch is narrowed down to the families that fail."""
    F, B, ks, _ = known_dlog_bases(curve, group)
    T = len(ks)
    table = device_table(hostemu, curve, group, c, precomp)
    nwin = curve.r.bit_length() // c + 1
    k = (c - 4) * 2 + precomp
    chunks = _chunks(c, precomp)
    tl, ch = TASK_LENS[k % 4], chunks[(k // 4 + k) % len(chunks)]
    off = 3 * (c % 2)
    plan = f"{curve.name} G{group} c={c} windows={nwin} precomp={precomp} task_len={tl} chunk={ch} off={off}"
    fams = FAMILIES + ("mixed",)
    SC = np.concatenate([pack(curve, c, f, PER_FAMILY, seeded("emu-scalars", curve.name, group, c, f)) for f in fams])
    KS = ff.pack_elements(ks[off:off + N], curve.r, curve.fr_limbs)

    def emu(lo, hi):
        out = np.zeros(3 * F.degree * curve.fp_limbs, dtype=np.uint64)
        assert msmemu.emu_msm_table(curve.curve_id, group, P(table), T, off + lo, P(SC[lo:]), hi - lo, c, precomp,
                                    tl, ch, P(out)) == 0
        got = ec.from_jac(F, ec.unpack_points(curve, group, out, ncoords=3)[0])
        return got == ec.scalar_mul(F, corelib.fr_dot(curve, KS[lo:hi], SC[lo:hi]), B)

    if not emu(0, N):
        bad = [f for j, f in enumerate(fams) if not emu(j * PER_FAMILY, (j + 1) * PER_FAMILY)]
        pytest.fail(f"{plan}: wrong sum; families that fail alone: {bad}")
