"""The batched MSM (out[b] = sum_i s_bi * bases[off + i] for every row b) walked on the CPU: msm.cuh's batched
decompose (every item's keys in its own bucket sets), the unchanged sort / accumulate / combine / chunk reduction over
all of the batch's sets, and one Horner per item, compiled for the host with the PTX carry chains emulated
(tests/emu/msm_batch_emu.cpp, emu_msm_batch) - on every curve and group, plain and precomputed tables, against the
known discrete logs of the bases."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from msm_families import pack, seeded
from oracle import corelib, ec, ff
from oracle.params import CURVES
from test_msm_plans_emulation import P, device_table, known_dlog_bases  # noqa: F401

PAIRS = [(c, g) for c in CURVES.values() for g in (1, 2)]
WINDOWS = (4, 7)
BATCHES = (1, 3, 4)
TASK_LEN, CHUNK = 3, 4


@pytest.fixture(scope="module")
def batchemu():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call(["make", "-C", os.path.join(root, "gnark_b200", "csrc"), "../../tests/_build/libgb200_msmbatchemu.so"])
    lib = ctypes.CDLL(os.path.join(root, "tests", "_build", "libgb200_msmbatchemu.so"))
    u32, i = ctypes.c_uint32, ctypes.c_int
    lib.emu_msm_batch.argtypes = [i, i, ctypes.c_void_p, u32, u32, ctypes.c_void_p, u32, u32, i, i, u32, u32,
                                  ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.emu_decompose_single.argtypes = [i, u32, u32, ctypes.c_void_p, u32, i, i, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def rows(curve, c, batch, n, rng):
    """batch scalar rows of n: an all-zero row, two equal rows and a row that is another's negation when the batch
    has room for them, the rest drawn from the 'mixed' family"""
    sc = np.stack([pack(curve, c, "mixed", n, rng) for _ in range(batch)])
    if batch >= 3:
        sc[1] = 0
        sc[2] = sc[0]
    if batch >= 4:
        neg = [(curve.r - s) % curve.r for s in ff.unpack_elements(sc[0], curve.r, curve.fr_limbs)]
        sc[3] = ff.pack_elements(neg, curve.r, curve.fr_limbs)
    return np.ascontiguousarray(sc)


def run(batchemu, curve, group, table, T, off, sc, c, precomp, keys=None, vals=None):
    batch, n = sc.shape[0], sc.shape[1]
    F = ff.base_field(curve, group)
    out = np.zeros((batch, 3 * F.degree * curve.fp_limbs), dtype=np.uint64)
    rc = batchemu.emu_msm_batch(curve.curve_id, group, P(table), T, off, P(sc), n, batch, c, precomp, TASK_LEN, CHUNK,
                                P(out), None if keys is None else P(keys), None if vals is None else P(vals))
    assert rc == 0
    return [ec.from_jac(F, ec.unpack_points(curve, group, o, ncoords=3)[0]) for o in out]


@pytest.mark.parametrize("precomp", (0, 1), ids=("plain", "precomp"))
@pytest.mark.parametrize("curve,group", PAIRS, ids=[f"{c.name}-g{g}" for c, g in PAIRS])
def test_batch_known_dlogs(hostemu, batchemu, curve, group, precomp):
    """every batch size at windows 4 and 7, over the whole table and over a range that starts past 0 and ends at the
    table's end; item b is (sum_i k_(off+i) s_bi) B, the zero row infinity, equal rows equal, a negated row negated"""
    F, B, ks, _ = known_dlog_bases(curve, group)
    T = len(ks)
    KS = ff.pack_elements(ks, curve.r, curve.fr_limbs)
    for c in WINDOWS:
        table = device_table(hostemu, curve, group, c, precomp)
        for batch in BATCHES:
            for off in (0, 5):
                n = T - off
                rng = seeded("batch-emu", curve.name, group, c, precomp, batch, off)
                sc = rows(curve, c, batch, n, rng)
                got = run(batchemu, curve, group, table, T, off, sc, c, precomp)
                what = f"{curve.name} G{group} c={c} precomp={precomp} batch={batch} off={off}"
                for b in range(batch):
                    want = ec.scalar_mul(F, corelib.fr_dot(curve, np.ascontiguousarray(KS[off:]), sc[b]), B)
                    assert got[b] == want, f"{what} item {b}"
                if batch >= 3:
                    assert got[1] is ec.INF and got[2] == got[0], what
                if batch >= 4:
                    assert got[3] == ec.affine_neg(F, got[0]), what


@pytest.mark.parametrize("precomp", (0, 1), ids=("plain", "precomp"))
@pytest.mark.parametrize("curve", list(CURVES.values()), ids=[c.name for c in CURVES.values()])
def test_batch_of_one_is_the_single_decompose(hostemu, batchemu, curve, precomp):
    """batch = 1: the batched decompose writes exactly the keys and values of the single MSM's decompose"""
    _, _, ks, _ = known_dlog_bases(curve, 1)
    T = len(ks)
    for c in WINDOWS:
        off = 2
        n = T - off
        sc = rows(curve, c, 1, n, seeded("batch-one", curve.name, c, precomp))
        nwin = curve.r.bit_length() // c + 1
        kb, vb = np.zeros(n * nwin, dtype=np.uint32), np.zeros(n * nwin, dtype=np.uint32)
        ko, vo = np.full_like(kb, 7), np.full_like(vb, 7)
        table = device_table(hostemu, curve, 1, c, precomp)
        run(batchemu, curve, 1, table, T, off, sc, c, precomp, kb, vb)
        assert batchemu.emu_decompose_single(curve.curve_id, T, off, P(sc), n, c, precomp, P(ko), P(vo)) == 0
        assert np.array_equal(kb, ko) and np.array_equal(vb, vo), f"{curve.name} c={c} precomp={precomp}"
