"""The batched polynomial kernels behind b200_poly_eval_batch, b200_kzg_open_batch and b200_kzg_fold_open, walked on the
CPU: plonk.cuh's per-thread steps and point tables compiled for the host with the PTX carry chains emulated, driven over
the device's grid (tests/emu/kzg_batch_emu.cpp) - one row per polynomial, 2048-coefficient evaluation / division blocks,
and the per-row sum scan over 1024-element blocks with its block totals scanned per row.  Every row is compared with the
big-int oracle (ntt.poly_eval, plonk.div_by_linear) on all four curves, at sizes on both sides of a scan block (1024), an
evaluation / division block (2048) and the scan's second recursion level (2^20, BN254)."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from oracle import ff, ntt, plonk
from oracle.params import CURVES

SIZES = (0, 1, 2, 3, 1023, 1024, 1025, 2047, 2048, 2049)
BATCHES = (1, 3, 7)
POINTS = ("zero", "one", "r-1", "root", "shared", "mixed")
CURVE_LIST = list(CURVES.values())
P = lambda a: a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module")
def kzgemu():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call(["make", "-C", os.path.join(root, "gnark_b200", "csrc"), "../../tests/_build/libgb200_kzgbatchemu.so"])
    lib = ctypes.CDLL(os.path.join(root, "tests", "_build", "libgb200_kzgbatchemu.so"))
    vp, sz, i = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    lib.emu_poly_eval_batch.argtypes = [i, vp, sz, sz, vp, vp]
    lib.emu_poly_div_batch.argtypes = [i, vp, sz, sz, vp, vp, vp]
    lib.emu_poly_fold.argtypes = [i, vp, sz, sz, vp, vp]
    lib.emu_kzg_pow_len.argtypes = [sz]
    lib.emu_kzg_pow_len.restype = ctypes.c_uint32
    return lib


def root_of_unity(curve, logn):
    return pow(curve.root_of_unity, 1 << (curve.two_adicity - logn), curve.r)


def make_points(curve, kind, batch, rng):
    r = curve.r
    w = root_of_unity(curve, 11)
    if kind == "zero":
        return [0] * batch
    if kind == "one":
        return [1] * batch
    if kind == "r-1":
        return [r - 1] * batch
    if kind == "root":
        return [pow(w, b + 1, r) for b in range(batch)]
    if kind == "shared":
        return [rng.randrange(r)] * batch
    cycle = [0, rng.randrange(r), 1, w, r - 1, 0, rng.randrange(r)]       # "mixed": zero and non-zero points side by side
    return [cycle[b % len(cycle)] for b in range(batch)]


def make_rows(curve, batch, n, rng):
    """random rows; with room for them an all-zero row and a row equal to another"""
    rows = [[rng.randrange(curve.r) for _ in range(n)] for _ in range(batch)]
    if batch >= 3:
        rows[1] = [0] * n
        rows[2] = list(rows[0])
    return rows


def pack_rows(curve, rows, n):
    flat = [v for row in rows for v in row]
    return np.ascontiguousarray(ff.pack_elements(flat, curve.r, curve.fr_limbs).reshape(-1)) if flat else \
        np.zeros(1, dtype=np.uint64)


def unpack(curve, arr, count):
    return ff.unpack_elements(arr.reshape(-1)[:count * curve.fr_limbs], curve.r, curve.fr_limbs) if count else []


def run_and_check(kzgemu, curve, rows, n, pts, what):
    batch = len(rows)
    fl = curve.fr_limbs
    polys = pack_rows(curve, rows, n)
    points = ff.pack_elements(pts, curve.r, fl)
    before = polys.copy()
    vals = np.zeros(batch * fl, dtype=np.uint64)
    q = np.zeros(max(1, batch * n) * fl, dtype=np.uint64)
    rems = np.zeros(batch * fl, dtype=np.uint64)
    assert kzgemu.emu_poly_eval_batch(curve.curve_id, P(polys), n, batch, P(points), P(vals)) == 0
    assert kzgemu.emu_poly_div_batch(curve.curve_id, P(polys), n, batch, P(points), P(q), P(rems)) == 0
    assert np.array_equal(polys, before), f"{what}: the input polynomials changed"
    got_v, got_r, got_q = unpack(curve, vals, batch), unpack(curve, rems, batch), unpack(curve, q, batch * n)
    for b in range(batch):
        want = ntt.poly_eval(curve.r, rows[b], pts[b])
        wq, wr = plonk.div_by_linear(curve.r, rows[b], pts[b])
        assert got_v[b] == want, f"{what} item {b}: value"
        assert got_r[b] == wr == want, f"{what} item {b}: remainder"
        assert got_q[b * n:(b + 1) * n] == (wq + [0] if n else []), f"{what} item {b}: quotient"


@pytest.mark.parametrize("kind", POINTS)
@pytest.mark.parametrize("curve", CURVE_LIST, ids=[c.name for c in CURVE_LIST])
def test_eval_and_division(kzgemu, curve, kind):
    """every size and batch: values, remainders and quotients row by row against the oracle"""
    for n in SIZES:
        for batch in BATCHES:
            rng = random.Random(f"kzg-emu-{curve.name}-{kind}-{n}-{batch}")
            run_and_check(kzgemu, curve, make_rows(curve, batch, n, rng), n, make_points(curve, kind, batch, rng),
                          f"{curve.name} n={n} batch={batch} points={kind}")


def test_second_scan_level_bn254(kzgemu):
    """2^20 + 1 coefficients: 1025 scan blocks per row, whose block totals take a second scan level of two blocks"""
    curve = CURVES["bn254"]
    n = (1 << 20) + 1
    rng = random.Random("kzg-emu-2^20")
    rows = make_rows(curve, 2, n, rng)
    run_and_check(kzgemu, curve, rows, n, [rng.randrange(curve.r), 0], "bn254 n=2^20+1")


@pytest.mark.parametrize("curve", CURVE_LIST, ids=[c.name for c in CURVE_LIST])
def test_fold(kzgemu, curve):
    """out[j] = sum_b gamma^b p_b[j] with gamma = 0, 1, r - 1 and a random one"""
    r = curve.r
    for n in (1, 3, 1025):
        for batch in (1, 3, 7):
            rng = random.Random(f"kzg-fold-{curve.name}-{n}-{batch}")
            rows = make_rows(curve, batch, n, rng)
            polys = pack_rows(curve, rows, n)
            for gamma in (0, 1, r - 1, rng.randrange(r)):
                out = np.zeros(n * curve.fr_limbs, dtype=np.uint64)
                g = ff.pack_elements([gamma], r, curve.fr_limbs)
                assert kzgemu.emu_poly_fold(curve.curve_id, P(polys), n, batch, P(g), P(out)) == 0
                want = [sum(pow(gamma, b, r) * rows[b][j] for b in range(batch)) % r for j in range(n)]
                assert unpack(curve, out, n) == want, f"{curve.name} n={n} batch={batch} gamma={gamma}"


def test_pow_table_length(kzgemu):
    """ceil(log2 n) + 1 entries: every power a thread's base below n needs, and the point itself"""
    for n, want in ((1, 1), (2, 2), (3, 3), (4, 3), (1024, 11), (1025, 12), (1 << 20, 21), ((1 << 20) + 1, 22)):
        assert kzgemu.emu_kzg_pow_len(n) == want, n
