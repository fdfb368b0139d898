"""Per-point logic of k_plonk_constraints (gnark_b200/csrc/plonk.cuh) compiled for the host with the PTX carry chains
emulated, on all four curves and with 0 to 3 blinding coefficients per polynomial (Z unblinded included), against
plonk.numerator of the big-int oracle.  The hardware side of the same kernel is tests/test_gpu_plonk_kernels.py."""
import ctypes
import random

import numpy as np
import pytest

from oracle import ff, ntt, plonk
from oracle.params import CURVES


def P(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize("counts", [(2, 2, 2, 3), (0, 1, 3, 0), (3, 0, 1, 2)], ids=lambda k: "".join(map(str, k)))
@pytest.mark.parametrize("c", list(CURVES.values()), ids=lambda c: c.name)
def test_constraint_kernel_blinding_counts(hostemu, c, counts):
    rng = random.Random(7600 + sum(k << (2 * i) for i, k in enumerate(counts)))
    r, L = c.r, c.fr_limbs
    logn, rho = 4, 4
    n = 1 << logn
    polys = {k: [rng.randrange(r) for _ in range(n)] for k in plonk.POLYS}
    alpha, beta, gamma = (rng.randrange(r) for _ in range(3))
    blind = {k: [rng.randrange(r) for _ in range(m)] for k, m in zip("lroz", counts)}
    want = plonk.numerator(c, n, rho, polys, alpha, beta, gamma, blind)
    dom0, dom1 = ntt.Domain(c, n), ntt.Domain(c, rho * n)
    pe = lambda v: ff.pack_elements(v, r, L)
    abg = pe([alpha, beta, gamma])
    bl = [pe(blind[k] or [0]) for k in "lroz"]          # a valid pointer even where the count is 0
    nbl = (ctypes.c_int * 4)(*counts)
    blp = (ctypes.c_void_p * 4)(*[b.ctypes.data for b in bl])
    out = np.zeros((rho * n, L), dtype=np.uint64)
    for i in range(rho):
        coset = dom1.coset_gen * pow(dom1.generator, i, r) % r
        on_coset = [pe(plonk.coset_values(c, dom0, polys[k], coset)) for k in plonk.POLYS]
        pp = (ctypes.c_void_p * 12)(*[a.ctypes.data for a in on_coset])
        assert hostemu.emu_plonk_constraints_coset(c.curve_id, pp, P(abg), blp, nbl, logn, i, rho, P(out)) == 0
    assert np.array_equal(out, pe(want)), (c.name, counts)
