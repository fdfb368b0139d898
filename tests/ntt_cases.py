"""Pass plans and input families for the Fr NTT plan tests (test_gpu_ntt_plans.py, test_ntt_plans_emulation.py).

The radix-2 NTT (gnark_b200/csrc/ntt_impl.cuh) runs the log2(n) stages as passes over shared-memory tiles, as planned by
ntt_make_plan (ntt.cuh).  `make_plan` restates that planner in Python, so that a test can say which plans a sweep of
sizes and tile overrides reaches; test_ntt_plans_emulation.py pins it to the C++.  `family` draws the input vectors:
residues uniform over all of [0, r) and the structured vectors where a butterfly's carries and reductions sit at their
edges."""
import numpy as np

from oracle import ff

MAX_TILE_LOG = 11     # NTT_MAX_TILE_LOG
MAX_PASSES = 8        # NTT_MAX_PASSES
DEFAULT_TILE_LOG = 8  # NTT_DEFAULT_TILE_LOG: the tile GB200_NTT_TILE_LOG overrides (6..11)

FAMILIES = ("uniform", "zero", "r_minus_1", "one_hot_first", "one_hot_last", "constant", "zero_r_minus_1")


def passes_needed(logn, tile_log):
    """first pass: tile_log stages, then at most tile_log - 2 per pass"""
    if logn <= tile_log:
        return 1
    smax = tile_log - 2
    return 1 + (logn - tile_log + smax - 1) // smax


def make_plan(logn, tile_log=MAX_TILE_LOG):
    """[(lo_bit, S, cb), ...] in increasing bit order, as ntt_make_plan builds it"""
    tile_log = max(tile_log, 3)
    # a tile that would need more than MAX_PASSES passes is widened to the smallest one that does not
    while tile_log < MAX_TILE_LOG and passes_needed(logn, tile_log) > MAX_PASSES:
        tile_log += 1
    s0 = min(logn, tile_log)
    plan = [(0, s0, 0)]
    bit = s0
    while bit < logn:
        smax = tile_log - 2
        rem = logn - bit
        np_ = (rem + smax - 1) // smax
        s = (rem + np_ - 1) // np_
        plan.append((bit, s, min(tile_log - s, bit)))
        bit += s
    return plan


def cb_clamped(logn, tile_log):
    """passes after the first whose contiguous low bits were cut to lo_bit (the tile is not filled)"""
    return [p for p in make_plan(logn, tile_log)[1:] if p[2] == p[0] and p[0] + p[1] < tile_log]


def _below(a, r_limbs):
    """rows of a (little-endian 64-bit limbs) whose value is below r"""
    lt = np.zeros(a.shape[0], dtype=bool)
    eq = np.ones(a.shape[0], dtype=bool)
    for l in range(a.shape[1] - 1, -1, -1):
        lt |= eq & (a[:, l] < r_limbs[l])
        eq &= a[:, l] == r_limbs[l]
    return lt


def uniform(curve, n, rng):
    """n residues uniform over all of [0, r): random limbs cut to r's bit length, rows >= r drawn again"""
    L = curve.fr_limbs
    top = curve.r.bit_length() - 64 * (L - 1)
    r_limbs = np.array(ff.int_to_limbs(curve.r, L), dtype=np.uint64)
    out = np.empty((n, L), dtype=np.uint64)
    todo = np.arange(n)
    while todo.size:
        x = rng.integers(0, 1 << 64, size=(todo.size, L), dtype=np.uint64, endpoint=False)
        x[:, L - 1] &= np.uint64((1 << top) - 1)
        ok = _below(x, r_limbs)
        out[todo[ok]] = x[ok]
        todo = todo[~ok]
    return out


def family(curve, name, n, rng):
    """(n, fr_limbs) Montgomery residues of one family.  'r_minus_1' is the largest residue a limb vector can hold;
    the one-hot vectors hold the field's one at index 0 / n - 1; 'constant' repeats one uniform residue."""
    L = curve.fr_limbs
    rm1 = np.array(ff.int_to_limbs(curve.r - 1, L), dtype=np.uint64)
    if name == "uniform":
        return uniform(curve, n, rng)
    out = np.zeros((n, L), dtype=np.uint64)
    if name == "zero":
        pass
    elif name == "r_minus_1":
        out[:] = rm1
    elif name in ("one_hot_first", "one_hot_last"):
        out[0 if name == "one_hot_first" else n - 1] = ff.pack_elements([1], curve.r, L)[0]
    elif name == "constant":
        out[:] = uniform(curve, 1, rng)[0]
    elif name == "zero_r_minus_1":
        out[1::2] = rm1
    else:
        raise ValueError(name)
    return out
