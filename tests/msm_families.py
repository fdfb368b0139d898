"""Scalar families for the MSM plan tests (test_gpu_msm_plans.py, test_msm_plans_emulation.py).

The bucket MSM (gnark_b200/csrc/msm.cuh) cuts every scalar into signed c-bit digits: a digit of 2^(c-1) or more
becomes negative and carries into the next window, the top window never does, and a window that divides the scalar's
bit length leaves an extra top window that only a carry can reach.  Each family below aims at one of those edges for
a given window c; `candidates` returns canonical values below r, and `pack` draws a Montgomery scalar vector from
them (so vectors of 2^20 and more cost one small pack and a numpy gather)."""
import random

import numpy as np

from oracle import ff

FAMILIES = ("uniform", "zero", "zero_one", "r_minus_1", "window_edges", "carry_every_digit", "max_positive_digit",
            "above_half_digit", "top_window_max")


def num_windows(bits, c):
    """msm_num_windows of msm.cuh"""
    return bits // c + 1


def _every_digit(r, c, d):
    """d in every window: the most full windows that stay below r, and the same pattern cut to bits - 1 bits"""
    bits = r.bit_length()
    nwin = num_windows(bits, c)
    word = lambda k: sum(d << (c * j) for j in range(k))
    out = [word(nwin) & ((1 << (bits - 1)) - 1)]
    for k in range(nwin, 0, -1):
        if word(k) < r:
            out.append(word(k))
            break
    return out


def candidates(r, c, family, rng):
    """canonical values (all < r) of one family at window c; 'uniform' has none (see pack)"""
    bits = r.bit_length()
    nwin = num_windows(bits, c)
    half = 1 << (c - 1)
    if family == "uniform":
        return []
    if family == "zero":
        vals = [0]
    elif family == "zero_one":
        vals = [0, 1]
    elif family == "r_minus_1":
        vals = [r - 1, (r - 1) // 2]
    elif family == "window_edges":            # 2^(ck) - 1: all-ones digits below window k; 2^(ck): a lone digit 1
        vals = [(1 << (c * k)) - 1 for k in range(1, nwin + 1)] + [1 << (c * k) for k in range(nwin)]
    elif family == "carry_every_digit":       # 2^(c-1): negative digit, carry into every next window
        vals = _every_digit(r, c, half)
    elif family == "max_positive_digit":      # 2^(c-1) - 1: largest digit that stays positive, no carry
        vals = _every_digit(r, c, half - 1)
    elif family == "above_half_digit":        # 2^(c-1) + 1: smallest digit that goes negative
        vals = _every_digit(r, c, half + 1)
    elif family == "top_window_max":
        # the highest window with bits of its own (when c divides the bit length the window above it holds only
        # carries) at the largest value r allows, with random, all-ones and all-carry windows below it
        s = c * (nwin - 1) if bits % c else c * (nwin - 2)
        top = (r - 1) >> s
        room = min(1 << s, r - (top << s))
        vals = [(top << s) + rng.randrange(room) for _ in range(4)]
        vals += [(top << s) - 1, (top << s) + sum(half << (c * j) for j in range(s // c)), r - 1]
    else:
        raise ValueError(family)
    vals = sorted({v for v in vals if 0 <= v < r})
    assert vals, (family, c)
    return vals


def uniform(curve, n, rng):
    """n random Montgomery scalars below 2^(bits-1) (their canonical values are spread over all of [0, r))"""
    L = curve.fr_limbs
    g = np.random.default_rng(rng.randrange(1 << 63))
    a = g.integers(0, 1 << 64, size=(n, L), dtype=np.uint64, endpoint=False)
    top = curve.r.bit_length() - 1 - 64 * (L - 1)
    a[:, L - 1] &= np.uint64((1 << top) - 1)
    return a


def pack(curve, c, family, n, rng):
    """(n, fr_limbs) Montgomery scalars of one family; 'mixed' draws every entry from a random family"""
    if family == "uniform":
        return uniform(curve, n, rng)
    g = np.random.default_rng(rng.randrange(1 << 63))
    if family == "mixed":
        vals = sorted({v for f in FAMILIES[1:] for v in candidates(curve.r, c, f, rng)})
        cand = ff.pack_elements(vals, curve.r, curve.fr_limbs)
        out = cand[g.integers(len(vals), size=n)]
        pick = g.random(n) < 0.25
        out[pick] = uniform(curve, int(pick.sum()), rng)
        return np.ascontiguousarray(out)
    vals = candidates(curve.r, c, family, rng)
    cand = ff.pack_elements(vals, curve.r, curve.fr_limbs)
    return np.ascontiguousarray(cand[g.integers(len(vals), size=n)])


def seeded(*key):
    """a Random seeded from the key's text (stable across processes, unlike hash())"""
    return random.Random("/".join(map(str, key)))
