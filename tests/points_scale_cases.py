"""Inputs and independent answers for the point-scaling tests (test_points_scale_emulation.py on the CPU,
test_gpu_points_scale.py on the device): out[i] = (c * t^i) * P[i] with known discrete logs P[i] = k_i * B, so that the
answer is ((c t^i k_i) mod r) * B."""
import random

from oracle import ec, ff

W = 5           # a 5-bit window width: its digit and window edges are bit-pattern edges for any method


def scalar_edges(curve):
    """scalars at bit-pattern edges: 0, 1, 2^(W-1) and 2^W - 1 and their neighbours, r - 1, r - 2, all ones below the
    top W-bit window (2^(W (nwin - 1)) - 1), and the largest values below r whose top window is all ones"""
    r = curve.r
    bits = curve.r.bit_length()
    nwin = bits // W + 1
    ks = [0, 1, 2, 3, (1 << (W - 1)) - 1, 1 << (W - 1), (1 << (W - 1)) + 1, (1 << W) - 1, 1 << W, r - 1, r - 2,
          (1 << (W * (nwin - 1))) - 1, (1 << (W * (nwin - 1))) + (1 << (W * (nwin - 1) - 1))]
    top_lo = W * (nwin - 1) if W * (nwin - 1) < bits else W * (nwin - 2)
    for j in range(bits - top_lo + 1):
        k = ((1 << (bits - j)) - 1) >> top_lo << top_lo          # top window bits all ones, the rest zero
        if k < r:
            ks.append(k)
            ks.append(k | ((1 << top_lo) - 1))                   # ... and every bit below as well
    return [k for k in dict.fromkeys(ks) if 0 <= k < r]


def dlogs(curve, group, n, seed):
    """discrete logs k_i of the inputs: random, with the point at infinity at index 3 and P, -P side by side at 5, 6"""
    rng = random.Random(f"pscale/{curve.name}/{group}/{n}/{seed}")
    k = [rng.randrange(1, curve.r) for _ in range(n)]
    if n > 3:
        k[3] = 0
    if n > 6:
        k[6] = curve.r - k[5]
    return k


def expected_dlogs(curve, ks, c, t):
    r = curve.r
    out, tp = [], 1
    for k in ks:
        out.append(c * tp % r * k % r)
        tp = tp * t % r
    return out


def oracle_points(curve, group, base, ks):
    """[k * base] packed, by the big-int oracle"""
    F = ff.base_field(curve, group)
    return ec.pack_points(curve, group, [ec.scalar_mul(F, k, base) for k in ks])


def fr(curve, v):
    return ff.pack_elements([v], curve.r, curve.fr_limbs)[0]
