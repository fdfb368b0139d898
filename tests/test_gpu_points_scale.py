"""b200_points_scale and b200_points_decode on the device (the point work of a Groth16 MPC contribution, G1 and G2 of
all four curves): known discrete logs from 2^0 to 2^20 points against b200_fixed_base_batch (an independent device
path pinned against the oracles by the fixed-base tests) and the big-int oracle, the phase-1 and phase-2 updates
checked by their trapdoors, the decoder's round trip, and the refusals."""
import random

import numpy as np
import pytest

from oracle import ec, encoding, ff, kzg_srs
from oracle.params import BLS12_381, BN254, CURVES
from points_scale_cases import dlogs, expected_dlogs, fr
from util import pick_base

pytestmark = pytest.mark.gpu
CURVE_LIST = list(CURVES.values())
CASES = [(c, g) for c in CURVE_LIST for g in (1, 2)]
IDS = [f"{c.name}-g{g}" for c, g in CASES]


def to_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64).reshape(-1)).cuda()


def from_dev(t, like):
    return t.cpu().numpy().view(np.uint64).reshape(like.shape)


def check(got, want, what):
    if not np.array_equal(got, want):
        bad = np.nonzero(~np.all(got == want, axis=1))[0]
        pytest.fail(f"{what}: outputs {bad[:8].tolist()} differ ({len(bad)} of {len(want)})")


def fixed_base(curve, group, base, ks):
    """[k * base] by b200_fixed_base_batch"""
    from gnark_b200 import lib
    if len(ks) == 0:
        return ec.pack_points(curve, group, [None])[:0]
    K = ff.pack_elements(ks, curve.r, curve.fr_limbs)
    return lib.fixed_base_batch(curve.curve_id, group, ec.pack_points(curve, group, [base])[0], K)


def scale(gpu, curve, group, pts, c, t, on_device=False):
    """b200_points_scale on a copy of pts (host) or a device tensor of it"""
    tt = None if t is None else fr(curve, t)
    if on_device:
        d = to_dev(pts)
        gpu.points_scale(curve.curve_id, group, d, fr(curve, c), tt)
        return from_dev(d, pts)
    out = pts.copy()
    gpu.points_scale(curve.curve_id, group, out, fr(curve, c), tt)
    return out


def spot_check(curve, group, base, got, want_dlogs, idx):
    F = ff.base_field(curve, group)
    for i in idx:
        assert ec.unpack_points(curve, group, got[i:i + 1])[0] == ec.scalar_mul(F, want_dlogs[i], base), (curve.name, i)


@pytest.mark.parametrize("curve,group", CASES, ids=IDS)
def test_known_discrete_logs(gpu, curve, group):
    """P_i = k_i B (an infinity, a P, -P pair) scaled by c t^i at 1 .. 2^16 + 1 points from host buffers and 2^20 points
    in a device tensor; every point byte for byte against fixed_base(c t^i k_i), a sample against the oracle"""
    _, B = pick_base(curve, group)
    rng = random.Random(f"pscale-gpu/{curve.name}/{group}")
    r = curve.r
    for n, on_dev in ((1, False), (2, False), (63, False), (64, False), (65, False), (1000, False), (4097, False),
                      ((1 << 16) + 1, False), (1 << 20, True)):
        ks = dlogs(curve, group, n, 1)
        pts = fixed_base(curve, group, B, ks)
        c, t = rng.randrange(2, r), rng.randrange(2, r)
        want_k = expected_dlogs(curve, ks, c, t)
        got = scale(gpu, curve, group, pts, c, t, on_dev)
        check(got, fixed_base(curve, group, B, want_k), f"{curve.name} G{group} n={n}")
        spot_check(curve, group, B, got, want_k, sorted({0, n - 1, rng.randrange(n), rng.randrange(n)}))


@pytest.mark.parametrize("curve,group", CASES, ids=IDS)
def test_scalar_edges_past_one_block(gpu, curve, group):
    """n = 200 (three full 64-point blocks and a partial one): c = 0, (1, 1), t = None, c = r - 1, t = 0, t = 1"""
    _, B = pick_base(curve, group)
    r, n = curve.r, 200
    ks = dlogs(curve, group, n, 2)
    pts = fixed_base(curve, group, B, ks)
    c = random.Random(curve.name).randrange(2, r)
    assert not scale(gpu, curve, group, pts, 0, c).any()
    check(scale(gpu, curve, group, pts, 1, 1), pts, "c = 1, t = 1")
    check(scale(gpu, curve, group, pts, 1, None), pts, "c = 1, t = None")
    for cc, t in ((r - 1, c), (r - 1, r - 1), (c, 1), (c, None)):
        check(scale(gpu, curve, group, pts, cc, t), fixed_base(curve, group, B, expected_dlogs(curve, ks, cc, 1 if t is None else t)),
              f"c={cc} t={t}")
    got = scale(gpu, curve, group, pts, c, 0)
    check(got[:1], fixed_base(curve, group, B, [c * ks[0] % r]), "t = 0")
    assert not got[1:].any()


def commons(curve, tau, alpha, beta, N):
    """SrsCommons for (tau, alpha, beta) by fixed-base batches: G1.Tau (2N - 1), G2.Tau (N), AlphaTau, BetaTau, G2.Beta"""
    r = curve.r
    _, g1 = pick_base(curve, 1)
    _, g2 = pick_base(curve, 2)
    pw = [1]
    for _ in range(2 * N - 2):
        pw.append(pw[-1] * tau % r)
    return {"g1_tau": fixed_base(curve, 1, g1, pw), "g2_tau": fixed_base(curve, 2, g2, pw[:N]),
            "alpha_tau": fixed_base(curve, 1, g1, [alpha * p % r for p in pw[:N]]),
            "beta_tau": fixed_base(curve, 1, g1, [beta * p % r for p in pw[:N]]),
            "g2_beta": fixed_base(curve, 2, g2, [beta])}


@pytest.mark.parametrize("curve,N", [(c, 1 << 10) for c in CURVE_LIST] + [(BN254, 1 << 20)],
                         ids=[f"{c.name}-2^10" for c in CURVE_LIST] + ["bn254-2^20"])
def test_phase1_update_by_trapdoor(gpu, curve, N):
    """phase1.go:104-147 applied with four b200_points_scale calls (Tau[1:] of G1 and G2 by (tau', tau'), AlphaTau by
    (alpha', tau'), BetaTau by (beta', tau')) and G2.Beta on the host equals the commons of (tau0 tau', alpha0 alpha',
    beta0 beta')"""
    rng = random.Random(f"phase1/{curve.name}/{N}")
    r = curve.r
    t0, a0, b0, t1, a1, b1 = (rng.randrange(2, r) for _ in range(6))
    s = commons(curve, t0, a0, b0, N)
    for key, group, c in (("g1_tau", 1, t1), ("g2_tau", 2, t1), ("alpha_tau", 1, a1), ("beta_tau", 1, b1)):
        off = 1 if key in ("g1_tau", "g2_tau") else 0
        v = s[key][off:]
        gpu.points_scale(curve.curve_id, group, v, fr(curve, c), fr(curve, t1))
    F2 = ff.base_field(curve, 2)
    s["g2_beta"] = ec.pack_points(curve, 2, [ec.scalar_mul(F2, b1, ec.unpack_points(curve, 2, s["g2_beta"])[0])])
    want = commons(curve, t0 * t1 % r, a0 * a1 % r, b0 * b1 % r, N)
    for key in want:
        check(s[key], want[key], f"{curve.name} N={N} {key}")


@pytest.mark.parametrize("curve", CURVE_LIST, ids=[c.name for c in CURVE_LIST])
def test_phase2_update_by_trapdoor(gpu, curve):
    """phase2.go:110-135: Z and PKK scaled by 1/delta' match their discrete logs times 1/delta', each SigmaCKK[j] by
    sigma_j matches sigma_j times its logs; Z of N - 1 points at N = 2^10, device-resident PKK"""
    rng = random.Random(f"phase2/{curve.name}")
    r = curve.r
    _, g1 = pick_base(curve, 1)
    delta = rng.randrange(2, r)
    dinv = pow(delta, -1, r)
    z = [rng.randrange(r) for _ in range((1 << 10) - 1)]
    pkk = [rng.randrange(r) for _ in range(777)]
    ckk = [[rng.randrange(r) for _ in range(m)] for m in (5, 130)]
    sigma = [rng.randrange(2, r) for _ in ckk]
    Z = fixed_base(curve, 1, g1, z)
    scale_z = Z.copy()
    gpu.points_scale(curve.curve_id, 1, scale_z, fr(curve, dinv))
    check(scale_z, fixed_base(curve, 1, g1, [v * dinv % r for v in z]), "Z")
    PKK = fixed_base(curve, 1, g1, pkk)
    check(scale(gpu, curve, 1, PKK, dinv, None, on_device=True), fixed_base(curve, 1, g1, [v * dinv % r for v in pkk]), "PKK")
    for j, (logs, s) in enumerate(zip(ckk, sigma)):
        C = fixed_base(curve, 1, g1, logs)
        check(scale(gpu, curve, 1, C, s, None), fixed_base(curve, 1, g1, [v * s % r for v in logs]), f"SigmaCKK[{j}]")


def encode_run(curve, group, pts, compressed):
    if group == 1:
        return b"".join(encoding.encode_g1(curve, p, compressed) for p in pts)
    if not compressed and curve.g2_degree == 2:
        return b"".join(encoding.encode_g2_raw(curve, p) for p in pts)
    return b"".join(encoding.encode_g2(curve, p, compressed) for p in pts)


def curve_point(curve, group):
    """a point of the curve itself (y^2 = x^3 + b, or the twist's b' on G2), x the smallest integer that has one: the
    decoder checks its points against b, which pick_base's derived bases need not satisfy"""
    p = curve.p
    for x in range(1, 1000):
        if group == 1 or curve.name == "bw6-761":
            b = encoding._b(curve) if group == 1 else encoding.twist_b(curve)
            y = encoding.sqrt_fp(p, (x ** 3 + b) % p)
        else:
            b0, b1 = encoding.twist_b(curve)
            y = encoding.sqrt_fp2(curve, ((x ** 3 + b0) % p, b1 % p))
            x = (x, 0)
        if y is not None:
            return x, y
    raise AssertionError("no point")


@pytest.mark.parametrize("curve,group", CASES, ids=IDS)
def test_decode_round_trip(gpu, curve, group):
    """compressed and raw encodings by oracle/encoding.py, infinity included, to host and device outputs"""
    B = curve_point(curve, group)
    ks = [0] + [random.Random(f"dec/{curve.name}/{group}").randrange(1, curve.r) for _ in range(70)]
    pts = fixed_base(curve, group, B, ks)
    plist = ec.unpack_points(curve, group, pts)
    for compressed, enc in ((True, gpu.POINTS_COMPRESSED), (False, gpu.POINTS_RAW)):
        blob = encode_run(curve, group, plist, compressed)
        check(gpu.points_decode(curve.curve_id, group, blob, len(plist), enc), pts, f"compressed={compressed}")
        d = to_dev(np.zeros_like(pts))
        gpu.points_decode(curve.curve_id, group, blob, len(plist), enc, out=d)
        check(from_dev(d, pts), pts, f"compressed={compressed} device")


def test_decode_ethereum_ceremony(gpu):
    """the compressed BLS12-381 points of tests/golden/eth_kzg_srs_v1.bin: 2 x 4096 G1 and the G2 points"""
    blob = open(kzg_srs.PATH, "rb").read()
    mono, lag, g2 = kzg_srs.load()
    n1 = 2 * kzg_srs.N
    got = gpu.points_decode(BLS12_381.curve_id, 1, blob[:48 * n1], n1, gpu.POINTS_COMPRESSED)
    check(got, ec.pack_points(BLS12_381, 1, list(mono) + list(lag)), "G1")
    got = gpu.points_decode(BLS12_381.curve_id, 2, blob[48 * n1:48 * n1 + 96 * kzg_srs.N_G2], kzg_srs.N_G2,
                            gpu.POINTS_COMPRESSED)
    check(got, ec.pack_points(BLS12_381, 2, g2), "G2")


def test_decode_names_the_bad_point(gpu):
    C = BN254
    _, B = pick_base(C, 1)
    pts = ec.unpack_points(C, 1, fixed_base(C, 1, B, list(range(1, 11))))
    blob = bytearray(encode_run(C, 1, pts, False))
    blob[7 * 64 + 63] ^= 1                                  # y of point 7 off by one bit: off the curve
    out = np.full((10, 8), 7, dtype=np.uint64)
    with pytest.raises(gpu.B200Error, match="point 7: point not on the curve"):
        gpu.points_decode(C.curve_id, 1, bytes(blob), 10, gpu.POINTS_RAW, out=out)
    assert (out == 7).all()


def test_refusals_leave_the_buffer_untouched(gpu):
    import ctypes
    C = BN254
    _, B = pick_base(C, 1)
    pts = fixed_base(C, 1, B, list(range(1, 70)))
    keep = pts.copy()
    lib = gpu.load()
    one = fr(C, 1)
    P = gpu.ptr
    cases = [
        (lambda: lib.b200_points_scale(0, 4, 1, P(pts), 69, 0, P(one), None), "unknown curve"),
        (lambda: lib.b200_points_scale(0, -1, 1, P(pts), 69, 0, P(one), None), "unknown curve"),
        (lambda: lib.b200_points_scale(0, 0, 3, P(pts), 69, 0, P(one), None), "unknown group"),
        (lambda: lib.b200_points_scale(0, 0, 0, P(pts), 69, 0, P(one), None), "unknown group"),
        (lambda: lib.b200_points_scale(0, 0, 1, P(pts), 69, 0, None, None), "null c"),
        (lambda: lib.b200_points_scale(0, 0, 1, None, 69, 0, P(one), None), "null points"),
        (lambda: lib.b200_points_scale(0, 0, 1, P(pts), 1 << 32, 0, P(one), None), "32-bit point indices"),
    ]
    d = to_dev(pts)
    cases.append((lambda: lib.b200_points_scale(0, 0, 1, P(d), 1 << 32, 1, P(one), None), "32-bit point indices"))
    blob = encode_run(C, 1, ec.unpack_points(C, 1, pts), True)
    raw = np.frombuffer(blob, dtype=np.uint8).copy()
    for bad in ((5, 1, 2, "unknown curve"), (0, 7, 2, "unknown group"), (0, 1, 3, "unknown encoding"),
                (0, 1, 0, "unknown encoding")):
        cases.append((lambda b=bad: lib.b200_points_decode(0, b[0], b[1], P(raw), 69, b[2], P(pts), 0), bad[3]))
    cases += [
        (lambda: lib.b200_points_decode(0, 0, 1, None, 69, 2, P(pts), 0), "null bytes"),
        (lambda: lib.b200_points_decode(0, 0, 1, P(raw), 69, 2, None, 0), "null out"),
        (lambda: lib.b200_points_decode(0, 0, 1, P(raw), 1 << 32, 2, P(pts), 0), "32-bit point indices"),
        (lambda: lib.b200_points_decode(0, 0, 1, P(raw), 1 << 32, 2, P(d), 1), "32-bit point indices"),
    ]
    for call, msg in cases:
        with pytest.raises(gpu.B200Error, match=msg):
            gpu.check(call())
        assert np.array_equal(pts, keep), msg
        assert np.array_equal(from_dev(d, pts), keep), msg
    # n = 0 does nothing, with or without a buffer
    gpu.check(lib.b200_points_scale(0, 0, 1, None, 0, 0, P(one), None))
    gpu.check(lib.b200_points_decode(0, 0, 1, None, 0, 2, None, 0))
    assert ctypes.sizeof(ctypes.c_size_t) == 8
