#!/usr/bin/env python3
"""Time b200_points_ntt (device-resident points, inverse transform = kzg.ToLagrangeG1) on cuda:0 with CUDA events,
after a warm-up call whose result is checked against known discrete logs: points d_k * G in, (iNTT(d))_i * G expected
(Fr transform of the C++ oracle, points of b200_fixed_base_batch).  One JSON line per (curve, log2n), with the card's
name, power limit and SM clock beside the numbers.

Multiplier-pipe share (the convention of DESIGN.md §3): Fp products of the transform counted from the code, times the
IMAD.WIDE of one Montgomery product (2N^2 + N for N 32-bit limbs: the 136 of a 254-bit product), over kernel time,
against SMs x 32 IMAD.WIDE lanes/clk x the SM clock read after the timed calls.  Products: a butterfly is two XYZZ
additions (add-2008-s, 14 products each) and, for a twiddle index j != 0, the double-and-add of points_ntt_mul by
w^-j: 9 products per doubling below the scalar's top bit and 14 per further set bit; the 1/n scaling is one more such
multiplication per point.  The batched affine conversion (about 6 products and 1/16 of an inversion per point) is left
out.  The count assumes no intermediate point at infinity, which holds for random inputs.

   python tools/sweep_points_ntt.py [--cases bn254:16,bn254:20,...] [--reps 2]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

DEFAULT = ("bn254:16,bls12-381:16,bls12-377:16,bw6-761:16,bn254:20,bls12-381:20,bls12-377:20,bw6-761:20,"
           "bn254:22,bls12-381:22")


def smi(*fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + ",".join(fields), "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return [x.strip() for x in out.split(",")]


def mul_cost(k):
    """Fp products of points_ntt_mul for the canonical scalar k"""
    return 0 if k == 0 else 9 * (k.bit_length() - 1) + 14 * (k.bit_count() - 1)


def products(curve, logn):
    """Fp products of one inverse transform of 2^logn points (see the module docstring)"""
    from oracle import ntt
    n, r = 1 << logn, curve.r
    dom = ntt.Domain(curve, n)
    cost = np.zeros(max(n // 2, 1), dtype=np.int64)
    t = 1
    for j in range(n // 2):
        cost[j] = mul_cost(t) if j else 0
        t = t * dom.generator_inv % r
    total = 0
    for beta in range(logn):
        stride = 1 << (logn - 1 - beta)
        total += (n >> (beta + 1)) * int(cost[::stride][:1 << beta].sum()) + 28 * (n // 2)
    return total + n * mul_cost(dom.cardinality_inv)


def random_fr(curve, n, rs):
    """n random Fr elements as a Montgomery limb array (every value below r is some element's Montgomery form)"""
    L = curve.fr_limbs
    K = rs.randint(0, 1 << 62, size=(n, L), dtype=np.int64).astype(np.uint64) * np.uint64(4)
    K[:, L - 1] %= np.uint64(curve.r >> (64 * (L - 1)))
    return K


def main():
    import torch
    from gnark_b200 import lib
    from oracle import ec
    from oracle.params import CURVES
    from points_ntt_cases import fr_transform
    from util import pick_base
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default=DEFAULT)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    lib.load()
    lib.init([0])
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    lib.set_stream(0, stream.cuda_stream)
    name, plimit, max_clk = smi("name", "power.limit", "clocks.max.sm")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rs = np.random.RandomState(5)
    for case in args.cases.split(","):
        cname, logn = case.split(":")
        curve, logn = CURVES[cname], int(logn)
        n = 1 << logn
        _, B = pick_base(curve, 1)
        base = ec.pack_points(curve, 1, [B])[0]
        K = random_fr(curve, n, rs)
        pts = lib.fixed_base_batch(curve.curve_id, 1, base, K)
        want = lib.fixed_base_batch(curve.curve_id, 1, base, fr_transform(curve, K, logn, True))
        dom = lib.Domain(curve.curve_id, logn)
        x = torch.from_numpy(pts.view(np.int64).reshape(-1)).cuda()
        dom.points_ntt(x)                                   # warm-up, checked
        ok = bool(np.array_equal(x.cpu().numpy().view(np.uint64).reshape(pts.shape), want))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            dom.points_ntt(x)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.reps
        clk = smi("clocks.sm")[0]
        dom.free()
        N32 = 2 * curve.fp_limbs
        prods = products(curve, logn)
        clk_hz = float(clk.split()[0]) * 1e6
        share = prods * (2 * N32 * N32 + N32) / (ms * 1e-3) / (sms * 32 * clk_hz)
        print(json.dumps({"curve": cname, "log2n": logn, "ms": round(ms, 3), "checked": ok,
                          "fp_products_per_butterfly": round((prods - n * mul_cost(pow(n, -1, curve.r))) / (logn * n / 2), 1),
                          "multiplier_share": round(share, 3), "gpu": name, "power_limit": plimit,
                          "sm_clock_after": clk, "sm_clock_max": max_clk, "sms": sms}), flush=True)
        if not ok:
            sys.exit(f"{case}: wrong result")


if __name__ == "__main__":
    main()
