#!/usr/bin/env python3
"""Time b200_points_scale (device-resident points, points[i] <- (c t^i) points[i]) on cuda:0 with CUDA events, for G1
and G2 of each curve at 2^16, 2^20 and 2^22 points, after a warm-up call whose result is checked against known
discrete logs: points k_i * B in, (c t^i k_i) * B expected, both from b200_fixed_base_batch.  One JSON line per
(curve, group, log2n) with points per second, the card's name and power limit.

The timed calls scale the warm-up's output again: their scalars are as random as the first ones.

Another build of the library (e.g. from a changed points_scale.cuh) is timed the same way with GB200_LIB=<its path>,
one process per build.

   python tools/sweep_points_scale.py [--cases bn254:1:16,bn254:2:20,...] [--reps 3]"""
import argparse
import json
import os
import random
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

DEFAULT = ",".join(f"{c}:{g}:{s}" for s in (16, 20, 22) for c in ("bn254", "bls12-381", "bls12-377", "bw6-761")
                   for g in (1, 2))


def smi(*fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + ",".join(fields), "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return [x.strip() for x in out.split(",")]


def main():
    import torch
    from gnark_b200 import lib
    from oracle import ec, ff
    from oracle.params import CURVES
    from util import pick_base
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default=DEFAULT)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    lib.load()
    lib.init([0])
    lib.set_stream(0, stream.cuda_stream)
    name, plimit = smi("name", "power.limit")
    rng = random.Random(11)
    for case in args.cases.split(","):
        cname, group, logn = case.split(":")
        curve, group, logn = CURVES[cname], int(group), int(logn)
        n, r = 1 << logn, curve.r
        _, B = pick_base(curve, group)
        base = ec.pack_points(curve, group, [B])[0]
        ks = [rng.randrange(1, r) for _ in range(n)]
        c, t = rng.randrange(2, r), rng.randrange(2, r)
        want_k, tp = [], 1
        for k in ks:
            want_k.append(c * tp % r * k % r)
            tp = tp * t % r
        pack = lambda v: ff.pack_elements(v, r, curve.fr_limbs)
        pts = lib.fixed_base_batch(curve.curve_id, group, base, pack(ks))
        want = lib.fixed_base_batch(curve.curve_id, group, base, pack(want_k))
        cm, tm = pack([c])[0], pack([t])[0]
        x = torch.from_numpy(pts.view(np.int64).reshape(-1)).cuda()
        lib.points_scale(curve.curve_id, group, x, cm, tm)          # warm-up, checked
        ok = bool(np.array_equal(x.cpu().numpy().view(np.uint64).reshape(pts.shape), want))
        if not ok:
            sys.exit(f"{case}: wrong result")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            lib.points_scale(curve.curve_id, group, x, cm, tm)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.reps
        print(json.dumps({"curve": cname, "group": group, "log2n": logn, "ms": round(ms, 3),
                          "points_per_s": round(n / (ms * 1e-3)), "checked": ok, "gpu": name, "power_limit": plimit}),
              flush=True)

if __name__ == "__main__":
    main()
