#!/usr/bin/env python3
"""Time b200_msm_indexed (k bases picked by index from a plain table of n points) against b200_msm over the dense
n-vector that scatters the same k entries, both from host memory - the second is what a caller without the indexed
entry point pays for a sparse Lagrange-form commitment (the BSB22 hint's kzg.Commit).  Defaults: BLS12-381 with
n = 2^22 and BN254 with n = 2^20, k = 2^4, 2^8, 2^12, 2^16, 2^20 distinct random indices.

Both calls are synchronous (staging, MSM, result download), so each is timed with a host clock around the call; the
median of --reps calls is reported.  Before the timed calls one warm-up call of each is checked: the indexed result
against known discrete logs ((sum_j k_{idx[j]} s_j) B, bases k_i B from b200_fixed_base_batch) and the dense result
against the indexed one.  One JSON line per (curve, n, k) with the card's name and power limit.

   python tools/sweep_msm_indexed.py [--cases bls12-381:22,bn254:20] [--ks 4,8,12,16,20] [--reps 9]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def smi(*fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + ",".join(fields), "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return [x.strip() for x in out.split(",")]


def random_fr(curve, n, rs):
    """n random Fr elements as a Montgomery limb array (every value below r is some element's Montgomery form)"""
    L = curve.fr_limbs
    K = rs.randint(0, 1 << 62, size=(n, L), dtype=np.int64).astype(np.uint64) * np.uint64(4)
    K[:, L - 1] %= np.uint64(curve.r >> (64 * (L - 1)))
    return K


def median_ms(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts))


def main():
    import torch
    from gnark_b200 import lib
    from oracle import corelib, ec
    from oracle.params import CURVES
    from util import jac_to_affine, pick_base
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="bls12-381:22,bn254:20")
    ap.add_argument("--ks", default="4,8,12,16,20", help="log2 of the index counts")
    ap.add_argument("--reps", type=int, default=9)
    args = ap.parse_args()
    lib.load()
    lib.init([0])
    name, plimit = smi("name", "power.limit")
    rs = np.random.RandomState(22)
    for case in args.cases.split(","):
        cname, logn = case.split(":")
        curve, n = CURVES[cname], 1 << int(logn)
        F, B = pick_base(curve, 1)
        ks = random_fr(curve, n, rs)
        d_ks = torch.from_numpy(ks.view(np.int64)).cuda()
        d_pts = torch.zeros((n, 2 * curve.fp_limbs), dtype=torch.int64, device="cuda")
        lib.fixed_base_batch(curve.curve_id, 1, ec.pack_points(curve, 1, [B])[0], d_ks, n=n, out=d_pts)
        del d_ks
        table = lib.Table(curve.curve_id, 1, d_pts, precomp=False, n=n, on_device=True)
        del d_pts
        torch.cuda.empty_cache()
        info = table.info()
        for lk in (int(x) for x in args.ks.split(",")):
            k = 1 << lk
            idx = np.sort(rs.choice(n, size=k, replace=False)).astype(np.uint32)
            rs.shuffle(idx)
            sc = random_fr(curve, k, rs)
            dense = np.zeros((n, curve.fr_limbs), dtype=np.uint64)
            dense[idx] = sc
            got = table.msm_indexed(idx, sc)                              # warm-up, checked
            want = ec.scalar_mul(F, corelib.fr_dot(curve, np.ascontiguousarray(ks[idx]), sc), B)
            ok = jac_to_affine(curve, 1, got) == want
            ok = ok and jac_to_affine(curve, 1, table.msm(dense)) == want
            t_idx = median_ms(lambda: table.msm_indexed(idx, sc), args.reps)
            t_dense = median_ms(lambda: table.msm(dense), args.reps)
            print(json.dumps({"curve": cname, "table_points": n, "table_window": info["window_bits"], "k": k,
                              "indexed_ms": round(t_idx, 3), "dense_msm_ms": round(t_dense, 3),
                              "speedup": round(t_dense / t_idx, 1), "checked": ok, "gpu": name,
                              "power_limit": plimit}), flush=True)
            if not ok:
                sys.exit(f"{case} k={k}: wrong result")
        table.free()


if __name__ == "__main__":
    main()
