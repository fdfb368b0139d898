#!/usr/bin/env python3
"""Time three ways of computing k MSMs of n scalars over the same n bases of a plain table of n points:
  (a) one b200_msm_batch call, from host scalars and (a') from device-resident scalars,
  (b) k synchronous b200_msm calls (host scalars),
  (c) k b200_msm_pipelined calls from device-resident scalars, then one b200_msm_join and a device synchronise.
Defaults: BN254 G1 and BLS12-381 G1, n = 2^8, 2^12, 2^16, 2^20, k = 1, 4, 16, 64.  Each table has exactly n points, so
b200_msm and the pipelined MSM use the window of an n-point table, as their callers would.

Every way ends in a host synchronisation, so each is timed with a host clock around it; the median of --reps runs is
reported.  Before the timed runs one warm-up of each way is checked: every item of (a) against known discrete logs
((sum_i k_i s_bi) B, bases k_i B from b200_fixed_base_batch), (a'), (b) and (c) against (a) in canonical affine bytes.  A
case whose workspace would not fit in free device memory is skipped (one JSON line saying so).  One JSON line per
(curve, n, k) with the card's name and power limit.

   python tools/sweep_msm_batch.py [--curves bn254,bls12-381] [--logn 8,12,16,20] [--ks 1,4,16,64] [--reps 5]"""
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


def batch_bytes(curve, n, k):
    """device bytes of a batch call: scalars, the four key/value arrays, task partials (task length >= 8) and buckets"""
    c = min(16, max(4, n.bit_length() - 1 - 4))
    nwin = curve.r.bit_length() // c + 1
    m = k * n * nwin
    buckets = k * nwin << (c - 1)
    xyzz = 4 * 8 * curve.fp_limbs
    return k * n * 8 * curve.fr_limbs + 16 * m + (m // 8 + 2 * buckets) * xyzz


def main():
    import torch
    from gnark_b200 import lib
    from oracle import corelib, ec
    from oracle.params import CURVES
    from util import jac_to_affine, pick_base
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", default="bn254,bls12-381")
    ap.add_argument("--logn", default="8,12,16,20", help="log2 of the per-item scalar counts (= table points)")
    ap.add_argument("--ks", default="1,4,16,64", help="batch sizes")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    lib.load()
    lib.init([0])
    name, plimit = smi("name", "power.limit")
    rs = np.random.RandomState(4844)
    for cname in args.curves.split(","):
        curve = CURVES[cname]
        F, B = pick_base(curve, 1)
        for logn in (int(x) for x in args.logn.split(",")):
            n = 1 << logn
            ks = random_fr(curve, n, rs)
            d_ks = torch.from_numpy(ks.view(np.int64)).cuda()
            d_pts = torch.zeros((n, 2 * curve.fp_limbs), dtype=torch.int64, device="cuda")
            lib.fixed_base_batch(curve.curve_id, 1, ec.pack_points(curve, 1, [B])[0], d_ks, n=n, out=d_pts)
            del d_ks
            table = lib.Table(curve.curve_id, 1, d_pts, precomp=False, n=n, on_device=True)
            del d_pts
            torch.cuda.empty_cache()
            for k in (int(x) for x in args.ks.split(",")):
                row = {"curve": cname, "n": n, "k": k, "gpu": name, "power_limit": plimit}
                free, _ = torch.cuda.mem_get_info()
                if batch_bytes(curve, n, k) > 0.8 * free:
                    print(json.dumps({**row, "skipped": f"needs about {batch_bytes(curve, n, k) / 2**30:.1f} GiB"}), flush=True)
                    continue
                sc = np.ascontiguousarray(np.stack([random_fr(curve, n, rs) for _ in range(k)]))
                d_sc = torch.from_numpy(sc.view(np.int64)).cuda()
                d_out = torch.zeros((k, 3 * curve.fp_limbs), dtype=torch.int64, device="cuda")

                def way_a():
                    return table.msm_batch(sc)

                def way_a_dev():
                    return table.msm_batch(d_sc)

                def way_b():
                    return [table.msm(sc[b]) for b in range(k)]

                def way_c():
                    for b in range(k):
                        table.msm_pipelined(d_sc[b], d_out[b], n=n)
                    table.join()
                    torch.cuda.synchronize()

                aff = lambda j: lib.point_to_affine(curve.curve_id, 1, np.ascontiguousarray(j, dtype=np.uint64)).tobytes()
                got_a = way_a()                                               # warm-ups, checked
                ok = all(jac_to_affine(curve, 1, got_a[b]) == ec.scalar_mul(F, corelib.fr_dot(curve, ks, sc[b]), B)
                         for b in range(k))
                got_ad = way_a_dev()
                got_b = way_b()
                way_c()
                got_c = d_out.cpu().numpy().view(np.uint64)
                ok = ok and all(aff(x[b]) == aff(got_a[b]) for x in (got_ad, got_b, got_c) for b in range(k))
                t_a, t_ad, t_b, t_c = (median_ms(f, args.reps) for f in (way_a, way_a_dev, way_b, way_c))
                print(json.dumps({**row, "batch_ms": round(t_a, 3), "batch_dev_ms": round(t_ad, 3), "k_sync_msm_ms": round(t_b, 3),
                                  "k_pipelined_dev_ms": round(t_c, 3), "batch_vs_sync": round(t_b / t_a, 2),
                                  "batch_dev_vs_pipelined": round(t_c / t_ad, 2), "checked": ok}), flush=True)
                del d_sc, d_out
                torch.cuda.empty_cache()
                if not ok:
                    sys.exit(f"{cname} n={n} k={k}: wrong result")
            table.free()


if __name__ == "__main__":
    main()
