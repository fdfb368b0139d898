#!/usr/bin/env python3
"""Time KZG openings of k polynomials of n coefficients on an SRS of n points, per curve:
  open:  (a) one b200_kzg_open_batch call, against
         (b) k x (b200_poly_div_by_linear on a copy of the row + b200_msm of its n - 1 quotient coefficients), which is
             how openings are made without the batch call;
  fold:  (c) one b200_kzg_fold_open call (kzg.BatchOpenSinglePoint's H), against
         (d) the fold b200_plonk_batch_open does (k b200_vec_axpy launches into a zeroed buffer), one
             b200_poly_div_by_linear and one b200_msm.
The polynomials are device-resident in every way.  Defaults: BN254 and BLS12-381, n = 2^12, 2^16, 2^20, k = 1, 4, 16, 64.

Every way ends in a host synchronisation, so each is timed with a host clock around it; the median of --reps runs is
reported.  One warm-up of each way is checked first.  The SRS has a known trapdoor tau (points tau^i B from
b200_fixed_base_batch), so every proof must be ((p_b(tau) - y_b) / (tau - z_b)) B, with p_b(tau) a dot product against the
known discrete logs; (b) and (d) must give the same points and values as (a) and (c).  A case whose workspace estimate
exceeds 80 % of free device memory is skipped (one JSON line saying so).  One JSON line per (curve, n, k) with the card's
name and power limit, read in the same run.

   python tools/sweep_kzg.py [--curves bn254,bls12-381] [--logn 12,16,20] [--ks 1,4,16,64] [--reps 5]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from sweep_msm_batch import batch_bytes, median_ms, random_fr, smi  # noqa: E402


def open_bytes(curve, n, k):
    """device bytes of a batched opening: polynomials, quotients and the scan rows, plus the quotient MSM's workspace"""
    return 3 * k * n * 8 * curve.fr_limbs + batch_bytes(curve, n, k)


def main():
    import torch
    from gnark_b200 import lib
    from oracle import corelib, ec, ff
    from oracle.params import CURVES
    from util import jac_to_affine, pick_base
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", default="bn254,bls12-381")
    ap.add_argument("--logn", default="12,16,20", help="log2 of the coefficient counts (= SRS points)")
    ap.add_argument("--ks", default="1,4,16,64", help="batch sizes")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    lib.load()
    lib.init([0])
    name, plimit = smi("name", "power.limit")
    rs = np.random.RandomState(4844)
    for cname in args.curves.split(","):
        curve = CURVES[cname]
        r, fl = curve.r, curve.fr_limbs
        F, B = pick_base(curve, 1)
        pack = lambda vals: np.ascontiguousarray(ff.pack_elements(vals, r, fl))
        aff = lambda j: lib.point_to_affine(curve.curve_id, 1, np.ascontiguousarray(j, dtype=np.uint64)).tobytes()
        for logn in (int(x) for x in args.logn.split(",")):
            n = 1 << logn
            tau = int(rs.randint(2, 1 << 62)) * 2 ** 60 % r
            taus, acc = [], 1
            for _ in range(n):
                taus.append(acc)
                acc = acc * tau % r
            ks = pack(taus)
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
                if open_bytes(curve, n, k) > 0.8 * free:
                    print(json.dumps({**row, "skipped": f"needs about {open_bytes(curve, n, k) / 2**30:.1f} GiB"}), flush=True)
                    continue
                polys = np.ascontiguousarray(np.stack([random_fr(curve, n, rs) for _ in range(k)]))
                d_polys = torch.from_numpy(polys.view(np.int64)).cuda()
                zs = [int(rs.randint(1, 1 << 62)) * 2 ** 62 % r for _ in range(k)]
                points = pack(zs)
                z, gamma = points[0], pack([int(rs.randint(1, 1 << 62)) * 2 ** 61 % r])
                d_row = torch.empty(n * fl, dtype=torch.int64, device="cuda")
                d_fold = torch.empty(n * fl, dtype=torch.int64, device="cuda")

                def way_a():
                    return table.kzg_open_batch(d_polys, points, on_device=True)

                def way_b():
                    vals, proofs = [], []
                    for b in range(k):
                        d_row.copy_(d_polys[b].reshape(-1))
                        vals.append(lib.poly_div_by_linear(0, curve.curve_id, d_row, n, points[b]))
                        proofs.append(table.msm(d_row, n=n - 1, on_device=True))
                    return vals, proofs

                def way_c():
                    return table.kzg_fold_open(d_polys, z, gamma, on_device=True)

                def way_d():
                    d_fold.zero_()
                    g, gp = ff.unpack_elements(gamma, r, fl)[0], 1
                    for b in range(k):
                        lib.vec_axpy(0, curve.curve_id, d_fold, pack([gp]), d_polys[b], n)
                        gp = gp * g % r
                    lib.poly_div_by_linear(0, curve.curve_id, d_fold, n, z)
                    return table.msm(d_fold, n=n - 1, on_device=True)

                vals, proofs = way_a()                                       # warm-ups, checked
                ys = ff.unpack_elements(vals, r, fl)
                ok = True
                for b in range(k):
                    p_tau = corelib.fr_dot(curve, ks, np.ascontiguousarray(polys[b]))
                    want = (p_tau - ys[b]) * pow(tau - zs[b], -1, r) % r
                    ok = ok and jac_to_affine(curve, 1, proofs[b]) == ec.scalar_mul(F, want, B)
                vb, pb = way_b()
                ok = ok and all(np.array_equal(vb[b], vals[b]) and aff(pb[b]) == aff(proofs[b]) for b in range(k))
                h = way_c()
                g = ff.unpack_elements(gamma, r, fl)[0]
                f_tau = sum(pow(g, b, r) * corelib.fr_dot(curve, ks, np.ascontiguousarray(polys[b])) for b in range(k)) % r
                f_z = sum(pow(g, b, r) * y for b, y in
                          enumerate(ff.unpack_elements(lib.poly_eval_batch(0, curve.curve_id, d_polys, pack([zs[0]] * k),
                                                                           on_device=True), r, fl))) % r
                ok = ok and jac_to_affine(curve, 1, h) == ec.scalar_mul(F, (f_tau - f_z) * pow(tau - zs[0], -1, r) % r, B)
                ok = ok and aff(way_d()) == aff(h)
                t_a, t_b, t_c, t_d = (median_ms(fn, args.reps) for fn in (way_a, way_b, way_c, way_d))
                print(json.dumps({**row, "open_batch_ms": round(t_a, 3), "k_div_msm_ms": round(t_b, 3),
                                  "open_speedup": round(t_b / t_a, 2), "fold_open_ms": round(t_c, 3),
                                  "axpy_div_msm_ms": round(t_d, 3), "fold_speedup": round(t_d / t_c, 2), "checked": ok}),
                      flush=True)
                del d_polys, d_row, d_fold
                torch.cuda.empty_cache()
                if not ok:
                    sys.exit(f"{cname} n={n} k={k}: wrong result")
            table.free()


if __name__ == "__main__":
    main()
