#!/usr/bin/env python3
"""Time k Groth16 proofs of one circuit two ways: one b200_groth16_prove_batch call (ProveSolutionBatch) and k sequential
b200_groth16_prove calls (ProveSolution), from host witnesses to the three proof points.
Defaults: BN254 and BLS12-381, log n = 10, 14, 18, 20, k = 1, 4, 16, 64, on a precomputed-table key.

The circuit is oracle/groth16_fast.py's satisfied product network of n - 1 constraints; the key is built from the
instance of seed 1 with b200_fixed_base_batch, and the witnesses are the values of the instances of seeds 1..4 (item j
takes seed 1 + j % 4) on that key, as tests/test_gpu_groth16_batch.py does at 2^20.  Both ways end in a host
synchronisation, so each is timed with a host clock around it; the median of --reps runs is reported.  Before the timed
runs one warm-up of each way is checked: every proof point against oracle/groth16_fast.expected (dlog * generator and
the verifier's equation in the exponent), and the batch's proofs byte for byte against the sequential ones.

The host assembly (delta multiples and proof points, about 6 host scalar multiplications per proof) is timed on its own:
k b200_groth16_assemble calls on one host thread and on os.cpu_count() threads, the shape of the batch's assembly.
A point whose estimated device memory is above 80 % of the free memory is skipped, with one JSON line saying so.  One
JSON line per (curve, log n, k) with the card's name and power limit.

   python tools/sweep_groth16_batch.py [--curves bn254,bls12-381] [--logn 10,14,18,20] [--ks 1,4,16,64] [--reps 5]"""
import argparse
import dataclasses
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def smi(*fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + ",".join(fields), "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return [x.strip() for x in out.split(",")]


def median_ms(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts))


def batch_bytes(curve, n, k):
    """device bytes of a batch beyond the key: W, A, B, C and the filtered wires of k items, and the two largest live MSM
    workspaces (keys and values, task partials at task length >= 8, buckets) of a precomputed n-point table"""
    c = min(16, max(4, n.bit_length() - 1 - 4))
    nwin = curve.r.bit_length() // c + 1
    m = k * n * nwin
    xyzz = 4 * 8 * curve.fp_limbs
    return 6 * k * n * 8 * curve.fr_limbs + 2 * (16 * m + (m // 8 + 2 * (k << (c - 1))) * xyzz)


def main():
    import torch
    from gnark_b200 import groth16 as b200
    from gnark_b200 import lib
    from oracle import ec
    from oracle import groth16_fast as gf
    from oracle.params import CURVES
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", default="bn254,bls12-381")
    ap.add_argument("--logn", default="10,14,18,20")
    ap.add_argument("--ks", default="1,4,16,64")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    lib.load()
    lib.init([0])
    name, plimit = smi("name", "power.limit")
    threads = os.cpu_count() or 1
    for cname in args.curves.split(","):
        c = CURVES[cname]
        for logn in (int(x) for x in args.logn.split(",")):
            inst0 = gf.satisfied_instance(c, logn, seed=1)
            insts = [inst0] + [dataclasses.replace(inst0, v=gf.satisfied_instance(c, logn, seed=s).v) for s in (2, 3, 4)]
            fb = lambda group, dl: lib.fixed_base_batch(c.curve_id, group, ec.pack_points(c, group, [c.g1 if group == 1 else c.g2]),
                                                        np.ascontiguousarray(dl))
            kp = gf.key_points(inst0, fb)
            pk = b200.ProvingKey.from_arrays(c.curve_id, inst0.n, kp["alpha"], kp["beta"], kp["delta"], kp["A"], kp["B"],
                                             kp["Z"], kp["K"], kp["beta2"], kp["delta2"], kp["B2"], inst0.inf_a,
                                             inst0.inf_b, inst0.nb_public)
            del kp
            sols = []
            for inst in insts:
                a, b, cc = inst.solution_abc()
                sols.append(b200.R1CSSolution(W=inst.wires(), A=a, B=b, C=cc))
            pk.setup_device_pointers(b200.NewConfig(b200.WithDeviceID(0)))
            torch.cuda.empty_cache()
            for k in (int(x) for x in args.ks.split(",")):
                row = {"curve": cname, "logn": logn, "k": k, "gpu": name, "power_limit": plimit}
                free, _ = torch.cuda.mem_get_info()
                if batch_bytes(c, inst0.n, k) > 0.8 * free:
                    print(json.dumps({**row, "skipped": f"needs about {batch_bytes(c, inst0.n, k) / 2**30:.1f} GiB of "
                                                        f"{free / 2**30:.1f} GiB free"}), flush=True)
                    continue
                items = [sols[j % 4] for j in range(k)]
                rs = [(0x5EED << 64) + 977 * j for j in range(2 * k)]

                def batch():
                    it = iter(rs)
                    return b200.ProveSolutionBatch(pk, items, b200.WithDeviceID(0), b200.WithRandomness(lambda q: next(it)))

                def sequential():
                    it = iter(rs)
                    return [b200.ProveSolution(pk, sol, b200.WithDeviceID(0), b200.WithRandomness(lambda q: next(it)))
                            for sol in items]

                got_b, got_s = batch(), sequential()                         # warm-ups, checked
                ok = all(np.array_equal(getattr(x, f), getattr(y, f)) for x, y in zip(got_b, got_s) for f in ("Ar", "Bs", "Krs"))
                for j, p in enumerate(got_b):
                    e = gf.expected(insts[j % 4], rs[2 * j], rs[2 * j + 1])
                    ok = ok and gf.verify_points(insts[j % 4], ec.unpack_points(c, 1, p.Ar)[0], ec.unpack_points(c, 2, p.Bs)[0],
                                                 ec.unpack_points(c, 1, p.Krs)[0], e, with_pairing=False)
                t_b, t_s = median_ms(batch, args.reps), median_ms(sequential, args.reps)
                # host assembly alone: k b200_groth16_assemble calls (delta multiples + assembly), 1 thread and all threads
                L = lib.load()
                frl, fpl, deg = lib.CURVE_SHAPES[c.curve_id]
                msm = np.zeros(4 * 3 * fpl + 3 * fpl * deg, dtype=np.uint64)      # five points at infinity
                r_ = b200._fr_to_mont_limbs(rs[0], c.curve_id)
                s_ = b200._fr_to_mont_limbs(rs[1], c.curve_id)
                outs = [(np.zeros(2 * fpl, np.uint64), np.zeros(2 * fpl * deg, np.uint64), np.zeros(2 * fpl, np.uint64))
                        for _ in range(k)]

                def assemble(j):
                    ar, bs, krs = outs[j]
                    lib.check(L.b200_groth16_assemble(pk._handle, lib.ptr(msm),
                                                      lib.ptr(r_), lib.ptr(s_), lib.ptr(ar), lib.ptr(bs), lib.ptr(krs)))

                t_as1 = median_ms(lambda: [assemble(j) for j in range(k)], args.reps)
                with ThreadPoolExecutor(threads) as ex:
                    t_asn = median_ms(lambda: list(ex.map(assemble, range(k))), args.reps)
                print(json.dumps({**row, "batch_ms": round(t_b, 3), "k_prove_ms": round(t_s, 3),
                                  "batch_ms_per_proof": round(t_b / k, 3), "prove_ms_per_proof": round(t_s / k, 3),
                                  "speedup": round(t_s / t_b, 2), "assembly_1_thread_ms": round(t_as1, 3),
                                  f"assembly_{threads}_threads_ms": round(t_asn, 3), "checked": ok}), flush=True)
                if not ok:
                    sys.exit(f"{cname} 2^{logn} k={k}: wrong proof")
            pk.free_gpu_resources()
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
