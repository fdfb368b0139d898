#!/usr/bin/env python3
"""A/B sweep of the MSM tuning knobs on cuda:0, one JSON line per configuration (result checked against the
known-discrete-log oracle for every configuration before it is timed):

   python tools/sweep_msm.py <curve> <group> <log2 n> [--reps 10] [--set NAME=v1,v2,...]...

   e.g.  python tools/sweep_msm.py bn254 1 20 --set GB200_MSM_WINDOW=16,18,20,22 --set GB200_MSM_HYBRID=0,30,50

Knobs (read by the library at table upload / MSM time): GB200_MSM_WINDOW (window bits c), GB200_MSM_TASK_LEN,
GB200_MSM_CHUNK, GB200_MSM_PRECOMP.  The cartesian product of all --set lists is run.  (Round 2 measured and removed the other round-1 knobs:
hybrid / FP64-pipe accumulate, batched-affine levels, shared-memory accumulators, persistent grid - DESIGN.md §3.)
"""
import argparse
import itertools
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gnark_b200 import lib  # noqa: E402
from oracle import corelib, derive, ec, ff  # noqa: E402  (input generation + result check only)
from oracle.params import CURVES  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("curve")
    ap.add_argument("group", type=int)
    ap.add_argument("logn", type=int)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--set", action="append", default=[], help="NAME=v1,v2,...")
    args = ap.parse_args()
    import torch
    c = CURVES[args.curve]
    n = 1 << args.logn
    rs = np.random.RandomState(1)
    L = c.fr_limbs

    def rand_fr(count):
        a = rs.randint(0, 1 << 62, size=(count, L), dtype=np.int64).astype(np.uint64)
        a[:, L - 1] &= np.uint64((1 << (c.r.bit_length() - 64 * (L - 1) - 2)) - 1)
        return a
    base = derive.subgroup_point(c, args.group)
    F = ff.base_field(c, args.group)
    small = min(n, 1 << 14)
    ks = rand_fr(small)
    pts = np.tile(corelib.fixed_base(c, args.group, ec.pack_points(c, args.group, [base]), ks), (n // small, 1))
    sc = rand_fr(n)
    expected = ec.scalar_mul(F, corelib.fr_dot(c, np.tile(ks, (n // small, 1)), sc), base)
    lib.load(); lib.init([0])
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    lib.set_stream(0, stream.cuda_stream)
    d_sc = torch.from_numpy(sc.view(np.int64)).cuda()
    names = [s.split("=")[0] for s in args.set]
    lists = [s.split("=")[1].split(",") for s in args.set]
    for combo in itertools.product(*lists) if lists else [()]:
        env = dict(zip(names, combo))
        for k, v in env.items():
            os.environ[k] = v
        rec = {"curve": c.name, "group": args.group, "log2n": args.logn, **env}
        try:
            t = lib.Table(c.curve_id, args.group, pts, precomp=True)
            d_out = torch.zeros(3 * t.coord_limbs, dtype=torch.int64, device="cuda")
            t.msm_async(d_sc, d_out, n=n)
            lib.sync(0)
            got = ec.from_jac(F, ec.unpack_points(c, args.group, d_out.cpu().numpy().view(np.uint64), ncoords=3)[0])
            rec["correct"] = bool(got == expected)
            for _ in range(2):
                t.msm_async(d_sc, d_out, n=n)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            lib.sync(0)
            e0.record()
            for _ in range(args.reps):
                t.msm_async(d_sc, d_out, n=n)
            e1.record()
            lib.sync(0)
            rec["ms_standalone"] = e0.elapsed_time(e1) / args.reps
            d_outs = torch.zeros((args.reps, 3 * t.coord_limbs), dtype=torch.int64, device="cuda")
            for i in range(3):                 # warm the pipelined path (second stream, pool growth) before timing it
                t.msm_pipelined(d_sc, d_outs[i % args.reps], n=n)
            t.join()
            lib.sync(0)
            best = 1e9
            for _ in range(3):
                e0.record()
                for i in range(args.reps):
                    t.msm_pipelined(d_sc, d_outs[i], n=n)
                t.join()
                e1.record()
                lib.sync(0)
                best = min(best, e0.elapsed_time(e1) / args.reps)
            rec["ms_pipelined"] = best
            prof = [t.msm_profile(d_sc, d_out, n=n) for _ in range(3)]
            rec["stage_ms"] = {k: round(float(np.median([p[k] for p in prof])), 4) for k in prof[0]}
            rec["table"] = t.info()
            t.free()
        except Exception as e:  # keep sweeping
            rec["error"] = repr(e)
        print(json.dumps(rec), flush=True)
        for k in env:
            os.environ.pop(k, None)


if __name__ == "__main__":
    main()
