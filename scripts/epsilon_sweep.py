#!/usr/bin/env python
"""Epsilon-nondominated archive timings: dmo_epsilon_sort (device events) and the whole epsilon_get_best call, over
sizes, objective counts, epsilons (default 1e-9, coarse 0.05, "auto") and data (uniform random, near a front).

    python scripts/epsilon_sweep.py [--host] [--reps 3] [--quick]

--host also times the reference's epsilon_get_best on the host (needs the reference package: oracle/_ref or
$DMOSOPT_REF) where n <= 5 000, and prints the quadratic extrapolation of that time to every larger n, labelled as
such.  Medians of --reps runs after one warm-up.  Prints one JSON line per measurement, the card first.
"""

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def data(kind, n, M, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.random((n, M))
    x = np.abs(rng.standard_normal((n, M))) + 1e-3
    return x / np.linalg.norm(x, axis=1, keepdims=True) + 0.01 * rng.random((n, M))


def median_time(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--host", action="store_true")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--quick", action="store_true", help="the smallest size of each objective count only")
    a = ap.parse_args()

    from dmosopt_b200 import _lib
    from dmosopt_b200.MOASMO import epsilon_get_best

    _lib.context()
    print(json.dumps({"card": card()}), flush=True)
    ref = None
    if a.host:
        from oracle import reference_build

        path = reference_build.reference_path()
        if path is not None:
            sys.path.insert(0, path)
            from dmosopt import MOASMO as ref
    host = {}
    grid = [(M, n) for M in (2, 3) for n in (10**4, 10**5, 10**6)] + [(M, n) for M in (5, 10, 16) for n in (10**4, 10**5)]
    if a.quick:
        grid = [(M, n) for M, n in grid if n == 10**4]
    for M, n in grid:
        for kind in ("random", "front"):
            Y = data(kind, n, M, seed=M * 7 + n % 97)
            X = np.zeros((n, 1))
            for eps in (None, 0.05, "auto"):
                _, _, _, _, e = epsilon_get_best(X, Y, None, None, epsilons=eps, delete_duplicates=False)
                e = np.asarray(e, dtype=np.float64)

                def device_call():
                    _lib.timer_begin()
                    keep = _lib.epsilon_sort(Y, e)
                    return _lib.timer_end(), keep

                device_call()
                runs = [device_call() for _ in range(a.reps)]
                kept = len(runs[0][1])
                t_dev = float(np.median([r[0] for r in runs]))
                t_best = median_time(lambda: epsilon_get_best(X, Y, None, None, epsilons=eps), a.reps)
                rec = {"M": M, "n": n, "data": kind, "eps": "default" if eps is None else eps, "kept": kept,
                       "epsilon_sort_ms": round(t_dev, 3), "epsilon_get_best_ms": round(1e3 * t_best, 3)}
                if ref is not None:  # one host run per (M, data, eps) on the first 2 000 rows
                    k = (M, kind, str(eps))
                    if k not in host:
                        t0 = time.perf_counter()
                        ref.epsilon_get_best(X[:2000], Y[:2000], None, None, epsilons=eps)
                        host[k] = time.perf_counter() - t0
                    rec["reference_host_ms_at_2000"] = round(1e3 * host[k], 1)
                    rec["reference_host_ms_quadratic_extrapolation"] = round(1e3 * host[k] * (n / 2000) ** 2, 1)
                print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
