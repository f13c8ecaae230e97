#!/usr/bin/env python
"""Benchmark-function timings: every problem of ``dmosopt_b200.benchmarks`` at n 65 536 rows on the GPU, and the
reference's row-at-a-time functions on the host at a smaller n where dmosopt is importable.

    python scripts/benchmark_sweep.py [--n 65536] [--reps 7] [--ref-n 2048] [--out results/benchmark_sweep.json]

GPU: wall-clock median of --reps calls after one warm-up call, each call returning with its (n, n_obj) result on the
host (dmo_benchmark_eval synchronises).  Two inputs per problem: an ordinary host array (the call uploads it) and the
same rows with a device mirror, as the optimizer plugins hand back their offspring (no upload).  Host: the reference's
``dmosopt.benchmarks.moo_benchmarks`` called once per row, as dmosopt evaluates an objective, timed once over --ref-n
rows; reported as not measured when dmosopt cannot be imported.  Prints the card name and power limit first, then one
JSON line per measurement.
"""

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# (name, n_obj): default n_var per generate_problem_space (30 for ZDT, the reference examples' size)
PROBLEMS = [("zdt1", 2), ("zdt3", 2), ("dtlz1", 3), ("dtlz2", 3), ("dtlz3", 3), ("dtlz4", 3), ("dtlz5", 3), ("dtlz7", 3), ("wfg1", 2),
            ("wfg1", 3), ("wfg4", 3), ("maf1", 5), ("maf2", 5), ("maf4", 5), ("maf1", 10), ("maf2", 10), ("maf4", 10),
            ("maf1", 16), ("maf2", 16), ("maf4", 16)]


def device_line():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return f"device: {torch.cuda.get_device_properties(0).name}; nvidia-smi (name, power limit, max sm clock): {q.stdout.strip() or q.stderr.strip()}"


def median_s(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return float(np.median(ts))


def inputs(name, M, n, seed):
    from dmosopt_b200.benchmarks import generate_problem_space

    d = 30 if name.startswith("zdt") else len(generate_problem_space(name, M))
    X = np.random.default_rng(seed).random((n, d))
    if name.startswith("wfg"):
        X *= 2 * np.arange(1, d + 1)  # the reference's bounds [0, 2i]
    return X


def call(mod, name, X, M):
    fn = getattr(mod, name)
    return fn(X) if name.startswith("zdt") else fn(X, M)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--ref-n", type=int, default=2048)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from dmosopt_b200 import _lib
    from dmosopt_b200 import benchmarks as bm

    _lib.context()
    print(device_line(), flush=True)
    try:
        from dmosopt.benchmarks import moo_benchmarks as ref
    except ImportError:
        ref = None
    rows = []

    def emit(**kw):
        print(json.dumps(kw), flush=True)
        rows.append(kw)

    for i, (name, M) in enumerate(PROBLEMS):
        X = inputs(name, M, a.n, i)
        n, d = X.shape
        s_host = median_s(lambda: call(bm, name, X, M), a.reps)
        Xm, base = _lib.mirrored_readonly(X)
        s_dev = median_s(lambda: call(bm, name, Xm, M), a.reps)
        emit(what="gpu", problem=name, n_obj=M, n_var=d, n=n, host_input_ms=s_host * 1e3, device_input_ms=s_dev * 1e3,
             rows_per_s_device_input=n / s_dev, bytes_moved=n * (d + M) * 8)
        del Xm, base
        if ref is None or name.startswith("zdt"):  # the ZDT objectives live in the reference's example scripts
            emit(what="reference_host_row_at_a_time", problem=name, n_obj=M, n_var=d,
                 s="not measured" + ("" if ref is not None else ": dmosopt is not importable"))
            continue
        Xr = X[: a.ref_n]
        t = time.perf_counter()
        for x in Xr:
            call(ref, name, x, M)
        s = time.perf_counter() - t
        emit(what="reference_host_row_at_a_time", problem=name, n_obj=M, n_var=d, n=Xr.shape[0], s=s, rows_per_s=Xr.shape[0] / s)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
