#!/usr/bin/env python
"""One MOASMO.optimize surrogate epoch, resident against the per-generation plugin loop, at bench.py's shape.

    python scripts/epoch_sweep.py [--pop 65536] [--d 30] [--M 3] [--train 4096] [--gens 50] [--rounds 3]

NSGA2 (distance_metric=None, as MOASMO.epoch builds it) with a GPR_Matern surrogate (precision "auto", the
hyper-parameters kept at their initial values) fitted on DTLZ2 data; the training set is the epoch's ``initial`` rows, as
MOASMO.epoch passes it.  The two routes alternate in one process, --rounds times each after one warm-up epoch of each,
from identically seeded generators; every epoch's results must be identical between the routes (the script fails
otherwise).  Per route it prints the median over the rounds of: ms per generation (wall clock from the first
generation's start to the epoch's return, over the generations), candidates per second, host waits and H2D / D2H bytes
per generation (the library's own counters over the whole epoch, divided by the generations).  The card's name and power
limit come first.
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
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip().splitlines()
    except OSError:
        out = []
    return out[0] if out else "unknown"


def dtlz2(X, M):
    g = ((X[:, M - 1 :] - 0.5) ** 2).sum(axis=1)
    Y = np.ones((X.shape[0], M)) * (1.0 + g)[:, None]
    for i in range(M):
        for j in range(M - 1 - i):
            Y[:, i] *= np.cos(0.5 * np.pi * X[:, j])
        if i > 0:
            Y[:, i] *= np.sin(0.5 * np.pi * X[:, M - 1 - i])
    return Y


class GenerationClock:
    """A logger that notes when the first generation starts (the epoch logs one line per generation)."""

    def __init__(self):
        self.t_first = None

    def info(self, msg):
        if self.t_first is None and ": generation 1 of" in msg:
            self.t_first = time.perf_counter()


def epoch(fn, sm, X, Y, a):
    import dmosopt_b200 as b2
    from dmosopt_b200 import _lib

    model = b2.Model(objective=sm)
    opt = b2.NSGA2(popsize=a.pop, nInput=a.d, nOutput=a.M, model=model, distance_metric=None)
    xlb, xub = np.zeros(a.d), np.ones(a.d)
    clock = GenerationClock()
    _lib.synchronize()
    w0, (h0, d0) = _lib.wait_count(), _lib.transfer_bytes()
    gen = fn(a.gens, opt, model, a.d, a.M, xlb, xub, popsize=a.pop, initial=(X, Y), local_random=np.random.default_rng(a.seed), logger=clock)
    try:
        next(gen)
        raise RuntimeError("the epoch yielded although a surrogate is present")
    except StopIteration as ex:
        res = ex.value
    t = time.perf_counter() - clock.t_first
    w1, (h1, d1) = _lib.wait_count(), _lib.transfer_bytes()
    children = int(np.count_nonzero(res.gen_index > 0))
    return res, {"ms_per_gen": 1e3 * t / a.gens, "candidates_per_s": children / t, "waits_per_gen": (w1 - w0) / a.gens,
                 "h2d_bytes_per_gen": (h1 - h0) / a.gens, "d2h_bytes_per_gen": (d1 - d0) / a.gens}


def same(r, s):
    return all(getattr(r, f).dtype == getattr(s, f).dtype and np.array_equal(getattr(r, f), getattr(s, f))
               for f in ("best_x", "best_y", "gen_index", "x", "y"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pop", type=int, default=65536)
    ap.add_argument("--d", type=int, default=30)
    ap.add_argument("--M", type=int, default=3)
    ap.add_argument("--train", type=int, default=4096)
    ap.add_argument("--gens", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=2026)
    a = ap.parse_args()

    import dmosopt_b200 as b2
    from dmosopt_b200 import MOASMO

    print(json.dumps({"card": card(), "pop": a.pop, "d": a.d, "M": a.M, "train": a.train, "gens": a.gens, "rounds": a.rounds}), flush=True)
    rng = np.random.default_rng(a.seed)
    X = rng.random((a.train, a.d))
    Y = dtlz2(X, a.M)
    sm = b2.GPR_Matern(X, Y, a.d, a.M, np.zeros(a.d), np.ones(a.d), optimizer=None)
    routes = {"resident": MOASMO.optimize, "plugin": MOASMO.optimize_per_generation}
    rows = {k: [] for k in routes}
    for rnd in range(a.rounds + 1):  # round 0 warms up both routes
        res = {}
        for name, fn in routes.items():
            res[name], row = epoch(fn, sm, X, Y, a)
            if rnd > 0:
                rows[name].append(row)
        if not same(res["resident"], res["plugin"]):
            raise SystemExit(f"round {rnd}: the resident epoch's results differ from the plugin loop's")
    for name, rs in rows.items():
        out = {"route": name, "identical": True}
        for k in rs[0]:
            out[k] = float(np.median([r[k] for r in rs]))
        out["ms_per_gen_all"] = [round(r["ms_per_gen"], 3) for r in rs]
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
