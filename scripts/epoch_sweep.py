#!/usr/bin/env python
"""One MOASMO.optimize surrogate epoch, resident against the per-generation plugin loop, at bench.py's shape.

    python scripts/epoch_sweep.py [--pop 65536] [--d 30] [--M 3] [--train 4096] [--gens 50] [--rounds 3]
                                  [--surrogate GPR_Matern] [--precision auto] [--optimizer NSGA2] [--swarm-size 5]

NSGA2 (distance_metric=None, as MOASMO.epoch builds it) with a GPR_Matern surrogate (precision "auto", the
hyper-parameters kept at their initial values) fitted on DTLZ2 data; --optimizer SMPSO runs SMPSO with --swarm-size
swarms of --pop particles instead (2 * swarm_size * pop candidates per generation), --optimizer CMAES runs MO-CMA-ES with
its default parameters (mu = pop // 2, lambda_ = 1: pop // 2 offspring per generation); the training set is the epoch's ``initial`` rows, as
MOASMO.epoch passes it.  --surrogate EGP_Matern, SVGP_Matern, VGP_Matern, SIV_Matern, SPV_Matern, MDSPP_Matern or
MDGP_Matern (--precision fp64 or tensor) builds that class from seeded hyper-parameters instead, with no training: EGP
with one length scale per objective, the variational classes with their own inducing-point rule (SVGP: 0.2 N points per
output, VGP: every training point) and the optimal q, the deep GPs with 3 hidden units and 128 inducing points per layer
(MDSPP: 8 quadrature sites, MDGP: 10 draws).  These epochs also time a third route, "plugin_mean_only": the plugin loop
with the surrogate's ``evaluate`` replaced, inside this script only, by the mean-only predict.  Its results need not
equal the others' (the exact GP's mean-only tensor kernel agrees with the variance route's mean to 1e-5 only); whether
they do is reported.  MDGP's call counter is reset before every epoch, so that every route draws the same keys.  The two routes alternate in one process, --rounds times each after one warm-up epoch of each,
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


def surrogate(a, X, Y):
    """The --surrogate class on (X, Y) in the unit cube."""
    import dmosopt_b200 as b2
    from dmosopt_b200 import model_gpflow as mf
    from dmosopt_b200 import model_gpytorch as mg

    d, M, name = a.d, a.M, a.surrogate
    xlb, xub = np.zeros(d), np.ones(d)
    if name in ("GPR_Matern", "GPR_RBF"):
        return getattr(b2, name)(X, Y, d, M, xlb, xub, optimizer=None, precision=a.precision)
    rng = np.random.default_rng(a.seed + 1)
    if name == "EGP_Matern":
        ls = np.sqrt(d) * (0.3 + 0.3 * rng.random((M, 1)))
        hp = dict(lengthscale=np.broadcast_to(ls, (M, d)).copy(), outputscale=0.5 + rng.random(M), noise=np.full(M, 1e-3),
                  weight=0.1 * rng.standard_normal((M, d)), bias=0.1 * rng.standard_normal(M))
        return mg.EGP_Matern(X, Y, d, M, xlb, xub, hyperparameters=hp, precision=a.precision)
    if name in ("SVGP_Matern", "VGP_Matern", "SIV_Matern", "SPV_Matern"):
        ls = np.sqrt(d) * (0.4 + 0.6 * rng.random((M, d)))
        var = 0.5 + rng.random(M)
        if name == "SIV_Matern":
            ls[:], var[:] = ls[0], var[0]
        return getattr(mf, name)(X, Y, d, M, xlb, xub, hyperparameters=dict(lengthscales=ls, variance=var, likelihood_variance=1e-3),
                                 precision=a.precision, seed=a.seed, return_mean_variance=False)
    H, Z = 3, 128

    def chol(n, m):
        c = np.tril(0.3 * rng.standard_normal((n, m, m)), -1)
        c[:, np.arange(m), np.arange(m)] = 0.2 + 0.5 * rng.random((n, m))
        return c

    hp = {"hidden_inducing_points": np.broadcast_to(rng.random((Z, d)), (H, Z, d)).copy(), "hidden_outputscale": 0.5 + rng.random(H),
          "hidden_lengthscale": np.sqrt(d) * (0.3 + 0.4 * rng.random((H, d))), "hidden_variational_mean": rng.standard_normal((H, Z)),
          "hidden_chol_variational_covar": chol(H, Z), "mean_weights": 0.5 * rng.standard_normal(d), "mean_bias": float(rng.standard_normal()),
          "last_inducing_points": 1.5 * rng.standard_normal((M, Z, H)), "last_outputscale": 0.5 + rng.random(M),
          "last_lengthscale": 1.0 + rng.random((M, H)), "last_variational_mean": rng.standard_normal((M, Z)),
          "last_chol_variational_covar": chol(M, Z), "mean_constant": float(rng.standard_normal()),
          "task_noises": 1e-3 + 1e-2 * rng.random(M), "noise": 2e-3}
    if name == "MDSPP_Matern":
        hp["quad_sites"] = rng.standard_normal((8, H))
    return getattr(mg, name)(X, Y, d, M, xlb, xub, hyperparameters=hp, precision=a.precision)


def mean_only(sm):
    """The surrogate's evaluate as its mean-only predict (the third route's stand-in)."""
    from dmosopt_b200 import _lib

    kind, h, prec, dtype = sm.resident_posterior()
    if kind == _lib.POSTERIOR_DGP:
        def ev(x):
            seed, stream = sm._draw_key()
            return h.predict(np.asarray(x, dtype=np.float64), seed=seed, stream_id=stream, return_var=False, precision=prec)[0]
    else:
        def ev(x):
            return h.predict(np.asarray(x, dtype=np.float64), return_var=False, precision=prec)[0].astype(dtype)
    return ev


def epoch(fn, sm, X, Y, a, evaluate=None):
    import dmosopt_b200 as b2
    from dmosopt_b200 import _lib

    if hasattr(sm, "calls"):
        sm.calls = 0
    saved = sm.__dict__.get("evaluate")
    if evaluate is not None:
        sm.evaluate = evaluate
    model = b2.Model(objective=sm)
    if a.optimizer == "SMPSO":
        opt = b2.SMPSO(popsize=a.pop, nInput=a.d, nOutput=a.M, model=model, distance_metric=None, swarm_size=a.swarm_size)
    elif a.optimizer == "CMAES":
        opt = b2.CMAES(popsize=a.pop, nInput=a.d, nOutput=a.M, model=model, distance_metric=None)
    else:
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
    finally:
        if evaluate is not None:
            if saved is None:
                del sm.evaluate
            else:
                sm.evaluate = saved
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
    ap.add_argument("--surrogate", default="GPR_Matern")
    ap.add_argument("--precision", default="auto")
    ap.add_argument("--optimizer", default="NSGA2", choices=("NSGA2", "SMPSO", "CMAES"))
    ap.add_argument("--swarm-size", type=int, default=5)
    a = ap.parse_args()

    import dmosopt_b200 as b2
    from dmosopt_b200 import MOASMO

    print(json.dumps({"card": card(), "pop": a.pop, "d": a.d, "M": a.M, "train": a.train, "gens": a.gens, "rounds": a.rounds,
                      "surrogate": a.surrogate, "precision": a.precision, "optimizer": a.optimizer,
                      "swarm_size": a.swarm_size if a.optimizer == "SMPSO" else None}), flush=True)
    rng = np.random.default_rng(a.seed)
    X = rng.random((a.train, a.d))
    Y = dtlz2(X, a.M)
    sm = surrogate(a, X, Y)
    routes = {"resident": (MOASMO.optimize, None), "plugin": (MOASMO.optimize_per_generation, None)}
    if a.surrogate not in ("GPR_Matern", "GPR_RBF"):
        routes["plugin_mean_only"] = (MOASMO.optimize_per_generation, mean_only(sm))
    rows = {k: [] for k in routes}
    identical = {k: True for k in routes}
    for rnd in range(a.rounds + 1):  # round 0 warms up every route
        res = {}
        for name, (fn, ev) in routes.items():
            res[name], row = epoch(fn, sm, X, Y, a, ev)
            if rnd > 0:
                rows[name].append(row)
        if not same(res["resident"], res["plugin"]):
            raise SystemExit(f"round {rnd}: the resident epoch's results differ from the plugin loop's")
        if "plugin_mean_only" in res:
            identical["plugin_mean_only"] &= same(res["resident"], res["plugin_mean_only"])
    for name, rs in rows.items():
        out = {"route": name, "identical": identical[name]}
        for k in rs[0]:
            out[k] = float(np.median([r[k] for r in rs]))
        out["ms_per_gen_all"] = [round(r["ms_per_gen"], 3) for r in rs]
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
