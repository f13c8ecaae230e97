#!/usr/bin/env python
"""Feasibility model timings: the GPU fit against the reference's grid search on the host, the rank at n 131 072
against scikit-learn's pipelines, and one constrained NSGA-II update on the resident path against the host path.

    python scripts/feasibility_sweep.py [--host] [--reps 5] [--out results/feasibility_sweep.json]

--host also fits with scikit-learn (the reference's GridSearchCV(n_jobs=-1) pipeline) where that takes seconds, and
times its rank.  Wall-clock medians of --reps runs after one warm-up; every timed call returns with its results on the
host.  Prints one JSON line per measurement.
"""

import argparse
import json
import os
import sys
import time
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def data(N, d, J, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.random((N, d))
    W = rng.standard_normal((d, J))
    S = X @ W
    C = S - np.quantile(S, 0.4, axis=0)
    return X, np.where(rng.random(C.shape) < 0.1, -C, C)


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return float(np.median(ts)), fn


def sklearn_fit(X, C):
    from sklearn.decomposition import PCA
    from sklearn.linear_model import LogisticRegression
    from sklearn.model_selection import GridSearchCV
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import StandardScaler

    clfs = []
    for j in range(C.shape[1]):
        ppl = make_pipeline(PCA(), StandardScaler(), LogisticRegression(tol=0.01, penalty="l1", solver="saga"))
        grid = {"pca__n_components": range(1, X.shape[1]), "logisticregression__C": np.logspace(-4, 4, 4)}
        clfs.append(GridSearchCV(ppl, grid, n_jobs=-1).fit(X, (C[:, j] > 0).astype(int)))
    return clfs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--host", action="store_true")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import warnings

    warnings.filterwarnings("ignore")
    from dmosopt_b200 import _lib
    from dmosopt_b200.feasibility import LogisticFeasibilityModel

    _lib.context()
    rows = []

    def emit(**kw):
        kw["cores"] = os.cpu_count()
        print(json.dumps(kw), flush=True)
        rows.append(kw)

    # ---- fit
    for N in (1000, 4096):
        for d in (10, 30, 90):
            for J in (2, 8):
                X, C = data(N, d, J)
                t, _ = timed(lambda: LogisticFeasibilityModel(X, C), max(1, a.reps // 2))
                m = LogisticFeasibilityModel(X, C)
                left = sum(v["not_converged"] for v in m.fit_info["per_constraint"].values())
                iters = np.concatenate([v["iters"].ravel() for v in m.fit_info["per_constraint"].values()])
                emit(what="fit_gpu", N=N, d=d, J=J, s=t, problems=int(iters.size), max_newton=int(iters.max()), not_converged=int(left))
                if a.host and N * d * J <= 1000 * 30 * 2:
                    t0 = time.perf_counter()
                    sklearn_fit(X, C)
                    emit(what="fit_sklearn_host", N=N, d=d, J=J, s=time.perf_counter() - t0)
    # ---- rank at n 131 072
    n = 131072
    for d in (10, 30, 90):
        X, C = data(1000, d, 2, seed=1)
        m = LogisticFeasibilityModel(X, C)
        Q = np.random.default_rng(2).random((n, d))
        t, _ = timed(lambda: m.rank(Q), a.reps)
        emit(what="rank_gpu_host_rows", n=n, d=d, J=2, s=t, bytes_read=n * d * 8)
        mirrored, base = _lib.mirrored_readonly(Q)
        t, _ = timed(lambda: m.rank(mirrored), a.reps)
        emit(what="rank_gpu_device_rows", n=n, d=d, J=2, s=t, GBps=n * d * 8 / t / 1e9)
        if a.host and d <= 30:
            clfs = sklearn_fit(X, C)
            t, _ = timed(lambda: np.mean(np.stack([c.predict_proba(Q)[:, 1] for c in clfs]), axis=0), a.reps)
            emit(what="rank_sklearn_host", n=n, d=d, J=2, s=t)
    # ---- one constrained NSGA-II update at pop 65 536, d 30
    import dmosopt_b200 as b2
    from dmosopt_b200.MOEA import remove_worst

    d, M, pop = 30, 2, 65536
    X, C = data(2000, d, 2, seed=3)
    fm = LogisticFeasibilityModel(X, C)
    rng = np.random.default_rng(4)

    def f(x):
        return np.column_stack((x[:, 0], 1 - np.sqrt(x[:, 0]) + x[:, 1:].mean(axis=1)))

    opt = b2.NSGA2(popsize=pop, nInput=d, nOutput=M, model=types.SimpleNamespace(objective=None, feasibility=fm), distance_metric=None)
    x0 = rng.random((pop, d))
    opt.initialize_strategy(x0, f(x0), np.column_stack((np.zeros(d), np.ones(d))), rng)
    res, host = [], []
    for _ in range(a.reps + 1):
        x_gen, state = opt.generate()
        y_gen = f(np.asarray(x_gen))
        parm, obj = np.array(opt.state.population_parm), opt.state.population_obj.copy()
        t = time.perf_counter()
        remove_worst(np.vstack((x_gen, parm)), np.vstack((y_gen, obj)), pop, x_distance_metrics=[fm.rank], y_distance_metrics=None,
                     return_perm=True)
        host.append(time.perf_counter() - t)
        t = time.perf_counter()
        opt.update(x_gen, y_gen, state)
        res.append(time.perf_counter() - t)
    emit(what="nsga2_update_resident", pop=pop, d=d, J=2, s=float(np.median(res[1:])))
    emit(what="nsga2_update_host_path", pop=pop, d=d, J=2, s=float(np.median(host[1:])))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
