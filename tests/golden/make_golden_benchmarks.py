#!/usr/bin/env python
"""Generate tests/golden/benchmarks.npz from the *reference itself*: ``dmosopt.benchmarks.moo_benchmarks``.

Run with the reference package importable (a checkout of dmosopt on PYTHONPATH):

    PYTHONPATH=<dmosopt checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_benchmarks.py

Records, one decision vector at a time as the reference evaluates them:
* ``wfg1`` at (n_obj, n_var) = (2, 11), (3, 12) and the few-variable (4, 5), inputs scaled to [0, 2i] as the reference's
  runner scales them, plus rows holding nan, negative and infinite entries (np.max propagates nan);
* ``maf1``, ``maf2``, ``maf4`` at (3, 12), (5, 14), (10, 19) and (16, 25), inputs in [0, 1];
* the WFG1 shapes at which the reference raises (an empty np.max window), with the exception's type, and two that do
  not (an empty string);
* ``generate_problem_space`` for every problem name at n_obj 3, 5 and 10, for an unknown name, and with n_var given.
``tests/golden/trs.npz`` keeps the DTLZ / WFG4 / ZDT rows.  Nothing outside ``tests/golden/`` is written.
"""

import os
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

NAMES = ["dtlz1", "dtlz2", "dtlz3", "dtlz4", "dtlz5", "dtlz7", "wfg1", "wfg4", "maf1", "maf2", "maf4"]
WFG1_SHAPES = [(2, 11), (3, 12), (4, 5)]
MAF_SHAPES = [(3, 12), (5, 14), (10, 19), (16, 25)]
WFG1_RAISING = [(4, 6), (4, 12), (5, 14), (10, 19), (16, 25), (4, 5), (2, 2)]  # the last two are the edges that do not
SPACES = [(nm, M, None) for nm in NAMES + ["zdt1"] for M in (3, 5, 10)] + [("wfg1", 3, 7), ("maf2", 10, 12), ("zdt1", 2, 30)]


def rows(fn, X, M):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # nan / negative inputs: invalid-value warnings, as in the reference
        return np.vstack([np.asarray(fn(x, n_obj=M), dtype=np.float64).ravel() for x in X])


def main():
    from dmosopt.benchmarks import moo_benchmarks as mb

    rng = np.random.default_rng(20261016)
    out, keys = {}, []
    for M, d in WFG1_SHAPES:
        X = rng.random((24, d)) * 2 * np.arange(1, d + 1)
        X[20, 0] = np.nan  # first window, first entry
        X[21, d - 1] = np.nan  # last window and the mean
        X[22, M - 1] = -0.5 * (M + 1)  # y < 0: y ** 0.02 is nan
        X[23, d // 2] = np.inf
        key = f"wfg1_{M}_{d}"
        out[key + "_X"], out[key + "_Y"] = X, rows(mb.wfg1, X, M)
        keys.append(key)
    for nm in ("maf1", "maf2", "maf4"):
        for M, d in MAF_SHAPES:
            X = rng.random((20, d))
            key = f"{nm}_{M}_{d}"
            out[key + "_X"], out[key + "_Y"] = X, rows(getattr(mb, nm), X, M)
            keys.append(key)
    out["keys"] = np.array(keys)
    raised = []
    for M, d in WFG1_RAISING:
        try:
            mb.wfg1(rng.random(d) * 2 * np.arange(1, d + 1), n_obj=M)
            raised.append("")
        except Exception as e:  # noqa: BLE001 - record whatever the reference raises
            raised.append(type(e).__name__)
    out["wfg1_raising_shapes"], out["wfg1_raising_errors"] = np.array(WFG1_RAISING), np.array(raised)
    for i, (nm, M, d) in enumerate(SPACES):
        sp = mb.generate_problem_space(nm, M, d)
        out[f"space{i}_args"] = np.array([nm, str(M), "" if d is None else str(d)])
        out[f"space{i}_names"] = np.array(list(sp.keys()))
        out[f"space{i}_bounds"] = np.array(list(sp.values()), dtype=np.float64)
    out["n_spaces"] = np.array(len(SPACES))
    path = os.path.join(HERE, "benchmarks.npz")
    np.savez_compressed(path, **out)
    print(f"wrote benchmarks.npz  ({os.path.getsize(path)} bytes); wfg1 raises: {dict(zip(map(tuple, WFG1_RAISING), raised))}")


if __name__ == "__main__":
    main()
