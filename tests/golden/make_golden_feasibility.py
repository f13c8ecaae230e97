#!/usr/bin/env python
"""Generate tests/golden/feasibility.npz from the *reference itself*: ``dmosopt.feasibility.LogisticFeasibilityModel``.

Run with the reference package importable (a checkout of dmosopt on PYTHONPATH):

    PYTHONPATH=<dmosopt checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_feasibility.py

The reference fits with saga from a row order drawn from NumPy's global stream inside joblib workers, so its pick is
not repeatable; the fixture records whatever it picked (k, C and the fitted pipeline of every constraint) together with
its ``predict_proba`` and ``rank`` on query rows.  Nothing outside ``tests/golden/`` is written.
"""

import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def tnk(X):
    """Constraints of the TNK problem (examples/example_dmosopt_tnk.py of dmosopt), x in [0, pi]^2."""
    c0 = -(np.square(X[:, 0]) + np.square(X[:, 1]) - 1.0 - 0.1 * np.cos(16.0 * np.arctan(X[:, 0] / X[:, 1])))
    c1 = 2 * (np.square(X[:, 0] - 0.5) + np.square(X[:, 1] - 0.5)) - 1
    return np.column_stack((c0, c1))


def datasets():
    rng = np.random.default_rng(20261016)
    out = {}
    X = rng.uniform(0.0, np.pi, (200, 2))
    out["tnk"] = (X, tnk(X), rng.uniform(0.0, np.pi, (500, 2)))
    d = 30
    X = rng.random((300, d))
    w = rng.standard_normal(d)
    C = np.column_stack((X @ w - np.median(X @ w) + 0.1 * rng.standard_normal(300), np.ones(300), X[:, 0] + X[:, 1] - 0.9))
    out["d30"] = (X, C, rng.random((400, d)))
    d = 5
    X = rng.random((120, d))
    c1 = -np.ones(120)
    c1[37] = 1.0  # one feasible row: its fold trains on one class
    out["single"] = (X, np.column_stack((X[:, 2] - 0.5, c1)), rng.random((200, d)))
    return out


def main():
    from dmosopt.feasibility import LogisticFeasibilityModel

    arrays = {}
    for name, (X, C, Q) in datasets().items():
        np.random.seed(7)
        m = LogisticFeasibilityModel(X, C)
        arrays[f"{name}_X"], arrays[f"{name}_C"], arrays[f"{name}_query"] = X, C, Q
        arrays[f"{name}_proba"] = m.predict_proba(Q)[:, :, 1]
        arrays[f"{name}_rank"] = m.rank(Q)
        for j, clf in enumerate(m.clfs):
            p = f"{name}_{j}_"
            if clf is None:
                arrays[p + "k"] = np.array(0)
                continue
            pca, sc, lr = (clf.best_estimator_[i] for i in range(3))
            arrays[p + "k"] = np.array(pca.n_components_)
            arrays[p + "C"] = np.array(clf.best_params_["logisticregression__C"])
            arrays[p + "pca_mean"], arrays[p + "components"] = pca.mean_, pca.components_
            arrays[p + "scaler_mean"], arrays[p + "scaler_scale"] = sc.mean_, sc.scale_
            arrays[p + "coef"], arrays[p + "intercept"] = lr.coef_[0], np.array(lr.intercept_[0])
        print(name, [None if c is None else (c.best_params_["pca__n_components"], c.best_params_["logisticregression__C"]) for c in m.clfs])
    path = os.path.join(HERE, "feasibility.npz")
    np.savez_compressed(path, **arrays)
    print(f"wrote feasibility.npz  ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
