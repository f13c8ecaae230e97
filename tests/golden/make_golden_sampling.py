#!/usr/bin/env python
"""Generate tests/golden/sampling.npz from the *reference itself*: ``dmosopt.sampling.glp`` and ``dmosopt.discrepancy``.

Run with the reference package importable (a checkout of dmosopt on PYTHONPATH):

    PYTHONPATH=<dmosopt checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_sampling.py

Nothing outside ``tests/golden/`` is written.  Takes about a minute (the reference's CD2 is a Python triple loop).
"""

import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# (n, s, maxiter, seed) -> branch:
GLP_CASES = [
    (13, 3, 0, 1),   # column combinations, lattice 13
    (11, 2, 5, 2),   # column combinations, lattice 11, decorrelated
    (12, 3, 0, 3),   # column combinations, plusone (lattice 13)
    (10, 2, 5, 4),   # column combinations, plusone (lattice 11), decorrelated
    (12, 1, 0, 5),   # column combinations, s = 1
    (2, 3, 0, 6),    # column combinations, plusone, no combination (3 columns of 2): the (3, 3) uniform draw
    (60, 6, 0, 7),   # power vectors, plusone, 61 prime
    (60, 6, 5, 8),   # the same, decorrelated
    (100, 10, 0, 9),  # power vectors, plusone, 101 prime
    (150, 4, 0, 10),  # power vectors, plusone, 151 prime
    (61, 5, 0, 11),  # power vectors, 61 prime
    (67, 8, 5, 12),  # power vectors, 67 prime, decorrelated
    (90, 30, 0, 13),  # power vectors, plusone, lattice 91 of exponent 12: no candidate, the (91, 30) uniform draw
    (90, 30, 5, 14),  # the same, decorrelated
]
METRICS = ("MD2", "CD2", "SD2", "WD2", "MinDist", "corrscore")


def save(name, **arrays):
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **arrays)
    print(f"wrote {name}.npz  ({os.path.getsize(path)} bytes)")


def main():
    from dmosopt import GLP, discrepancy, sampling

    out = {"glp_cases": np.array(GLP_CASES, dtype=np.int64)}
    designs = []
    for c, (n, s, maxiter, seed) in enumerate(GLP_CASES):
        rng = np.random.default_rng(seed)
        X = sampling.glp(n, s, rng, maxiter=maxiter)
        out[f"glp_{c}"] = X
        out[f"glp_{c}_next"] = rng.random(4)  # the generator's state after the call
        if (n, s) == (90, 30):  # no candidate survives: the result is the discarded draw
            assert GLP.PowerGenVector(91, 30).shape[0] == 0 and X.shape == (91, 30)
            if maxiter == 0:
                assert np.array_equal(X, np.random.default_rng(seed).uniform(0, 1, size=[91, 30]))
        if maxiter == 0 and X.shape[0] <= 150:
            designs.append(X)
        print(f"glp n={n} s={s} maxiter={maxiter}: {X.shape}")
    rng = np.random.default_rng(99)
    designs += [rng.random((20, 3)), rng.random((50, 5)), rng.random((37, 8)), rng.random((2, 4))]
    for i, X in enumerate(designs):
        out[f"disc_{i}_X"] = X
        out[f"disc_{i}"] = np.array([float(getattr(discrepancy, m)(X)) for m in METRICS])
    out["disc_count"] = np.array(len(designs))
    save("sampling", **out)


if __name__ == "__main__":
    main()
