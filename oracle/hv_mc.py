"""Oracle: the Monte-Carlo hypervolume estimators (row A16 of SURVEY.md section 8a, the non-'box' branches).

Test infrastructure only (see oracle/__init__.py).

NumPy restatement, one sample at a time, of
  * ``_compute_standard_mc``          -> dmosopt/hv.py:191-241
  * ``_run_fpras_round`` / ``compute_hypervolume_fpras``  -> dmosopt/hv_adaptive.py:188-348
  * ``compute_hypervolume_mcm2rv``    -> dmosopt/hv_adaptive.py:356-460
on the front csrc/hv_mc.cu estimates: the rows strictly inside ref, then their non-dominated subset.  The random
stream is NumPy's; the GPU draws the same random variables from Philox.
"""

import math

import numpy as np


def filtered_front(F, ref):
    F = np.asarray(F, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    P = F[np.all(F < ref, axis=1)]
    keep = [i for i in range(len(P)) if not np.any(np.all(P <= P[i], axis=1) & np.any(P < P[i], axis=1))]
    return P[keep]


def fpras(F, ref, epsilon, delta, rng):
    """(estimate, N, tests): box i with probability v_i / W, x uniform in it, xi = tests until a row f_k < x."""
    P = filtered_front(F, ref)
    n, _ = P.shape
    v = np.prod(ref - P, axis=1)
    W = v.sum()
    budget = int(8 * (1 + epsilon) * n * np.log(2 / delta) / epsilon**2)
    tests, sum_xi, N = 0, 0, 0
    while tests < budget:
        j = rng.choice(n, p=v / W)
        x = rng.uniform(P[j], ref)
        xi = 0
        while tests < budget:
            xi += 1
            tests += 1
            if np.all(x > P[rng.integers(n)]):
                sum_xi += xi
                N += 1
                break
    return (W / n) * sum_xi / max(N, 1), N, tests


def mcm2rv(F, ref, epsilon, delta, rng):
    """(estimate, N, S): x uniform in [ideal, ref]; for dominated x, eta = [f_k <= x] for one uniform row k; stop at S >= R."""
    P = filtered_front(F, ref)
    n, _ = P.shape
    W = np.prod(ref - P, axis=1).sum()
    ideal = P.min(axis=0)
    R = int(math.floor((4 * (1 + epsilon * (1 - epsilon)) * np.log(2 / delta)) / (epsilon**2 * (1 - epsilon) ** 2)))
    S = N = 0
    while S < R:
        x = rng.uniform(ideal, ref)
        if not np.any(np.all(P <= x, axis=1)):
            continue
        N += 1
        S += int(np.all(P[rng.integers(n)] <= x))
    return (W / n) * N / S, N, S


def monte_carlo(F, ref, n_samples, rng):
    P = filtered_front(F, ref)
    lo = P.min(axis=0)
    X = rng.uniform(lo, ref, size=(n_samples, P.shape[1]))
    dom = np.any(np.all(X[:, None, :] >= P[None, :, :], axis=2), axis=1)
    return float(np.prod(ref - lo) * dom.mean())
