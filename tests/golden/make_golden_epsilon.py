#!/usr/bin/env python
"""Generate tests/golden/epsilon.npz from the *reference itself*: ``dmosopt.MOEA.EpsilonSort`` and
``dmosopt.MOASMO.epsilon_get_best``.

Run from the repository root with the reference package importable (a checkout of dmosopt on PYTHONPATH):

    PYTHONPATH=<dmosopt checkout>:. PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_epsilon.py

Class cases ``cls_<name>``: rows Y, epsilons, and the tag-alongs (row indices) the archive holds after ``sortinto`` of
every row in order.  ``epsilon_get_best`` cases ``gb_<name>``: x, y, f, c, the epsilons argument and the five returned
values.  The reference squares with libm ``pow``, which can differ from a correctly rounded square by one ulp; random
cases are kept only where, in every box, the best and second-best distances are equal or more than 4 ulp apart, so the
recorded pick does not hang on that last bit.  Nothing outside ``tests/golden/`` is written.
"""

import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import epsilon as oe  # noqa: E402


def robust(Y, eps):
    """Every box's best and second-best distances are equal or more than 4 ulp apart."""
    _, box, dist = oe.boxes_and_dist(Y, eps)
    _, inv = np.unique(box, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    for g in np.unique(inv):
        d = np.sort(dist[inv == g])
        if len(d) > 1 and np.isfinite(d[0]):
            gap = d[1] - d[0]
            if gap != 0 and gap <= 4 * np.spacing(d[1]):
                return False
    return True


def near_front(rng, n, M, noise):
    x = np.abs(rng.standard_normal((n, M))) + 1e-3
    return x / np.linalg.norm(x, axis=1, keepdims=True) + noise * rng.random((n, M))


def class_cases():
    rng = np.random.default_rng(20261016)
    cases = {}
    for M in (2, 3, 5, 10, 16):
        n = 400 if M <= 5 else 250
        cases[f"rand{M}"] = (rng.random((n, M)), [1e-9] * M)
        cases[f"rand{M}_coarse"] = (rng.random((n, M)), [0.1] * M)
        cases[f"front{M}"] = (near_front(rng, n, M, 0.02), [0.02] * M)
    # dyadic grid: shared boxes, exact distance ties (permuted offsets), duplicate rows
    for M in (2, 3, 5):
        Y = rng.integers(0, 24, (300, M)) / 8.0
        Y[:, -1] = 3.0 * (M - 1) - Y[:, :-1].sum(axis=1) + rng.integers(0, 8, 300) / 8.0  # around a plane: many boxes survive
        Y[rng.integers(0, 300, 60)] = Y[rng.integers(0, 300, 60)]
        cases[f"dyadic{M}"] = (Y, [0.5] * M)
        base = rng.integers(0, 6, (100, M)).astype(float)
        base[:, -1] = 5.0 * (M - 1) - base[:, :-1].sum(axis=1)
        off = rng.integers(0, 4, (100, M)) / 8.0
        Yp = np.vstack([base + off, base + off[:, ::-1], base + np.roll(off, 1, axis=1)])
        cases[f"perm{M}"] = (Yp[rng.permutation(len(Yp))], [1.0] * M)
    cases["negative3"] = (rng.standard_normal((300, 3)) * 5 - 2, [0.25, 0.5, 1.0])
    Y = rng.random((200, 3)) * 4
    Y[rng.integers(0, 200, 15), rng.integers(0, 3, 15)] = np.nan
    Y[rng.integers(0, 200, 8), rng.integers(0, 3, 8)] = np.inf
    Y[rng.integers(0, 200, 8), rng.integers(0, 3, 8)] = -np.inf
    cases["naninf3"] = (Y, [1.0, 3.0, 1.5])
    cases["eps_zero_nan"] = (rng.random((300, 3)), [0.0, np.nan, 0.1])
    cases["eps_negative"] = (rng.random((300, 3)) - 0.5, [0.1, -0.2, 0.15])
    cases["eps_inf"] = (rng.integers(0, 4, (120, 2)) - 1.5, [np.inf, 1.0])
    cases["wide_rows"] = (rng.random((300, 5)), [0.05, 0.05, 0.05])
    cases["n1"] = (rng.random((1, 4)), [0.1] * 4)
    return cases


def get_best_cases():
    rng = np.random.default_rng(7)
    n, d, M = 300, 4, 3
    x = rng.random((n, d))
    y = near_front(rng, n, M, 0.05)
    y[10] = y[3]
    y[200] = y[3]
    f = rng.random((n, 2))
    c = rng.standard_normal((n, 2)) + 1.0
    out = {
        "default": (x, y, f, c, True, None),
        "scalar": (x, y, None, None, True, 0.05),
        "auto": (x, y, f, c, True, "auto"),
        "list": (x, y, f, None, True, [0.02, 0.05, 0.1]),
        "infeasible": (x, y, f, -np.abs(c), True, 0.05),
        "nofilter": (x, y, f, c, False, 0.05),
        "n1": (x[:1], y[:1], f[:1], c[:1], True, "auto"),
    }
    return out


def main():
    from dmosopt import MOASMO, MOEA

    warnings.simplefilter("ignore")
    data = {}
    for name, (Y, eps) in class_cases().items():
        assert name.startswith(("dyadic", "perm", "eps_inf")) or robust(Y, eps), name
        s = MOEA.EpsilonSort(eps)
        for i in range(Y.shape[0]):
            s.sortinto(Y[i], tagalong=i)
        data[f"cls_{name}_Y"] = Y
        data[f"cls_{name}_eps"] = np.asarray(eps, dtype=np.float64)
        data[f"cls_{name}_idx"] = np.asarray(s.tagalongs, dtype=np.int64)
        print(f"{name}: n {Y.shape[0]} M {len(eps)} kept {len(s.tagalongs)}")
    for name, (x, y, f, c, feas, eps) in get_best_cases().items():
        bx, by, bf, bc, be = MOASMO.epsilon_get_best(x, y, f, c, feasible=feas, epsilons=eps)
        p = f"gb_{name}_"
        data[p + "x"], data[p + "y"] = x, y
        if f is not None:
            data[p + "f"] = f
        if c is not None:
            data[p + "c"] = c
        data[p + "feasible"] = np.array(feas)
        data[p + "eps_arg"] = np.array("none" if eps is None else eps if isinstance(eps, str) else np.asarray(eps, dtype=np.float64))
        data[p + "bx"], data[p + "by"], data[p + "beps"] = bx, by, np.asarray(be, dtype=np.float64)
        if bf is not None:
            data[p + "bf"] = bf
        if bc is not None:
            data[p + "bc"] = bc
        print(f"get_best {name}: kept {by.shape[0]}")
    np.savez_compressed(os.path.join(HERE, "epsilon.npz"), **data)


if __name__ == "__main__":
    main()
