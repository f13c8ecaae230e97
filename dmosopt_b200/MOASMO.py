"""Host-side mirror of dmosopt's MOASMO result helpers, backed by the CUDA library.

  * ``epsilon_get_best``   MOASMO.py:703-758 -> MOEA.get_duplicates (dmo_get_duplicates) + dmo_epsilon_sort
"""

import numpy as np
from scipy import stats

from . import MOEA, _lib


def epsilon_get_best(x, y, f, c, feasible=True, delete_duplicates=True, epsilons=None):
    """The epsilon-nondominated rows of a run's evaluations: (x[m], y[m], f[m], c[m], epsilons).

    As the reference: infeasible rows (some c <= 0) are dropped only when some row is feasible, then duplicate rows of
    y; ``epsilons`` is None (1e-9 per objective), a number, a sequence or "auto" (5 % of the inter-quartile range of the
    remaining y); an empty set returns early.  The archive is one ``dmo_epsilon_sort`` call over every row in order.
    Unlike the reference under NumPy 2 (``epsilons == "auto"`` raises ValueError on an array of several epsilons), a
    NumPy array is accepted like a list.
    """
    if feasible and c is not None:
        feasible = np.argwhere(np.all(c > 0.0, axis=1)).ravel()
        if len(feasible) > 0:
            x = x[feasible, :]
            y = y[feasible, :]
            if f is not None:
                f = f[feasible]
            c = c[feasible, :]

    if delete_duplicates:
        is_duplicate = MOEA.get_duplicates(y)
        x = x[~is_duplicate]
        y = y[~is_duplicate]
        if f is not None:
            f = f[~is_duplicate]
        if c is not None:
            c = c[~is_duplicate]

    if epsilons is None:
        epsilons = [1e-9] * y.shape[1]
    elif isinstance(epsilons, (int, float)):
        epsilons = [float(epsilons)] * y.shape[1]
    elif isinstance(epsilons, str) and epsilons == "auto":
        epsilons = 0.05 * stats.iqr(y, axis=0)

    if y.shape[0] == 0:
        return x, y, f, c, epsilons

    m = _lib.epsilon_sort(y, epsilons)
    return x[m], y[m], (None if f is None else f[m]), (None if c is None else c[m]), epsilons
