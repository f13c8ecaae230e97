"""Vectorised benchmark objective functions on the GPU (SURVEY.md section 8f row N4).

Same names, signatures, defaults and formulas as ``dmosopt/benchmarks/moo_benchmarks.py`` (dtlz1 :21, dtlz2 :59,
dtlz3 :97, dtlz4 :136, dtlz5 :174, dtlz7 :218, wfg1 :286, wfg4 :335, and the many-objective MaF suite maf1 :384,
maf2 :422, maf4 :460) plus the two example objectives ZDT1 / ZDT3 (examples/example_dmosopt_zdt1.py:9-20,
examples/example_dmosopt_zdt3.py:9-21).  The reference functions take ONE decision vector; these take one (returning a
1-D array, drop-in) or a whole (n, n_var) matrix (returning (n, n_obj)), evaluated by dmo_benchmark_eval for
2 <= n_obj <= 16.  A matrix with a device mirror, such as the offspring an optimizer plugin's ``generate`` returns, is
read where it already is.

``generate_problem_space`` builds the reference's parameter space for a problem (moo_benchmarks.py:505-554).
WFG1 and WFG4 take only the default position parameter k = n_obj - 1.  WFG1 refuses, with ``ValueError``, the shapes
where the reference's ``np.max`` meets an empty window; at n_obj >= 4 and the default n_var = n_obj + 9 that is every
shape.
"""

import numpy as np

from . import _lib


def _eval(name, x, n_obj, **kw):
    x = np.asarray(x, dtype=np.float64)
    if x.ndim == 1:
        return _lib.benchmark_eval(name, x[None, :], n_obj, **kw)[0]
    return _lib.benchmark_eval(name, x, n_obj, **kw)


def _default_k(name, n_obj, k):
    if k is not None and k != n_obj - 1:
        raise NotImplementedError(f"{name}: only the reference's default position parameter k = n_obj - 1 is built")


def zdt1(x):
    return _eval("zdt1", x, 2)


def zdt3(x):
    return _eval("zdt3", x, 2)


def dtlz1(x, n_obj=3):
    return _eval("dtlz1", x, n_obj)


def dtlz2(x, n_obj=3):
    return _eval("dtlz2", x, n_obj)


def dtlz3(x, n_obj=3):
    return _eval("dtlz3", x, n_obj)


def dtlz4(x, n_obj=3, alpha=100.0):
    return _eval("dtlz4", x, n_obj, alpha=alpha)


def dtlz5(x, n_obj=3):
    return _eval("dtlz5", x, n_obj)


def dtlz7(x, n_obj=3):
    return _eval("dtlz7", x, n_obj)


def wfg1(x, n_obj=3, k=None):
    _default_k("wfg1", n_obj, k)
    n_var = np.shape(x)[-1]
    ll = n_var - (n_obj - 1)
    if (n_obj - 2) * ll >= n_var:  # the window of shape coordinate n_obj - 2 starts at or past the last variable
        raise ValueError(f"wfg1: n_obj={n_obj}, n_var={n_var}: the shape window [{(n_obj - 2) * ll}, {(n_obj - 1) * ll}) is empty; "
                         f"the reference's np.max fails there (it needs (n_obj - 2) (n_var - n_obj + 1) < n_var)")
    return _eval("wfg1", x, n_obj)


def wfg4(x, n_obj=3, k=None):
    _default_k("wfg4", n_obj, k)
    return _eval("wfg4", x, n_obj)


def maf1(x, n_obj=5):
    return _eval("maf1", x, n_obj)


def maf2(x, n_obj=5):
    return _eval("maf2", x, n_obj)


def maf4(x, n_obj=5):
    return _eval("maf4", x, n_obj)


def generate_problem_space(problem_name, n_obj, n_var=None):
    """dmosopt's ``space`` dict ``{"x1": [lo, hi], ...}`` for a benchmark problem.

    n_var defaults by family: n_obj + 4 for dtlz1 / dtlz3, n_obj + 19 for dtlz7, n_obj + 9 for the other DTLZ, every
    WFG (k = n_obj - 1 position and 10 distance variables) and every MaF problem, n_obj + 10 for any other name.
    WFG bounds are [0, 2i] for x_i; every other name, known or not, gets [0, 1]."""
    if n_var is None:
        if problem_name in ("dtlz1", "dtlz3"):
            n_var = n_obj + 4
        elif problem_name == "dtlz7":
            n_var = n_obj + 19
        elif problem_name.startswith(("dtlz", "wfg", "maf")):
            n_var = n_obj + 9
        else:
            n_var = n_obj + 10
    wfg = problem_name.startswith("wfg")
    return {f"x{i + 1}": [0.0, 2.0 * (i + 1) if wfg else 1.0] for i in range(n_var)}
