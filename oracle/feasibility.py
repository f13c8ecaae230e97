"""NumPy / SciPy restatement of the logistic feasibility model (dmosopt/feasibility.py) as dmosopt_b200.feasibility
defines it: stratified folds, the covariance-eigh PCA, the scaler, the L1-logistic optimum and the grid choice.

The L1 problem min_w,b C sum log(1 + exp(-s_i (z_i w + b))) + |w|_1 is solved independently of the GPU's proximal
Newton: L-BFGS-B on w = u - v with u, v >= 0 (a smooth bound-constrained problem) to gtol 1e-12.
"""

import numpy as np
from scipy.optimize import minimize

C_GRID = np.logspace(-4, 4, 4)
N_FOLDS = 5


def test_folds(c, n_splits=N_FOLDS):
    """StratifiedKFold(n_splits, shuffle=False) test-fold id of each row (sklearn's _make_test_folds)."""
    c = np.asarray(c).ravel()
    _, y_idx, y_inv = np.unique(c, return_index=True, return_inverse=True)
    _, class_perm = np.unique(y_idx, return_inverse=True)
    enc = class_perm[y_inv.ravel()]
    ncls = len(y_idx)
    order = np.sort(enc)
    alloc = np.asarray([np.bincount(order[i::n_splits], minlength=ncls) for i in range(n_splits)])
    folds = np.empty(len(c), dtype=int)
    for k in range(ncls):
        folds[enc == k] = np.arange(n_splits).repeat(alloc[:, k])
    return folds


def pca(X):
    """(mean, components (d, d)) as PCA(svd_solver="covariance_eigh"): eigh of (X^T X - n m m^T) / (n - 1), descending,
    each component's largest-|.| entry positive (svd_flip on V)."""
    X = np.asarray(X, dtype=np.float64)
    n = X.shape[0]
    m = X.mean(axis=0)
    C = X.T @ X - n * np.outer(m, m)
    C /= n - 1
    _, V = np.linalg.eigh(C)
    V = V[:, ::-1].T.copy()
    idx = np.argmax(np.abs(V), axis=1)
    return m, V * np.sign(V[np.arange(len(V)), idx])[:, None]


def scaler(Z):
    """StandardScaler's mean_ and scale_ (population std; a column constant to rounding keeps scale 1)."""
    n = Z.shape[0]
    m = Z.mean(axis=0)
    var = ((Z - m) ** 2).mean(axis=0)
    eps = np.finfo(np.float64).eps
    const = var <= n * eps * var + (n * m * eps) ** 2
    return m, np.where(const | (var == 0.0), 1.0, np.sqrt(var))


def objective(Z, y, C, w, b):
    t = Z @ w + b
    m = np.where(y > 0, t, -t)
    return C * np.sum(np.logaddexp(0.0, -m)) + np.sum(np.abs(w))


def l1_logistic(Z, y, C, gtol=1e-12):
    """(w, b, objective) minimising C sum log(1 + exp(-s_i (z_i w + b))) + |w|_1 (y in {0, 1}, s = 2 y - 1)."""
    n, k = Z.shape
    s = np.where(y > 0, 1.0, -1.0)

    def f(v):
        u, q, b = v[:k], v[k:2 * k], v[2 * k]
        t = Z @ (u - q) + b
        m = s * t
        loss = C * np.sum(np.logaddexp(0.0, -m)) + np.sum(u) + np.sum(q)
        r = -C * s * np.exp(-np.logaddexp(0.0, m))  # d loss / d t
        gw = Z.T @ r
        return loss, np.concatenate((gw + 1.0, -gw + 1.0, [np.sum(r)]))

    bounds = [(0.0, None)] * (2 * k) + [(None, None)]
    res = minimize(f, np.zeros(2 * k + 1), jac=True, method="L-BFGS-B", bounds=bounds,
                   options={"gtol": gtol, "ftol": 1e-16, "maxiter": 100000, "maxfun": 200000, "maxcor": 30})
    w = res.x[:k] - res.x[k:2 * k]
    w, b = _polish(Z, y, C, w, res.x[2 * k])
    return w, b, objective(Z, y, C, w, b)


def _polish(Z, y, C, w, b, steps=8):
    """Newton steps on the smooth problem of L-BFGS-B's support and signs (F is smooth there), kept while no sign flips
    and F does not grow, or grows by no more than its rounding (n eps |F|) while the gradient shrinks: at large C the
    bound-constrained search stops on its f-tolerance short of the optimum, and near the optimum a Newton step's
    decrease of F is below F's rounding."""
    s = np.where(y > 0, 1.0, -1.0)
    S = np.flatnonzero(w != 0.0)
    sg = np.sign(w[S])
    A = np.column_stack((Z[:, S], np.ones(len(Z))))
    F = objective(Z, y, C, w, b)
    slack = len(Z) * np.finfo(np.float64).eps

    def grad(w, b):
        t = Z @ w + b
        p = 1.0 / (1.0 + np.exp(-t))
        return p, A.T @ (C * (p - (s > 0))) + np.append(sg, 0.0)

    p, g = grad(w, b)
    for _ in range(steps):
        H = (A * (C * p * (1 - p))[:, None]).T @ A
        step = np.linalg.solve(H, -g)
        w2 = w.copy()
        w2[S] += step[:-1]
        b2 = b + step[-1]
        F2 = objective(Z, y, C, w2, b2)
        p2, g2 = grad(w2, b2)
        if np.any(np.sign(w2[S]) != sg) or F2 > F + slack * abs(F) or (F2 > F and np.max(np.abs(g2)) >= np.max(np.abs(g))):
            break
        w, b, F, p, g = w2, b2, F2, p2, g2
    return w, b


def dataset(X, train):
    """(mean, components (d-1, d), scaler mean, scaler scale, Z of all rows standardised) of the training rows."""
    d = X.shape[1]
    m, V = pca(X[train])
    V = V[: d - 1]
    U = (X - m) @ V.T
    sm, ss = scaler(U[train])
    return m, V, sm, ss, (U - sm) / ss


def grid_search(X, c, Cs=C_GRID, problems=False):
    """The feasibility model of one two-class constraint.  Returns (k, C, mean, comps (k, d), smean, sscale, coef,
    intercept) and, with problems=True, {(f, ci, k): (w, b, objective, held-out correct or None)} as well."""
    X = np.asarray(X, dtype=np.float64)
    N, d = X.shape
    if d < 2:
        raise ValueError("d == 1: the n_components grid is empty")
    c = np.asarray(c).astype(int)
    folds = test_folds(c)
    sets = [folds != f for f in range(N_FOLDS)] + [np.ones(N, dtype=bool)]
    detail = {}
    scores = np.full((len(Cs), d - 1, N_FOLDS), np.nan)
    prep = [dataset(X, tr) for tr in sets]
    for f, tr in enumerate(sets):
        if np.unique(c[tr]).size < 2:
            continue
        Z = prep[f][4]
        for ci, C in enumerate(Cs):
            for k in range(1, d):
                w, b, F = l1_logistic(Z[tr, :k], c[tr], C)
                cor = None
                if f < N_FOLDS:
                    te = ~tr
                    cor = int(np.count_nonzero((Z[te, :k] @ w + b > 0) == (c[te] > 0)))
                    scores[ci, k - 1, f] = cor / np.count_nonzero(te)
                detail[(f, ci, k)] = (w, b, F, cor)
    means = np.mean(scores, axis=2).ravel()
    best = 0 if np.all(np.isnan(means)) else int(np.nanargmax(means))
    ci, k = divmod(best, d - 1)
    k += 1
    m, V, sm, ss, Z = prep[N_FOLDS]
    w, b, _, _ = detail[(N_FOLDS, ci, k)]
    hp = (k, float(Cs[ci]), m, V[:k], sm[:k], ss[:k], w, float(b))
    return (hp, detail, means.reshape(len(Cs), d - 1)) if problems else hp


def fit(X, C):
    """Per constraint: None (single class) or the grid_search hyperparameters."""
    C = np.asarray(C)
    if np.asarray(X).shape[1] < 2:
        raise ValueError("d == 1: the n_components grid is empty")
    out = []
    for j in range(C.shape[1]):
        c = (C[:, j] > 0.0).astype(int)
        out.append(None if np.unique(c).size < 2 else grid_search(X, c))
    return out


def proba(hyper, x):
    """(J, n) feasible probabilities: centre, project, standardise, dot, expit."""
    x = np.asarray(x, dtype=np.float64)
    P = []
    for h in hyper:
        if h is None:
            P.append(np.ones(x.shape[0]))
            continue
        k, _, m, V, sm, ss, w, b = h
        z = (((x - m) @ np.asarray(V).reshape(k, -1).T) - sm) / ss
        P.append(1.0 / (1.0 + np.exp(-(z @ w + b))))
    return np.array(P)


def rank(hyper, x):
    return np.mean(proba(hyper, x), axis=0)
