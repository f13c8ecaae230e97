"""Logistic feasibility model on the GPU: a drop-in for ``dmosopt.feasibility.LogisticFeasibilityModel``.

For each constraint j the label is ``C[:, j] > 0``.  A constraint whose label takes one value has no classifier and a
feasible probability of 1.0 for every row, even when every training row was infeasible (as in the reference).
Otherwise the model is the reference's grid search over ``PCA(k) -> StandardScaler -> L1 logistic regression``:
k in 1 .. d-1, C in ``np.logspace(-4, 4, 4)``, 5-fold ``StratifiedKFold`` without shuffling, accuracy, the first best
grid point (C outermost, then k) refitted on all rows.

With ``fit="gpu"`` (the default) every (fold or all rows, C, k) problem is solved to optimality in one batch on the
GPU (csrc/feasibility.cu): ``C sum log(1 + exp(-s_i (z_i w + b))) + |w|_1`` by proximal Newton.  The reference stops
saga after a few epochs (``tol=0.01``) from a random row order, so its pick is not repeatable; the converged optimum is.
The folds and the d x d covariance eigendecompositions are computed here in NumPy.  The components are the
eigenvectors of the centred covariance in descending eigenvalue order, with the largest-magnitude entry of each made
positive: scikit-learn's ``covariance_eigh``, which its ``auto`` policy picks when n >= 10 d.  Below that it uses a
full or randomized SVD, which spans the same subspace up to rounding or approximation.

``fit="sklearn"`` runs the reference's grid search with scikit-learn on the host and reads the fitted pipelines out.
Either way ``rank`` / ``predict_proba`` / ``predict`` run on the GPU.  ``predict`` returns ones for a single-class
constraint with one row per query row (the reference's ``np.ones((x.shape[1],))`` only works when n == d).

``train_with_feasibility`` is a ``surrogate_custom_training`` callable for dmosopt's ``MOASMO.epoch``: the controller's
own ``feasibility_method_name`` route cannot build a model (it calls the class with an unbound name and logs the
error), so this is how a constrained run gets one.
"""

import logging
import time

import numpy as np

from . import _lib

logger = logging.getLogger(__name__)

C_GRID = np.logspace(-4, 4, 4)
N_FOLDS = 5
N_SETS = N_FOLDS + 1  # the folds, then all rows


def stratified_test_folds(c, n_splits=N_FOLDS):
    """Test-fold id of every row: StratifiedKFold(n_splits) without shuffling.  Classes are numbered in order of first
    appearance; the rows of the sorted labels are dealt round-robin to the folds, and each class fills its folds in
    row order."""
    c = np.asarray(c).ravel()
    if c.size < n_splits:
        raise ValueError(f"cannot split {c.size} rows into {n_splits} folds")
    _, first, inv = np.unique(c, return_index=True, return_inverse=True)
    enc = np.argsort(np.argsort(first, kind="stable"), kind="stable")[inv.ravel()]
    ncls = first.size
    counts = np.bincount(enc, minlength=ncls)
    if np.all(counts < n_splits):
        raise ValueError(f"n_splits={n_splits} cannot be greater than the number of members in each class")
    srt = np.sort(enc)
    alloc = np.array([np.bincount(srt[i::n_splits], minlength=ncls) for i in range(n_splits)])
    out = np.empty(c.size, dtype=np.int8)
    for k in range(ncls):
        out[enc == k] = np.repeat(np.arange(n_splits), alloc[:, k])
    return out


def pca_components(X):
    """(mean, components (d, d)) of the rows of X: eigenvectors of (X^T X - n mean mean^T) / (n - 1) in descending
    eigenvalue order, each signed so that its largest-magnitude entry is positive."""
    X = np.asarray(X, dtype=np.float64)
    n = X.shape[0]
    mean = np.mean(X, axis=0)
    cov = X.T @ X
    cov -= n * mean[:, None] * mean[None, :]
    cov /= n - 1
    _, vec = np.linalg.eigh(cov)
    V = np.ascontiguousarray(np.flip(vec, axis=1).T)
    sign = np.sign(V[np.arange(V.shape[0]), np.argmax(np.abs(V), axis=1)])
    return mean, V * sign[:, None]


def _check_shape(d, J, N=None):
    if d < 2:
        raise ValueError(f"LogisticFeasibilityModel: d={d}: PCA's n_components grid 1 .. d-1 is empty")
    if d > _lib.FEAS_MAX_D:
        raise ValueError(f"LogisticFeasibilityModel: d={d} exceeds the supported {_lib.FEAS_MAX_D} inputs")
    if not 1 <= J <= _lib.FEAS_MAX_J:
        raise ValueError(f"LogisticFeasibilityModel: {J} constraints outside the supported 1 .. {_lib.FEAS_MAX_J}")
    if N is not None and N > _lib.FEAS_MAX_N:
        raise ValueError(f"LogisticFeasibilityModel: {N} training rows exceed the supported {_lib.FEAS_MAX_N}")


class LogisticFeasibilityModel:
    """See the module docstring.  ``hyperparameters`` (a list with one entry per constraint: None for a single-class
    constraint, else (k, C, pca_mean (d,), components (k, d), scaler_mean (k,), scaler_scale (k,), coef (k,),
    intercept)) rebuilds a model bit for bit without fitting; X and C are then ignored."""

    def __init__(self, X, C, fit="gpu", hyperparameters=None, max_iter=100, tol=1e-11):
        t0 = time.time()
        self.fit_info = None
        if hyperparameters is None:
            X = np.ascontiguousarray(X, dtype=np.float64)
            C = np.asarray(C)
            if C.ndim == 1:
                C = C[:, None]
            if X.ndim != 2 or C.ndim != 2 or C.shape[0] != X.shape[0]:
                raise ValueError(f"LogisticFeasibilityModel: X {X.shape} and C {C.shape} do not match")
            _check_shape(X.shape[1], C.shape[1], X.shape[0])
            if fit == "gpu":
                hyperparameters = self._fit_gpu(X, C, max_iter, tol)
            elif fit == "sklearn":
                hyperparameters = self._fit_sklearn(X, C)
            else:
                raise ValueError(f"LogisticFeasibilityModel: fit must be 'gpu' or 'sklearn', got {fit!r}")
        self.hyperparameters = [None if h is None else tuple(h) for h in hyperparameters]
        self._build()
        self.stats = {"feasibility_fit_time": time.time() - t0}

    # ---------------------------------------------------------------- fitting
    def _fit_gpu(self, X, C, max_iter, tol):
        N, d = X.shape
        km = d - 1
        labels = (C > 0.0).astype(np.uint8).T
        two = [j for j in range(labels.shape[0]) if np.unique(labels[j]).size > 1]
        hyper = [None] * labels.shape[0]
        info = {"constraints": two, "C": C_GRID.copy(), "per_constraint": {}}
        if not two:
            self.fit_info = info
            return hyper
        folds = np.stack([stratified_test_folds(labels[j]) for j in two])
        pmean = np.empty((N_SETS * len(two), d))
        pcomp = np.empty((N_SETS * len(two), km, d))
        for a, j in enumerate(two):
            for f in range(N_SETS):
                rows = X if f == N_FOLDS else X[folds[a] != f]
                m, V = pca_components(rows)
                pmean[a * N_SETS + f], pcomp[a * N_SETS + f] = m, V[:km]
        out = _lib.feas_fit(X, labels[two], folds, pmean, pcomp, C_GRID, max_iter=max_iter, tol=tol)
        nC = C_GRID.size
        shape = (len(two), N_SETS, nC, km)
        iters = out["iters"].reshape(shape)
        correct = out["correct"].reshape(shape)
        for a, j in enumerate(two):
            ntest = np.array([np.count_nonzero(folds[a] == f) for f in range(N_FOLDS)], dtype=np.float64)
            frac = correct[a, :N_FOLDS] / ntest[:, None, None]
            frac[iters[a, :N_FOLDS] < 0] = np.nan  # the fold's training rows hold one class
            scores = np.mean(frac, axis=0)  # (nC, km): C outermost, then k (ParameterGrid order)
            flat = scores.ravel()
            best = 0 if np.all(np.isnan(flat)) else int(np.nanargmax(flat))
            ci, k = divmod(best, km)
            k += 1
            p = ((a * N_SETS + N_FOLDS) * nC + ci) * km + (k - 1)
            s = a * N_SETS + N_FOLDS
            coef = out["coef"][p]
            hyper[j] = (k, float(C_GRID[ci]), pmean[s].copy(), pcomp[s, :k].copy(), out["scaler_mean"][s, :k].copy(),
                        out["scaler_scale"][s, :k].copy(), coef[:k].copy(), float(coef[d - 1]))
            fitted = iters[a] >= 0
            conv = out["converged"].reshape(shape)[a].astype(bool)
            info["per_constraint"][j] = {
                "cv_scores": scores, "best": (k, float(C_GRID[ci])), "iters": iters[a], "objective": out["objective"].reshape(shape)[a],
                "kkt": out["kkt"].reshape(shape)[a], "converged": conv, "correct": correct[a],
                "coef": out["coef"].reshape(shape + (d,))[a], "not_converged": int(np.count_nonzero(fitted & ~conv)),
            }
            if np.any(fitted & ~conv):
                logger.warning(f"feasibility model: {np.count_nonzero(fitted & ~conv)} L1-logistic problems of constraint {j} "
                               f"did not reach the KKT tolerance in {max_iter} iterations")
        self.fit_info = info
        return hyper

    def _fit_sklearn(self, X, C):
        from sklearn.decomposition import PCA
        from sklearn.linear_model import LogisticRegression
        from sklearn.model_selection import GridSearchCV, StratifiedKFold
        from sklearn.pipeline import Pipeline
        from sklearn.preprocessing import StandardScaler

        hyper = []
        for j in range(C.shape[1]):
            c = (C[:, j] > 0.0).astype(int)
            if np.unique(c).size < 2:
                hyper.append(None)
                continue
            pipe = Pipeline([("pca", PCA()), ("scaler", StandardScaler()),
                             ("clf", LogisticRegression(tol=0.01, penalty="l1", solver="saga"))])
            grid = {"pca__n_components": range(1, X.shape[1]), "clf__C": C_GRID}
            gs = GridSearchCV(pipe, grid, cv=StratifiedKFold(N_FOLDS), n_jobs=-1).fit(X, c)
            b = gs.best_estimator_
            pca, sc, clf = b.named_steps["pca"], b.named_steps["scaler"], b.named_steps["clf"]
            hyper.append((int(pca.n_components_), float(gs.best_params_["clf__C"]), pca.mean_.copy(), pca.components_.copy(),
                          sc.mean_.copy(), sc.scale_.copy(), clf.coef_[0].copy(), float(clf.intercept_[0])))
        self.fit_info = {"fit": "sklearn"}
        return hyper

    # ---------------------------------------------------------------- device model
    def _build(self):
        hp = self.hyperparameters
        J = len(hp)
        fitted = [h for h in hp if h is not None]
        if not fitted:
            self.d = None
            self._dev = None
            return
        d = int(np.asarray(fitted[0][2]).size)
        _check_shape(d, J)
        km = d - 1
        k = np.zeros(J, dtype=np.int32)
        mean = np.zeros((J, d))
        comps = np.zeros((J, km, d))
        smean = np.zeros((J, km))
        sscale = np.ones((J, km))
        coef = np.zeros((J, km))
        b = np.zeros(J)
        for j, h in enumerate(hp):
            if h is None:
                continue
            kj = int(h[0])
            if not 1 <= kj <= km or np.asarray(h[2]).size != d:
                raise ValueError(f"feasibility model: constraint {j} has k={kj} components of d={np.asarray(h[2]).size} inputs")
            k[j] = kj
            mean[j] = h[2]
            comps[j, :kj] = np.asarray(h[3]).reshape(kj, d)
            smean[j, :kj], sscale[j, :kj], coef[j, :kj] = h[4], h[5], h[6]
            b[j] = h[7]
        self.d = d
        self._dev = _lib.FeasModel(k, mean, comps, smean, sscale, coef, b)

    def _eval(self, x, proba=False, decision=False):
        if self._dev is None:  # every constraint is single-class
            n = np.asarray(x).shape[0] if not hasattr(x, "data_ptr") else int(x.shape[0])
            J = len(self.hyperparameters)
            return np.ones(n), np.ones((J, n)), np.full((J, n), np.inf)
        if isinstance(x, np.ndarray) and _lib.mirror_ptr(x) is None:
            x = np.ascontiguousarray(x, dtype=np.float64)
        elif not isinstance(x, np.ndarray) and not hasattr(x, "data_ptr"):
            x = np.ascontiguousarray(x, dtype=np.float64)
        return self._dev.eval(x, rank=True, proba=proba, decision=decision)

    @property
    def device_model(self):
        """The device-side model (None when every constraint is single-class): the key of the resident NSGA-II update."""
        return self._dev

    # ---------------------------------------------------------------- reference interface
    def rank(self, x):
        """Mean over the constraints of the feasible probability, (n,).  Reads x's device mirror when it has one."""
        return self._eval(x)[0]

    def predict_proba(self, x):
        """(J, n, 2): [infeasible, feasible] probabilities per constraint, as the reference stacks them."""
        p = self._eval(x, proba=True)[1]
        return np.stack((1.0 - p, p), axis=-1)

    def predict(self, x):
        """(n, J) zeros and ones: the decision value is positive (ones for a single-class constraint)."""
        t = self._eval(x, decision=True)[2]
        return (t > 0.0).astype(np.int64).T


def _resolve_feasibility(name):
    if name in (None, "logreg"):
        return LogisticFeasibilityModel
    from dmosopt.config import import_object_by_path

    return import_object_by_path(name)


def train_with_feasibility(optimizer_cls, Xinit, Yinit, C, xlb, xub, file_path, options=None, **kw):
    """``surrogate_custom_training`` for dmosopt's MOASMO.epoch: returns (optimizer_cls, objective, feasibility, None).

    The objective is built by the running dmosopt's own ``MOASMO.train`` (its feasible rows, its duplicate removal).
    The feasibility model is fitted on all of Xinit and C, since it needs both classes; ``feasibility_method_name``
    "logreg" (or None) resolves to this module's model, any other import path is imported.  When the feasibility fit
    fails the error is logged and the feasibility model is None, as dmosopt does."""
    from dmosopt import MOASMO

    options = dict(options or {})
    nInput, nOutput = len(xlb), np.asarray(Yinit).shape[1]
    objective = None
    if options.get("surrogate_method_name") is not None:
        objective = MOASMO.train(
            nInput, nOutput, xlb, xub, Xinit, Yinit, C,
            surrogate_method_name=options["surrogate_method_name"],
            surrogate_method_kwargs=options.get("surrogate_method_kwargs") or {},
            surrogate_return_mean_variance=options.get("return_mean_variance", False),
            logger=kw.get("logger"), file_path=file_path,
        )
    feasibility = None
    if C is not None:
        try:
            cls = _resolve_feasibility(options.get("feasibility_method_name"))
            feasibility = cls(np.asarray(Xinit), np.asarray(C), **(options.get("feasibility_method_kwargs") or {}))
        except Exception as e:
            logger.warning(f"Unable to fit feasibility model: {e!r}")
    return optimizer_cls, objective, feasibility, None
