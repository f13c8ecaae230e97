"""Every L1-logistic solve of the GPU feasibility fit (csrc/feasibility.cu) certified on the host, at the kernels' tile,
block and constraint-batch thresholds.

Each case calls ``_lib.feas_fit`` (directly, or through ``LogisticFeasibilityModel`` with the call recorded) and holds
every (dataset, C, k) problem to the contracts below with oracle/feasibility_exact.py, which recomputes the scores, the
objective F, the gradient, the KKT measure and the held-out count in float64 with bounds derived operation by operation:
  * a problem whose training set holds both classes: the reported kkt and objective are within the bound of the host's,
    converged == (kkt <= tol max(1, C n_train)) on the reported values, 0 <= iters <= max_iter, coef[k:d-1] == 0, the
    held-out count lies in the host interval (one value on all but a stated number of rows), and fold 5 counts 0;
  * a problem whose training set is one class: iters -1, objective and kkt NaN, converged 0, correct -1, coef 0;
  * every dataset: the scaler is within its bounds of the host's mean and std of the scores over the training rows.
The thresholds each case straddles are named with the lines of csrc/feasibility.cu that set them.
"""

import numpy as np
import pytest

from dmosopt_b200.feasibility import C_GRID, N_SETS, pca_components, stratified_test_folds
from oracle import feasibility as of
from oracle import feasibility_exact as fx

pytestmark = pytest.mark.gpu

TOL = 1e-11
N_FOLDS = N_SETS - 1
ORACLE_K = (1, 32, 33, 64, 65, 87, 88)  # with d - 1: KP and nb steps, lanes past 32 / 64, the second block at k >= 88


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


# ---------------------------------------------------------------------------------------------- data
def noisy(rng, N, d, J=2, noise=0.1):
    """(X, labels (J, N)): linear constraints with unbalanced classes and ``noise`` of the labels flipped."""
    X = rng.random((N, d)) * np.linspace(1.0, 3.0, d)
    lab = []
    for j in range(J):
        a = X @ rng.standard_normal(d)
        lab.append(a > np.quantile(a, 0.35 + 0.25 * (j % 2)))
    lab = np.array(lab) ^ (rng.random((J, N)) < noise)
    return X, lab.astype(np.uint8)


def prepare(X, labels, folds=None):
    """Folds (stratified, or as given) and the PCA of every dataset, as LogisticFeasibilityModel forms them."""
    J, N = labels.shape
    d = X.shape[1]
    if folds is None:
        folds = np.stack([stratified_test_folds(labels[j]) for j in range(J)])
    pmean = np.empty((N_SETS * J, d))
    pcomp = np.empty((N_SETS * J, d - 1, d))
    for j in range(J):
        for f in range(N_SETS):
            m, V = pca_components(X if f == N_FOLDS else X[folds[j] != f])
            pmean[j * N_SETS + f], pcomp[j * N_SETS + f] = m, V[: d - 1]
    return np.ascontiguousarray(folds, dtype=np.int8), pmean, pcomp


def fit(L, X, labels, Cs=C_GRID, folds=None, max_iter=100, tol=TOL, prep=None):
    folds, pmean, pcomp = prep if prep is not None else prepare(X, labels, folds)
    out = L.feas_fit(X, labels, folds, pmean, pcomp, Cs, max_iter=max_iter, tol=tol)
    return dict(X=X, labels=labels, folds=folds, pmean=pmean, pcomp=pcomp, Cs=np.asarray(Cs, dtype=np.float64),
                max_iter=max_iter, tol=tol, out=out)


# ---------------------------------------------------------------------------------------------- the certificate
def certify(name, run, amb_max=0, oracle_sets=()):
    """Hold every problem of ``run`` to the contracts of the module docstring.  ``oracle_sets`` lists (j, f) datasets
    whose problems at k in ORACLE_K + (d - 1) are also solved by oracle.l1_logistic on the host scores: a converged
    problem's objective must be <= the oracle's (1 + 1e-9).  Returns the per-problem host certificates and prints the
    case's counts."""
    X, labels, folds, out = run["X"], run["labels"], run["folds"], run["out"]
    Cs, max_iter, tol = run["Cs"], run["max_iter"], run["tol"]
    J, N = labels.shape
    d = X.shape[1]
    km, nC = d - 1, Cs.size
    ks = np.arange(1, d)
    stats = dict(problems=0, one_class=0, certified=0, not_converged=0, early_exit=0, ambiguous=0, max_iters=0)
    certs = {}
    for j in range(J):
        y = labels[j]
        for f in range(N_SETS):
            s = j * N_SETS + f
            train = np.ones(N, dtype=bool) if f == N_FOLDS else folds[j] != f
            test = None if f == N_FOLDS else folds[j] == f
            sc = fx.Scores(X, run["pmean"][s], run["pcomp"][s], out["scaler_mean"][s], out["scaler_scale"][s])
            ok = fx.scaler_agrees(out["scaler_mean"][s], out["scaler_scale"][s], sc.U[train], sc.bU[train])
            assert ok.all(), (name, j, f, "scaler", np.flatnonzero(~ok))
            npos = int(np.count_nonzero(y[train]))
            for ci, C in enumerate(Cs):
                idx = (s * nC + ci) * km + ks - 1
                coef, iters, obj = out["coef"][idx], out["iters"][idx], out["objective"][idx]
                kkt, conv, cor = out["kkt"][idx], out["converged"][idx], out["correct"][idx]
                stats["problems"] += km
                if npos == 0 or npos == np.count_nonzero(train):
                    assert (np.all(iters == -1) and np.all(np.isnan(obj)) and np.all(np.isnan(kkt)) and np.all(conv == 0)
                            and np.all(cor == -1) and np.all(coef == 0.0)), (name, j, f, ci, "one-class training set")
                    stats["one_class"] += km
                    continue
                for k in ks:
                    assert np.all(coef[k - 1, k:d - 1] == 0.0), (name, j, f, ci, k, "coefficients past k")
                cert = fx.Certificate(sc, y, train, test, C, ks, coef)
                certs[(j, f, ci)] = cert
                where = (name, j, f, float(C))
                bad = np.flatnonzero(~(np.abs(kkt - cert.kkt) <= 2.0 * cert.bk))
                assert bad.size == 0, (*where, "kkt", ks[bad][:5], kkt[bad][:5], cert.kkt[bad][:5], cert.bk[bad][:5])
                bad = np.flatnonzero(~(np.abs(obj - cert.F) <= 2.0 * cert.bF))
                assert bad.size == 0, (*where, "objective", ks[bad][:5], obj[bad][:5], cert.F[bad][:5], cert.bF[bad][:5])
                gtol = cert.gtol_of(tol)
                assert np.array_equal(conv.astype(bool), kkt <= gtol), (*where, "converged flag")
                assert np.all((iters >= 0) & (iters <= max_iter)), (*where, "iters", iters)
                c = conv.astype(bool)
                assert np.all(cert.kkt[c] <= gtol + 2.0 * cert.bk[c]), (*where, "certified optimum")
                if f == N_FOLDS:
                    assert np.all(cor == 0), (*where, "fold 5 has no held-out rows")
                else:
                    bad = np.flatnonzero(~((cert.lo <= cor) & (cor <= cert.lo + cert.amb)))
                    assert bad.size == 0, (*where, "held-out count", ks[bad][:5], cor[bad][:5], cert.lo[bad][:5], cert.amb[bad][:5])
                    stats["ambiguous"] += int(np.sum(cert.amb))
                stats["certified"] += int(np.count_nonzero(c))
                stats["not_converged"] += int(np.count_nonzero(~c))
                stats["early_exit"] += int(np.count_nonzero(~c & (iters < max_iter)))
                stats["max_iters"] = max(stats["max_iters"], int(iters.max()))
                if (j, f) in oracle_sets:
                    for k in sorted({k for k in ORACLE_K if k < d} | {km}):
                        if not c[k - 1]:
                            continue
                        _, _, F = of.l1_logistic(sc.Z[train, :k], y[train], C)
                        assert obj[k - 1] <= F * (1 + 1e-9), (*where, k, "above the oracle", obj[k - 1], F)
    assert stats["ambiguous"] <= amb_max, (name, stats)
    print(f"[feasibility exact] {name}: {stats}")
    run["stats"] = stats
    return certs


def problem_index(run, j, f, ci, k):
    km = run["X"].shape[1] - 1
    return ((j * N_SETS + f) * run["Cs"].size + ci) * km + k - 1


# ---------------------------------------------------------------------------------------------- dimensions
# d 2: km = 1 (one problem per (dataset, C)); d 3: the odd shared-memory stride d | 1 of feas_scores_kernel (:61);
# d 32 / 33: the solve's shared layout R0 = max(KPmax^2, 32 KPmax) switches operand (:153-154); d 89 / 90: k >= 88 takes
# the second 4 x 4 block per thread (FS_MAXBLK, :33, :187-203), and every k crosses KP, nb, and feas_margin's lanes past
# 32 and 64 columns (:126-130).
@pytest.mark.parametrize("d", [2, 3, 32, 33, 89, 90])
def test_fit_across_dimensions(L, monkeypatch, d):
    from dmosopt_b200 import feasibility as feas

    X, lab = noisy(np.random.default_rng(100 + d), 1000, d)
    calls = []
    real = L.feas_fit

    def spy(*a, **kw):
        out = real(*a, **kw)
        calls.append((a, kw, out))
        return out

    monkeypatch.setattr(L, "feas_fit", spy)
    m = feas.LogisticFeasibilityModel(X, np.where(lab.T > 0, 1.0, -1.0))
    (a, kw, out), = calls
    run = dict(X=X, labels=a[1], folds=a[2], pmean=a[3], pcomp=a[4], Cs=np.asarray(a[5]), max_iter=kw["max_iter"],
               tol=kw["tol"], out=out)
    assert np.array_equal(run["labels"], lab)
    certs = certify(f"d {d}", run, amb_max=4, oracle_sets={(0, N_FOLDS), (0, 0)})
    assert run["stats"]["not_converged"] == 0, "at N 1000 every problem of the grid converges (in at most 7 steps)"
    # the model's pick: the first nanargmax of the mean held-out accuracy, recomputed from the certified counts
    km = d - 1
    for j in range(2):
        acc = np.full((C_GRID.size, km, N_FOLDS), np.nan)
        for f in range(N_FOLDS):
            for ci in range(C_GRID.size):
                cert = certs[(j, f, ci)]
                assert np.all(cert.amb == 0), "the pick is only checked where every count is certified"
                acc[ci, :, f] = cert.lo / cert.ntest
        best = int(np.nanargmax(acc.mean(axis=2).ravel()))
        ci, k = best // km, best % km + 1
        hp = m.hyperparameters[j]
        assert hp[:2] == (k, float(C_GRID[ci])), (j, hp[:2], (k, C_GRID[ci]))
        p = problem_index(run, j, N_FOLDS, ci, k)
        s = j * N_SETS + N_FOLDS
        assert np.array_equal(hp[6], out["coef"][p, :k]) and hp[7] == out["coef"][p, d - 1]
        assert np.array_equal(hp[4], out["scaler_mean"][s, :k]) and np.array_equal(hp[5], out["scaler_scale"][s, :k])
        assert np.array_equal(hp[2], run["pmean"][s]) and np.array_equal(hp[3], run["pcomp"][s, :k])


# ---------------------------------------------------------------------------------------------- rows
# N 5: one held-out row per fold; 32 = FS_ROWS, the Gram tile (:32, :215-216); 128 = ROW_TILE, the score kernels' rows
# (:34, :62-63); 256 = FS_THREADS, the thread stride of the scaler (:91) and of the class count (:169).
@pytest.mark.parametrize("d", [3, 34])
@pytest.mark.parametrize("N", [5, 31, 32, 33, 127, 128, 129, 255, 256, 257])
def test_fit_across_rows(L, N, d):
    rng = np.random.default_rng(1000 * d + N)
    X = rng.random((N, d)) * np.linspace(1.0, 3.0, d)
    a = X @ rng.standard_normal(d)
    # unbalanced classes: no training set splits evenly, so no intercept-only optimum sits at t = 0
    lab = np.stack([a > np.quantile(a, 0.4), X[:, 0] - X[:, -1] > np.quantile(X[:, 0] - X[:, -1], 0.7)]).astype(np.uint8)
    if N == 5:
        lab = np.array([[1, 0, 1, 0, 1], [0, 1, 1, 0, 1]], dtype=np.uint8)  # every 4-row training set keeps both classes
        folds = np.tile(np.arange(5, dtype=np.int8), (2, 1))
    else:
        folds = None
    run = fit(L, X, lab, folds=folds)
    # Up to N = 2 d the undecided held-out rows are counted, not limited: with fewer training rows than components the
    # trailing components are rounding noise that the scaler stretches to unit scale, so their scores carry bounds of
    # order one; and a training set split evenly (N 5: 2 + 2 rows) has the intercept-only optimum t = 0 at small C.
    certify(f"N {N} d {d}", run, amb_max=0 if N > 2 * d else 10**9)
    if N == 5:
        assert all(np.count_nonzero(run["folds"][0] == f) == 1 for f in range(N_FOLDS))


# ---------------------------------------------------------------------------------------------- the envelope
def test_fit_at_the_row_limit_d30(L):
    """N = FEAS_MAX_N = 65536 (:27) at d 30 over the reference grid."""
    X, lab = noisy(np.random.default_rng(7), 65536, 30)
    certify("N 65536 d 30", fit(L, X, lab), amb_max=200)


def test_fit_at_the_envelope_corner_d90(L):
    """N 65536, d 90, one constraint, one C, five Newton steps: the reported objective and KKT measure describe the
    returned w, converged or not."""
    X, lab = noisy(np.random.default_rng(8), 65536, 90, J=1)
    certify("N 65536 d 90 max_iter 5", fit(L, X, lab, Cs=[1.0], max_iter=5), amb_max=200)


def test_constraint_batches_equal_single_fits(L):
    """dmo_feas_fit splits the constraints into batches of jb = 2^31 / (48 N (d - 1)) (:490-491): 23 at N 65536, d 30,
    so J 32 runs a batch of 23 and a batch of 9 that reuses Z, with the output offset p0 (:501).  A problem reads only
    its own dataset and every sum runs in a fixed order, so constraints 0, 22 (the first batch's last), 23 (the second
    batch's first) and 31 must equal the same constraint fitted alone, bit for bit."""
    N, d, J = 65536, 30, 32
    assert (2**31) // (6 * N * (d - 1) * 8) == 23
    rng = np.random.default_rng(9)
    X = rng.random((N, d)) * np.linspace(1.0, 3.0, d)
    lab = []
    for j in range(J):
        a = X @ rng.standard_normal(d)
        lab.append(a > np.quantile(a, 0.2 + 0.6 * rng.random()))
    lab = (np.array(lab) ^ (rng.random((J, N)) < 0.1)).astype(np.uint8)
    prep = prepare(X, lab)
    run = fit(L, X, lab, Cs=[1.0], max_iter=3, prep=prep)
    certify("batches N 65536 d 30 J 32", run, amb_max=J * 200)
    out = run["out"]
    per = N_SETS * (d - 1)
    for j in (0, 22, 23, 31):
        one = fit(L, X, lab[j:j + 1], Cs=[1.0], max_iter=3,
                  prep=(prep[0][j:j + 1], prep[1][j * N_SETS:(j + 1) * N_SETS], prep[2][j * N_SETS:(j + 1) * N_SETS]))["out"]
        for key in ("scaler_mean", "scaler_scale"):
            assert np.array_equal(out[key][j * N_SETS:(j + 1) * N_SETS], one[key]), (j, key)
        for key in ("coef", "iters", "objective", "kkt", "converged", "correct"):
            assert np.array_equal(out[key][j * per:(j + 1) * per], one[key], equal_nan=True), (j, key)


# ---------------------------------------------------------------------------------------------- C, max_iter, tol
C16 = np.sort(np.concatenate((C_GRID, [1e-6, 1e-5, 1e-3, 1e-2, 0.1, 1.0, 10.0, 100.0, 1e3, 1e5, 1e6, 3.0])))


def test_sixteen_values_of_C(L):
    """FEAS_MAX_C = 16 values (:28) from 1e-6 to 1e6 holding the reference's four: the problems at those four equal a
    four-value call bit for bit (the decomposition p -> (s, ci, k) of :146 at nC 16 and 4)."""
    assert C16.size == 16 and np.all(np.isin(C_GRID, C16))
    X, lab = noisy(np.random.default_rng(11), 300, 6)
    prep = prepare(X, lab)
    r16 = fit(L, X, lab, Cs=C16, prep=prep)
    certify("16 C", r16, amb_max=4)
    r4 = fit(L, X, lab, Cs=C_GRID, prep=prep)
    km = X.shape[1] - 1
    for key in ("coef", "iters", "objective", "kkt", "converged", "correct"):
        a = r16["out"][key].reshape(2 * N_SETS, 16, km, -1)[:, np.searchsorted(C16, C_GRID)]
        assert np.array_equal(a, r4["out"][key].reshape(2 * N_SETS, 4, km, -1), equal_nan=True), key


def test_max_iter_zero_and_tol_zero(L):
    X, lab = noisy(np.random.default_rng(12), 300, 6)
    prep = prepare(X, lab)
    z = fit(L, X, lab, Cs=C16, max_iter=0, prep=prep)
    assert np.all(z["out"]["coef"] == 0.0) and np.all(z["out"]["iters"] == 0)
    certify("max_iter 0", z, amb_max=10**9)  # w = 0: every margin is 0, so every held-out row is undecided
    t = fit(L, X, lab, Cs=C_GRID, tol=0.0, prep=prep)
    certify("tol 0", t, amb_max=4)  # converged == (kkt <= 0)
    assert np.array_equal(t["out"]["converged"].astype(bool), t["out"]["kkt"] == 0.0)


def test_separable_labels_at_large_C(L):
    """At C 1e4 and 1e6 on separable labels the optimum runs off to |w| -> inf: Newton stops on the line search
    (:360) or on a subproblem without descent (:334) before the KKT tolerance.  The reported F and KKT measure must
    still describe the returned w, and the flag must say it did not converge."""
    rng = np.random.default_rng(13)
    X = rng.random((400, 5))
    lab = np.stack([X[:, 0] + X[:, 1] > 1.0, X[:, 2] > 0.5]).astype(np.uint8)
    run = fit(L, X, lab, Cs=[1.0, 1e4, 1e6], max_iter=100)
    certify("separable C 1 1e4 1e6", run, amb_max=20)
    it = run["out"]["iters"].reshape(2, N_SETS, 3, 4)
    cv = run["out"]["converged"].reshape(2, N_SETS, 3, 4)
    print(f"[feasibility exact] separable C 1e6: iters {np.unique(it[:, :, 2])}, converged {int(cv[:, :, 2].sum())} of {cv[:, :, 2].size}")


# ---------------------------------------------------------------------------------------------- labels and inputs
@pytest.mark.parametrize("kind", ["single_member_minority", "constant_column", "duplicate_rows", "separable"])
def test_label_and_input_edges(L, kind):
    rng = np.random.default_rng(14)
    N, d = 203, 5
    X = rng.random((N, d)) * np.linspace(1.0, 3.0, d)
    a = X @ rng.standard_normal(d)
    lab = np.stack([a > np.quantile(a, 0.4), X[:, 1] > np.quantile(X[:, 1], 0.7)])
    lab = lab ^ (rng.random(lab.shape) < 0.1)
    if kind == "single_member_minority":
        lab[1] = False
        lab[1, 40] = True  # the fold holding row 40 trains on one class
    elif kind == "constant_column":
        X[:, 2] = 0.25
    elif kind == "duplicate_rows":
        X[100:] = X[:103]
        lab[:, 100:] = lab[:, :103]
    elif kind == "separable":
        lab = np.stack([a > np.quantile(a, 0.4), X[:, 1] > np.quantile(X[:, 1], 0.7)])
    lab = lab.astype(np.uint8)
    run = fit(L, X, lab)
    certify(kind, run, amb_max=4)
    if kind == "single_member_minority":
        p = problem_index(run, 1, int(run["folds"][1, 40]), 0, 1)
        assert run["out"]["iters"][p] == -1 and run["out"]["correct"][p] == -1


# ---------------------------------------------------------------------------------------------- the evaluation kernel
def eval_model(rng, d, J):
    """Random fitted-model parameters (k mixes 0, 1 and d - 1) and their FeasModel."""
    km = d - 1
    ks = np.array([(d - 1, 1, 0)[j % 3] for j in range(J)], dtype=np.int32)
    mean = rng.random((J, d)) * 2.0
    comps = np.stack([np.linalg.qr(rng.standard_normal((d, d)))[0][:, :km].T for _ in range(J)])
    smean = rng.standard_normal((J, km)) * 0.1
    sscale = rng.random((J, km)) + 0.2
    coef = rng.standard_normal((J, km)) * np.logspace(-2, 1, km)
    b = rng.standard_normal(J)
    for j in range(J):
        coef[j, ks[j]:] = 0.0
    return ks, (mean, comps, smean, sscale, coef, b)


def eval_host(ks, par, X, rows):
    """(t, bt) of every constraint on X[rows], with the bound of oracle/feasibility_exact.py's margin."""
    mean, comps, smean, sscale, coef, b = par
    J = len(ks)
    t = np.full((J, rows.size), np.inf)
    bt = np.zeros((J, rows.size))
    for j, k in enumerate(ks):
        if k == 0:
            continue
        sc = fx.Scores(X[rows], mean[j], comps[j, :k], smean[j, :k], sscale[j, :k])
        w = coef[j, :k]
        t[j] = sc.Z @ w + b[j]
        bt[j] = (sc.bz @ np.abs(w) + fx.gamma(k + 1) * (np.abs(sc.Z) @ np.abs(w) + abs(b[j]))) * fx.SAFE
    return t, bt


# n 1 / 127 / 128 / 129 / 2^17 + 1 cross ROW_TILE (:393-394); d 2 / 3 / 89 / 90 the stride d | 1 (:392) and 93 KB of
# shared rows at d 90.
@pytest.mark.parametrize("d", [2, 3, 89, 90])
@pytest.mark.parametrize("J", [1, 32])
def test_eval_against_the_host(L, d, J):
    rng = np.random.default_rng(d * 100 + J)
    ks, par = eval_model(rng, d, J)
    if J == 1:
        ks[0] = d - 1
        par[4][0] = rng.standard_normal(d - 1)
    m = L.FeasModel(ks, *par)
    for n in (1, 127, 128, 129, 2**17 + 1):
        X = rng.random((n, d)) * 3.0 - 0.5
        r, P, T = m.eval(X, rank=True, proba=True, decision=True)
        zero = ks == 0
        assert np.all(T[zero] == np.inf) and np.all(P[zero] == 1.0)
        acc = np.zeros(n)
        for j in range(J):
            acc += P[j]
        assert np.array_equal(r, acc / J), "rank is the left-to-right sum of the probabilities over j, / J"
        # every row up to 1025, else the first two tiles, the last two and 2000 sampled rows
        rows = np.arange(n) if n <= 1025 else np.unique(np.concatenate(
            (np.arange(256), np.arange(n - 129, n), rng.integers(0, n, 2000))))
        t, bt = eval_host(ks, par, X, rows)
        live = ~zero
        assert np.all(np.abs(T[live][:, rows] - t[live]) <= 2.0 * bt[live]), (n, "decision")
        p = 1.0 / (1.0 + np.exp(-t[live]))
        assert np.all(np.abs(P[live][:, rows] - p) <= 2.0 * bt[live] / 4.0 + 8 * fx.UR * p), (n, "probability")
        if n == 129:
            Xm, _ = L.mirrored_readonly(X)
            assert L.mirror_ptr(Xm) is not None
            rm, Pm, Tm = m.eval(Xm, rank=True, proba=True, decision=True)
            assert np.array_equal(rm, r) and np.array_equal(Pm, P) and np.array_equal(Tm, T)
    c0 = L.launch_count()
    r0, P0, T0 = m.eval(np.empty((0, d)), rank=True, proba=True, decision=True)
    assert L.launch_count() == c0 and r0.shape == (0,) and P0.shape == (J, 0)
