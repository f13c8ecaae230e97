"""Host certificate of the GPU feasibility fit (csrc/feasibility.cu): every quantity a solve reports, recomputed in
float64 from the same inputs, with a rounding bound derived operation by operation.

Notation: u = 2^-53 is the unit roundoff, gamma(n) = n u / (1 - n u) bounds the rounding of any n-term sum or dot
product (any order, with or without FMA).  Every ``b*`` below is one-sided: it bounds the distance between an evaluation
that follows the standard model (the kernel's or this module's) and the exact real value of the same formula on the
same double inputs.  The GPU and the host value are therefore within twice the bound of each other.

  scores      D = x - mean                        |D - D*| <= u |D|
              U = sum_l V_cl D_l   (d terms)      bU = gamma(d + 1) A,  A = |D| |V|^T
              v = U - smean                       bv = bU + u |v|
              z = v / sscale                      bz = bv / sscale + u |z|
  margin      t = sum_{c<k} z_c w_c + b           bt = sum |w_c| bz_c + gamma(k + 1) (sum |z_c w_c| + |b|)
  loss        l = log(1 + exp(-s t))              1-Lipschitz in t; exp and log1p within 1 ulp each (CUDA's and
                                                  glibc's), so the evaluation adds 5 u l
              F = C sum_train l + |w|_1           bF = C (sum bt + (5 u + gamma(n)) sum l) + u C L + gamma(k) |w|_1
                                                       + u |F|
  gradient    p = 1 / (1 + exp(-t))               1/4-Lipschitz in t, evaluation 4 u p
              r = C (p - y)                       br = C (bt / 4 + 4 u p) + 2 u |r|
              g_c = sum_train r z_c               bg_c = sum |z_c| br + sum |r| bz_c + gamma(n) sum |r z_c|
  KKT         max(|g_b|, |g_c + sign w_c| (w_c != 0), max(0, |g_c| - 1) (w_c = 0)): each piece is 1-Lipschitz in g
              and its +-1 rounds once:            bk = max(bg_b, max_c bg_c + u (|g_c| + 1))
  scaler      m = sum U / n                       bm = (sum bU + gamma(n) sum |U|) / n + u |m|
              e = U - m, var = sum e^2 / n        be = bU + bm + u |e|,
                                                  bvar = (sum 2 |e| be + be^2 + gamma(n + 1) sum e^2) / n + u var
              sd = sqrt(var)                      bsd = min(bvar / sd, sqrt(bvar)) + u sd

Terms of second order in u (a product of two roundoffs, at most (90 + 65536)^2 u^2 relative) are covered by the factor
``SAFE`` = 1 + 2^-20 on every bound.  The held-out count of a problem is an interval: a row whose host margin is within
2 bt of zero may fall on either side on the GPU.
"""

import numpy as np

UR = 2.0**-53
EPS = np.finfo(np.float64).eps
SAFE = 1.0 + 2.0**-20


def gamma(n):
    n = np.asarray(n, dtype=np.float64)
    return n * UR / (1.0 - n * UR)


class Scores:
    """Host replay of one dataset's standardised scores: ``Z`` (N, d-1) from X, the dataset's PCA ``mean`` (d,) and
    ``comps`` (d-1, d), and the scaler ``smean`` / ``sscale`` (d-1,) the kernel returned; ``bz`` is Z's bound, ``U`` /
    ``bU`` the unstandardised scores and theirs (for the scaler check)."""

    def __init__(self, X, mean, comps, smean, sscale):
        X, mean, comps = (np.asarray(a, dtype=np.float64) for a in (X, mean, comps))
        d = X.shape[1]
        D = X - mean
        self.U = D @ comps.T
        self.bU = gamma(d + 1) * (np.abs(D) @ np.abs(comps).T) * SAFE
        v = self.U - smean
        self.Z = v / sscale
        self.bz = ((self.bU + UR * np.abs(v)) / sscale + UR * np.abs(self.Z)) * SAFE


def scaler(U, bU):
    """(m, bm, var, bvar, sd, bsd) of the score columns U (n, c) over the rows given: feas_scaler_kernel's mean and
    population variance about that mean, each with its bound."""
    n = U.shape[0]
    m = np.sum(U, axis=0) / n
    bm = ((np.sum(bU, axis=0) + gamma(n) * np.sum(np.abs(U), axis=0)) / n + UR * np.abs(m)) * SAFE
    e = U - m
    be = bU + bm + UR * np.abs(e)
    var = np.sum(e * e, axis=0) / n
    bvar = ((np.sum(2.0 * np.abs(e) * be + be * be, axis=0) + gamma(n + 1) * np.sum(e * e, axis=0)) / n + UR * var) * SAFE
    sd = np.sqrt(var)
    with np.errstate(divide="ignore", invalid="ignore"):
        lin = np.where(var > 0.0, bvar / sd, np.inf)
    bsd = (np.minimum(lin, np.sqrt(bvar)) + UR * sd) * SAFE
    return m, bm, var, bvar, sd, bsd


def scaler_agrees(smean, sscale, U, bU):
    """Per column, whether the kernel's (smean, sscale) is one the scaler rule allows: the mean within 2 bm of the host
    mean; the scale within 2 bsd of the host std, or exactly 1 where the column may be constant to rounding
    (var <= n eps var + (n m eps)^2, oracle.feasibility.scaler) or its variance may be 0."""
    n = U.shape[0]
    m, bm, var, bvar, sd, bsd = scaler(U, bU)
    ok_m = np.abs(smean - m) <= 2.0 * bm
    lo_v = np.maximum(var - 2.0 * bvar, 0.0)
    hi_v = var + 2.0 * bvar
    hi_m = np.abs(m) + 2.0 * bm
    lo_m = np.maximum(np.abs(m) - 2.0 * bm, 0.0)
    may_const = (lo_v * (1.0 - n * EPS) <= (n * hi_m * EPS) ** 2 * (1.0 + 8 * UR)) | (lo_v == 0.0)
    may_vary = hi_v * (1.0 - n * EPS) > (n * lo_m * EPS) ** 2 * (1.0 - 8 * UR)
    near = np.abs(sscale - sd) <= 2.0 * bsd
    ok_s = np.where(sscale == 1.0, may_const | near, may_vary & near)
    return ok_m & ok_s


class Certificate:
    """Host KKT measure, objective and held-out count of the problems (C, k_j) with coefficient rows ``coef`` (nk, d)
    (w = coef[:k], intercept coef[d - 1]) on one dataset: ``sc`` (Scores), labels ``y`` (N,) in {0, 1}, training mask
    ``train`` and held-out mask ``test`` (None for all rows).  Arrays are per problem:
      F, bF        objective and its bound
      g            (list) the gradient [g_w (k,), g_b]
      kkt, bk      KKT measure and its bound
      lo, amb      held-out rows surely correct, and rows whose side is not decided by the bound ([lo, lo + amb])"""

    def __init__(self, sc, y, train, test, C, ks, coef):
        ks = np.asarray(ks, dtype=np.int64)
        coef = np.asarray(coef, dtype=np.float64)
        d = coef.shape[1]
        km = d - 1
        nk = len(ks)
        W = np.zeros((km, nk))
        for j, k in enumerate(ks):
            W[:k, j] = coef[j, :k]
        b = coef[:, d - 1]
        y = np.asarray(y).astype(np.float64)
        Z, bz = sc.Z, sc.bz
        Zt, bzt, yt = Z[train], bz[train], y[train]
        n = Zt.shape[0]
        self.ntr = float(n)
        self.C = float(C)
        aW = np.abs(W)
        l1 = np.sum(aW, axis=0)

        def margins(Zr, bzr):
            T = Zr @ W + b
            S = np.abs(Zr) @ aW + np.abs(b)
            return T, (bzr @ aW + gamma(ks + 1) * S) * SAFE

        T, bt = margins(Zt, bzt)
        s = np.where(yt[:, None] > 0, T, -T)
        with np.errstate(over="ignore"):
            ell = np.logaddexp(0.0, -s)
            p = 1.0 / (1.0 + np.exp(-T))
        L = np.sum(ell, axis=0)
        self.F = C * L + l1
        self.bF = (C * (np.sum(bt, axis=0) + (5 * UR + gamma(n)) * L) + UR * C * L + gamma(ks) * l1
                   + UR * np.abs(self.F)) * SAFE
        r = C * (p - yt[:, None])
        ar = np.abs(r)
        br = C * (bt / 4.0 + 4 * UR * p) + 2 * UR * ar
        aZ = np.abs(Zt)
        G = Zt.T @ r
        BG = (aZ.T @ br + bzt.T @ ar + gamma(n) * (aZ.T @ ar)) * SAFE
        gb = np.sum(r, axis=0)
        bgb = (np.sum(br, axis=0) + gamma(n) * np.sum(ar, axis=0)) * SAFE
        self.g, self.kkt, self.bk = [], np.empty(nk), np.empty(nk)
        for j, k in enumerate(ks):
            g, bg, w = G[:k, j], BG[:k, j], W[:k, j]
            e = np.where(w != 0.0, np.abs(g + np.sign(w)), np.maximum(0.0, np.abs(g) - 1.0))
            self.kkt[j] = max(abs(gb[j]), np.max(e, initial=0.0))
            self.bk[j] = max(bgb[j], np.max(bg + UR * (np.abs(g) + 1.0), initial=0.0)) * SAFE
            self.g.append((g, gb[j]))
        self.lo = np.zeros(nk, dtype=np.int64)
        self.amb = np.zeros(nk, dtype=np.int64)
        self.ntest = 0
        if test is not None and np.any(test):
            Th, bth = margins(Z[test], bz[test])
            yh = y[test][:, None] > 0
            sure = np.abs(Th) > 2.0 * bth
            self.lo = np.count_nonzero(sure & ((Th > 0.0) == yh), axis=0)
            self.amb = np.count_nonzero(~sure, axis=0)
            self.ntest = int(np.count_nonzero(test))

    def tol_scale(self):
        """max(1, C n_train) as the kernel forms it."""
        return np.fmax(1.0, np.float64(self.C) * np.float64(self.ntr))

    def gtol_of(self, tol):
        return np.float64(tol) * self.tol_scale()

    def accepts(self, tol):
        """Problems whose exact KKT measure is certified <= tol max(1, C n_train) (a certified optimum)."""
        return self.kkt + self.bk <= self.gtol_of(tol)

    def rejects(self, tol):
        """Problems whose exact KKT measure is certified above tol max(1, C n_train)."""
        return self.kkt - self.bk > self.gtol_of(tol)
