"""Oracle: exact hypervolume and EHVI candidate selection (rows A16/A17 of SURVEY.md section 8a).

Test infrastructure only (see oracle/__init__.py).

Reference:
  * ``dmosopt/hv.py:123-189``  AdaptiveHyperVolume.compute_hypervolume(..., 'box'):
    keeps only points strictly inside ``ref`` (:159-162) then calls the box algorithm.
  * ``dmosopt/hv_box_decomposition.py:86-304``  HyperVolumeBoxDecomposition.compute_hypervolume
    (Lacour-Klamroth-Fonseca local-upper-bound decomposition).
  * ``dmosopt/hv_box_decomposition.py:306-437``  select_candidates / _compute_batch_ehvi /
    _decompose_dominated_space (the "HV contribution" selection used by CMAES / TRS through
    ``indicators.HypervolumeImprovement._do``, indicators.py:295-313).

``hypervolume`` below is the *true* hypervolume (minimisation), computed by
dimension sweep -- an independent algorithm, not a transliteration of the box
decomposition.  It equals the reference for every input whose first M-1
objectives are strictly positive; the reference silently loses volume
otherwise because its dummy defining points sit at 0 (hv_box_decomposition.py
:136-145, :228; SURVEY.md section 8a row A16) -- golden fixtures therefore use
positive objectives, and the divergence case is pinned as a documented
difference in tests/test_oracle_golden.py.
"""

import numpy as np
from scipy.stats import norm


def inside_ref(points, ref):
    """hv.py:159-162: keep points with ref > p in every objective."""
    points = np.asarray(points, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    return points[np.all(ref > points, axis=1)]


def _nondominated(P):
    """Drop weakly dominated points and exact duplicates (does not change the HV)."""
    n = P.shape[0]
    if n <= 1:
        return P
    P = np.unique(P, axis=0)
    le = (P[:, None, :] <= P[None, :, :]).all(axis=2)
    np.fill_diagonal(le, False)
    return P[~le.any(axis=0)]


def _hv2d(P, ref):
    """Staircase sweep: sort by f0, accumulate strips under the running min of f1."""
    o = np.argsort(P[:, 0], kind="stable")
    x = P[o, 0]
    y = P[o, 1]
    ymin = np.minimum.accumulate(y)
    xn = np.append(x[1:], ref[0])
    return float(np.sum((xn - x) * (ref[1] - ymin)))


def _hv_rec(P, ref):
    d = P.shape[1]
    if P.shape[0] == 0:
        return 0.0
    if d == 1:
        return float(ref[0] - P[:, 0].min())
    if d == 2:
        return _hv2d(P, ref)
    # slice along the last objective
    o = np.argsort(P[:, -1], kind="stable")
    P = P[o]
    z = P[:, -1]
    zn = np.append(z[1:], ref[-1])
    total = 0.0
    for i in range(P.shape[0]):
        h = zn[i] - z[i]
        if h > 0.0:
            total += h * _hv_rec(_nondominated(P[: i + 1, :-1]), ref[:-1])
    return total


def hypervolume(points, ref):
    """True hypervolume dominated by ``points`` and bounded by ``ref`` (minimisation)."""
    ref = np.asarray(ref, dtype=np.float64)
    P = inside_ref(points, ref)
    if P.shape[0] == 0:
        return 0.0
    return _hv_rec(_nondominated(P), ref)


# ---------------------------------------------------------------------------
# EHVI candidate selection (hv_box_decomposition.py:306-437)
# ---------------------------------------------------------------------------


def decompose_boxes(front, ref):
    """hv_box_decomposition.py:418-437: boxes between consecutive f0-sorted front points.

    lower = (-inf, front sorted by f0), upper = (front sorted by f0, ref); only boxes
    with upper > lower in *every* objective are kept.  (For a mutually
    non-dominated front this leaves the two end boxes -- the reference's
    heuristic box set, reproduced as is.)

    Points with equal f0 stay in front-row order (a stable sort), as on the GPU.  The
    reference sorts with numpy's default unstable ``argsort``, whose order among equal
    f0 depends on the machine (its AVX-512 sort differs from the scalar one); the
    boxes, and so the scores, depend on that order.
    """
    front = np.asarray(front, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    n, d = front.shape
    o = np.argsort(front[:, 0], kind="stable")
    sf = front[o]
    lower = np.full((n + 1, d), -np.inf)
    upper = np.full((n + 1, d), np.inf)
    lower[1:] = sf
    upper[:-1] = sf
    upper[-1] = ref
    valid = np.all(upper > lower, axis=1)
    return lower[valid], upper[valid]


def batch_ehvi(lower, upper, means, variances):
    """hv_box_decomposition.py:353-416: score_c = sum_b prod_j psi(b, j, c).

    psi = sigma (phi((l-mu)/sigma) - phi((u-mu)/sigma)) + mu (Phi((u-mu)/sigma) - Phi((l-mu)/sigma));
    infinite bounds give Phi = 0 / 1 and phi = 0.
    """
    means = np.asarray(means, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        std = np.sqrt(np.asarray(variances, dtype=np.float64))
    out = np.zeros(means.shape[0])
    if lower.shape[0] == 0:
        return out
    for i in range(means.shape[0]):
        mu = means[i][None, :]
        sd = std[i][None, :]
        with np.errstate(invalid="ignore", divide="ignore"):
            zl = (lower - mu) / sd
            zu = (upper - mu) / sd
        pl = np.where(np.isinf(lower), 0.0, norm.cdf(zl))
        pu = np.where(np.isinf(upper), 1.0, norm.cdf(zu))
        psi = sd * (norm.pdf(zl) - norm.pdf(zu)) + mu * (pu - pl)
        out[i] = np.sum(np.prod(psi, axis=1))
    return out


def ehvi_mp(lower, upper, means, variances, dps=50):
    """``batch_ehvi`` evaluated in mpmath at ``dps`` digits on the exact float64 inputs (small sizes only).

    Infinite bounds give Phi = 0 / 1 and phi = 0 exactly.  A zero variance gives z = +-inf (the same exact limits) where
    the bound differs from the mean and NaN where it equals it; a negative variance gives NaN, as float64 does.  The
    result is rounded to float64 once.
    """
    import mpmath

    lower = np.asarray(lower, dtype=np.float64)
    upper = np.asarray(upper, dtype=np.float64)
    means = np.asarray(means, dtype=np.float64)
    variances = np.asarray(variances, dtype=np.float64)
    out = np.zeros(means.shape[0])
    with mpmath.workdps(dps):
        mp = mpmath.mp

        def cdf_pdf(b, mu, sd):
            if np.isinf(b):
                return (mp.mpf(0) if b < 0 else mp.mpf(1)), mp.mpf(0)
            if sd == 0:
                if b == mu:
                    return None
                return (mp.mpf(0) if b < mu else mp.mpf(1)), mp.mpf(0)
            z = (mp.mpf(b) - mp.mpf(mu)) / sd
            return mp.ncdf(z), mp.npdf(z)

        for c in range(means.shape[0]):
            if np.any(np.isnan(variances[c])) or np.any(variances[c] < 0) or np.any(np.isnan(means[c])):
                out[c] = np.nan if lower.shape[0] else 0.0
                continue
            sd = [mp.sqrt(mp.mpf(v)) for v in variances[c]]
            total = mp.mpf(0)
            nan = False
            for b in range(lower.shape[0]):
                prod = mp.mpf(1)
                for j in range(means.shape[1]):
                    lo = cdf_pdf(lower[b, j], means[c, j], sd[j])
                    up = cdf_pdf(upper[b, j], means[c, j], sd[j])
                    if lo is None or up is None:
                        nan = True
                        break
                    prod *= sd[j] * (lo[1] - up[1]) + mp.mpf(means[c, j]) * (up[0] - lo[0])
                if nan:
                    break
                total += prod
            out[c] = np.nan if nan else float(total)
    return out


EPS = 2.0**-52  # ulp(1); a float64 operation's rounding is at most EPS / 2 of its result


def ehvi_bound(lower, upper, means, variances):
    """Bound on |score - exact| for any float64 evaluation of ``batch_ehvi``'s formula in its order of operations
    (the GPU kernel, scipy), derived operation by operation; NaN where the score is NaN.

    With e = EPS = ulp(1) and s = sqrt(v) (one rounding):
      z  = (b - mu) / s        |dz| <= 2 e |z|           (subtract, divide and the rounding of s)
      Phi(z)                   dPhi <= 5 ulp(Phi) + phi(z) |dz|        (CUDA's normcdf: 5 ulp; scipy's ndtr held to the same)
      phi(z) = c exp(-z z / 2) dphi <= phi (|z| |dz| + e z^2 + 3 e) + 2 ulp(phi)   (argument, exp's 2 ulp, the constant)
    infinite bounds give Phi = 0 / 1 and phi = 0 exactly (and so does z = +-inf from a zero variance), with no error.
      A = phi_l - phi_u        dA <= dphi_l + dphi_u + e |A|
      B = Phi_u - Phi_l        dB <= dPhi_u + dPhi_l + e |B|
      psi = s A + mu B         dpsi <= s (dA + e |A|) + |mu| dB + 2 e (s |A| + |mu| |B|)
    The product over j adds M e prod|psi| on top of sum_j dpsi_j prod_{i != j} (|psi_i| + dpsi_i) (which also covers the
    second-order terms), and the sum over the nb boxes adds nb e sum_b |prod_b|.
    """
    from scipy.special import ndtr

    lower = np.asarray(lower, dtype=np.float64)
    upper = np.asarray(upper, dtype=np.float64)
    means = np.asarray(means, dtype=np.float64)
    variances = np.asarray(variances, dtype=np.float64)
    nb, M = lower.shape
    out = np.zeros(means.shape[0])
    if nb == 0:
        return out
    e = EPS

    def terms(b, mu, sd):
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            z = (b - mu) / sd
            exact = np.isinf(b) | np.isinf(z)
            zf = np.where(exact, 0.0, z)
            cdf = np.where(np.isinf(b), (b > 0).astype(np.float64), ndtr(z))
            pdf = np.where(exact, 0.0, norm.pdf(zf))
            dz = 2 * e * np.abs(zf)
            dcdf = np.where(exact, 0.0, 5 * np.spacing(np.abs(cdf)) + pdf * dz)
            # where phi underflows to 0 its exact value is below the smallest subnormal
            dpdf = np.where(exact, 0.0, np.where(pdf > 0, pdf * (np.abs(zf) * dz + e * zf * zf + 3 * e), 0.0) + 2 * np.spacing(pdf))
        return cdf, pdf, dcdf, dpdf

    for c in range(means.shape[0]):
        mu = means[c][None, :]
        with np.errstate(invalid="ignore"):
            sd = np.sqrt(variances[c])[None, :]
        pl, dl, dpl, ddl = terms(lower, mu, sd)
        pu, du, dpu, ddu = terms(upper, mu, sd)
        A = dl - du
        B = pu - pl
        dA = ddl + ddu + e * np.abs(A)
        dB = dpu + dpl + e * np.abs(B)
        psi = np.abs(sd * A + mu * B)
        dpsi = sd * (dA + e * np.abs(A)) + np.abs(mu) * dB + 2 * e * (sd * np.abs(A) + np.abs(mu) * np.abs(B))
        with np.errstate(invalid="ignore", over="ignore"):
            prod = np.prod(psi, axis=1)
            dprod = M * e * prod
            for j in range(M):
                others = np.prod(np.delete(psi + dpsi, j, axis=1), axis=1)
                dprod = dprod + dpsi[:, j] * others
            out[c] = np.sum(dprod) + nb * e * np.sum(prod)
    return out


def select_candidates(front, means, variances, ref, k):
    """hv_box_decomposition.py:306-351: indices of the k largest scores (+ the scores).

    Ties are broken by candidate index (stable), the reference uses numpy's
    default unstable argsort.
    """
    lower, upper = decompose_boxes(front, ref)
    score = batch_ehvi(lower, upper, means, variances)
    sel = np.argsort(-score, kind="stable")[:k]
    return sel, score
