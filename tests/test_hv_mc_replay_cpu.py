"""The draw-for-draw replay of the Monte-Carlo hypervolume estimators (oracle/hv_mc_replay.py), checked without a GPU.

  * it equals a literal restatement written here, one sample, one Philox call and one trial at a time, with the
    binary-search box choice and the sequential stopping rules, on small cases of every route;
  * it is an honest estimator: within epsilon of exact volumes, and its mean N agrees with the NumPy-stream
    restatement of the reference's estimators (oracle/hv_mc.py);
  * R, M1 and theta as the code forms them agree with a 50-digit evaluation to within the code's rounding;
  * every case tests/test_gpu_hv_mc_exact.py runs reaches the edge it claims.
"""

import math
import os

import mpmath
import numpy as np
import pytest

from oracle import hv_exact, hv_mc
from oracle import hv_mc_cases as cases
from oracle import hv_mc_replay as rp
from oracle.philox import philox4x32_10, u01_53


# ------------------------------------------------------------------------------------------ literal restatement
def draw(seed, s, stream, purpose, d):
    hi = (d << 32) | ((stream & 0xFFFFFF) << 8) | purpose
    return [int(w) for w in philox4x32_10(seed, np.uint64(s), np.uint64(hi))]


def uniforms(seed, s, stream, purpose, M):
    u = []
    for c in range((16 + 2) // 2):
        if 2 * c <= M:
            r = draw(seed, s, stream, purpose, c)
            u.append(float(u01_53(r[0], r[1])))
            if 2 * c + 1 <= M:
                u.append(float(u01_53(r[2], r[3])))
    return u


def binary_search(cdf, u):
    lo, hi = 0, len(cdf) - 1
    while lo < hi:
        mid = (lo + hi) >> 1
        if cdf[mid] > u:
            hi = mid
        else:
            lo = mid + 1
    return lo


class Literal:
    def __init__(self, F, ref, seed, stream):
        self.ref = [float(r) for r in ref]
        self.P = [list(map(float, p)) for p in hv_mc.filtered_front(F, ref)]
        self.n, self.M, self.seed, self.stream = len(self.P), len(self.ref), seed, stream
        self.W, self.cdf, self.ideal = 0.0, [], list(self.P[0])
        for p in self.P:
            v = 1.0
            for j in range(self.M):
                v *= self.ref[j] - p[j]
                self.ideal[j] = min(self.ideal[j], p[j])
            self.W += v
            self.cdf.append(self.W)
        self.cdf = [c / self.W for c in self.cdf]
        self.U = 1.0
        for j in range(self.M):
            self.U *= self.ref[j] - self.ideal[j]
        self.tests = self.N = self.sum_xi = self.next = 0

    def point(self, s, purpose):
        u = uniforms(self.seed, s, self.stream, purpose, self.M)
        i = binary_search(self.cdf, u[0])
        return [self.P[i][j] + (self.ref[j] - self.P[i][j]) * u[1 + j] for j in range(self.M)]

    def fpras(self, target):
        while self.tests < target:
            s = self.next
            self.next += 1
            x = self.point(s, rp.P_FPRAS_SAMPLE)
            t = 0
            while self.tests < target:
                w = draw(self.seed, s, self.stream, rp.P_FPRAS_TRIAL, t >> 2)[t & 3]
                k = (w * self.n) >> 32
                t += 1
                self.tests += 1
                if all(x[j] > self.P[k][j] for j in range(self.M)):
                    self.N += 1
                    self.sum_xi += t
                    break

    def fpras_value(self):
        return (self.W / self.n) * (self.sum_xi / max(self.N, 1))

    def scan(self, s, purpose, eta):
        u = uniforms(self.seed, s, self.stream, purpose, self.M)
        x = [self.ideal[j] + (self.ref[j] - self.ideal[j]) * u[1 + j] for j in range(self.M)]
        tests = 0
        for p in self.P:
            tests += 1
            if all(p[j] <= x[j] for j in range(self.M)):
                e = False
                if eta:
                    k = (draw(self.seed, s, self.stream, rp.P_MCM_ETA, 0)[0] * self.n) >> 32
                    e = all(self.P[k][j] <= x[j] for j in range(self.M))
                    tests += 1
                return True, e, tests
        return False, False, tests

    def mcm2rv(self, eps, delta):
        R = math.floor((4.0 * (1.0 + eps * (1.0 - eps)) * math.log(2.0 / delta)) / (eps * eps * (1.0 - eps) * (1.0 - eps)))
        N = S = tests = s = 0
        while S < R:
            dom, e, t = self.scan(s, rp.P_MCM_SAMPLE, True)
            s += 1
            tests += t
            N += dom
            S += e
        return (self.W / self.n) * (N / S), N, tests

    def monte_carlo(self, n_samples):
        dom = tests = samples = s = 0
        for _ in range(1000):
            for _ in range(n_samples):
                d, _, t = self.scan(s, rp.P_MC_SAMPLE, False)
                s += 1
                dom += d
                tests += t
            samples += n_samples
            if dom:
                break
        return self.U * (dom / n_samples), samples, tests

    def probe_mean(self):
        total = 0.0
        for p in range(50):
            x = self.point(p, rp.P_PROBE_SAMPLE)
            c = sum(all(x[j] > q[j] for j in range(self.M)) for q in self.P)
            xi = self.n
            for t in range(self.n if c else 0):
                r = draw(self.seed, p, self.stream, rp.P_PROBE_TRIAL, t)
                if float(u01_53(r[0], r[1])) * (self.n - t) < c:
                    xi = t + 1
                    break
            total += xi
        return total / 50


def literal(F, ref, algo, eps, delta, n_samples, seed, stream):
    lt = Literal(F, ref, seed, stream)
    n, W, U = lt.n, lt.W, lt.U
    if algo == "monte_carlo":
        return lt.monte_carlo(n_samples) + ("MonteCarlo",)
    M1 = 8.0 * (1.0 + eps) * n * math.log(2.0 / delta) / (eps * eps)
    if algo == "mcm2rv":
        return lt.mcm2rv(eps, delta) + ("MCM2RV",)
    if algo == "fpras":
        lt.fpras(int(M1))
        return lt.fpras_value(), max(lt.N, 1), lt.tests, "FPRAS"
    if W / U > 5.0:
        return lt.mcm2rv(eps, delta) + ("MCM2RV",)
    if W / U >= 1.2:
        m = lt.probe_mean()
        if m > 20.0:
            return lt.mcm2rv(eps, delta) + ("MCM2RV",)
        if m >= 5.0:
            Rv = (4.0 * (1.0 + eps * (1.0 - eps)) * math.log(2.0 / delta)) / (eps * eps * (1.0 - eps) * (1.0 - eps))
            cum = 0.0
            for f in (0.01, 0.02, 0.04, 0.08):
                cum += f
                lt.fpras(int(cum * M1))
                V = lt.fpras_value()
                e1 = eps / math.sqrt(cum)
                with np.errstate(all="ignore"):
                    th = [float(n * n * (Vb * Vb + (U - Vb) * W) / (W * W) * (Rv / M1))
                          for Vb in (np.float64(V) / np.float64(1.0 - e1), np.float64(V) / np.float64(1.0 + e1))]
                if th[0] < (1.0 - cum) * 0.85:
                    v, N, t = lt.mcm2rv(eps, delta)
                    return v, N, t + lt.tests, "Hybrid-MCM2RV"
                if th[1] > (1.0 - cum) * 1.15:
                    break
            lt.fpras(int(M1))
            return lt.fpras_value(), max(lt.N, 1), lt.tests, "Hybrid-FPRAS"
    lt.fpras(int(M1))
    return lt.fpras_value(), max(lt.N, 1), lt.tests, "FPRAS"


SMALL = [
    ("fpras", lambda: (cases.sphere(np.random.default_rng(1), 6, 3), np.full(3, 1.1)), 0.3, 0.3, 0, 3, 1),
    ("fpras", lambda: (cases.sphere(np.random.default_rng(2), 5, 16), np.full(16, 1.2)), 0.4, 0.3, 0, cases.HIGH_SEED, cases.LAST_STREAM),
    ("mcm2rv", lambda: (cases.sphere(np.random.default_rng(3), 7, 2), np.full(2, 1.1)), 0.3, 0.3, 0, 4, 2),
    ("mcm2rv", lambda: (cases.sphere(np.random.default_rng(4), 5, 9), np.full(9, 1.2)), 0.3, 0.3, 0, cases.HIGH_SEED, 7),
    ("monte_carlo", lambda: cases.staircase(9, 3, 1), 0, 0, 300, 5, 0),
    ("monte_carlo", lambda: cases.corners(3, 0.942), 0, 0, 3, 3, 0),
    ("hybrid", lambda: cases.disjoint(3, 5, 5), 0.3, 0.3, 0, 6, 0),
    ("hybrid", lambda: cases.bumped(181), 0.3, 0.25, 0, 7, 0),  # level 3
    ("hybrid", lambda: cases.bumped(206), 0.3, 0.25, 0, 7, 0),
]


@pytest.mark.parametrize("k", range(len(SMALL)))
def test_replay_equals_the_literal_restatement(k):
    algo, build, eps, delta, ns, seed, stream = SMALL[k]
    F, ref = build()
    v, info = rp.hypervolume_mc(F, ref, algo, eps, delta, ns, seed, stream)
    want = literal(F, ref, algo, eps, delta, ns, seed, stream)
    assert (v, info["samples"], info["tests"], info["algorithm"]) == want
    if k == 7:
        assert info["record"]["level3"], "the level-3 case no longer reaches level 3"


# ------------------------------------------------------------------------------------------ an honest estimator
def integer_front(rng, n, M, S=24):
    """n mutually non-dominated integer rows (a random slice of a simplex-like front) and an integer ref."""
    K = hv_exact.simplex_front(M, n, rng, S) if M <= 8 else rng.integers(0, S, (n, M))
    return np.asarray(K, dtype=np.float64), np.full(M, S + 2.0)


@pytest.mark.parametrize("M", [3, 5, 10])
@pytest.mark.parametrize("algo", ["fpras", "mcm2rv", "hybrid"])
def test_estimates_within_epsilon_of_exact(M, algo):
    rng = np.random.default_rng(M)
    K, R = integer_front(rng, 8, M)
    P = hv_mc.filtered_front(K, R)
    exact = float(hv_exact.hv_exact(P, R) if M <= 8 else hv_exact.hv_incl_excl(P, R))
    eps = 0.05
    misses = 0
    for seed in range(6):
        v, _ = rp.hypervolume_mc(K, R, algo, eps, 0.1, seed=seed, stream=seed)
        misses += abs(v - exact) > eps * exact
    assert misses <= 1, (misses, exact)


def test_mean_n_agrees_with_the_reference_random_variables():
    """Same random variables, different streams: over 24 runs the mean N of the replay and of the NumPy restatement of
    the reference's estimators agree within four standard errors."""
    rng = np.random.default_rng(30)
    x = rng.random((12, 6)) + 0.2
    F = x / np.linalg.norm(x, axis=1, keepdims=True)
    ref = np.full(6, 1.1)
    gen = np.random.default_rng(2026)
    for algo in ("fpras", "mcm2rv"):
        a = np.array([rp.hypervolume_mc(F, ref, algo, 0.15, 0.25, seed=77, stream=s)[1]["samples"] for s in range(24)], dtype=np.float64)
        b = np.array([getattr(hv_mc, algo)(F, ref, 0.15, 0.25, gen)[1] for _ in range(24)], dtype=np.float64)
        se = math.sqrt(a.var(ddof=1) / 24 + b.var(ddof=1) / 24)
        assert abs(a.mean() - b.mean()) <= 4.0 * se, (algo, a.mean(), b.mean(), se)


# ------------------------------------------------------------------------------------------ host formulas
@pytest.mark.parametrize("eps,delta", [(0.01, 0.25), (0.05, 0.1), (0.1, 0.25), (0.3, 0.01), (0.9, 0.9), (0.5, 0.5)])
def test_budgets_and_theta_against_50_digits(eps, delta):
    """M1, R and theta take a handful of float64 operations each: within 1e-15 relative of the 50-digit values, and
    M1's truncation and R's floor are the real ones wherever the real value is not within that of an integer."""
    mpmath.mp.dps = 50
    e, d = mpmath.mpf(eps), mpmath.mpf(delta)
    Rx = 4 * (1 + e * (1 - e)) * mpmath.log(2 / d) / (e * e * (1 - e) ** 2)
    Rv = rp.mcm2rv_rv(eps, delta)
    assert abs(Rv / Rx - 1) < 1e-15
    if abs(Rx - mpmath.nint(Rx)) > 1e-12 * Rx:
        assert math.floor(Rv) == int(mpmath.floor(Rx))
    for nf in (1, 7, 40, 2000):
        M1x = 8 * (1 + e) * nf * mpmath.log(2 / d) / (e * e)
        M1 = rp.budget_m1(eps, delta, nf)
        assert abs(M1 / M1x - 1) < 1e-15
        if abs(M1x - mpmath.nint(M1x)) > 1e-12 * M1x:
            assert int(M1) == int(mpmath.floor(M1x))
        for cum, target in rp.level3_targets(M1):
            assert abs(cum - [0.01, 0.03, 0.07, 0.15][rp.level3_targets(M1).index((cum, target))]) < 1e-16
            assert target == int(cum * M1)
    nf, U, W, V = 40, 0.8, 2.5, 0.6
    M1x = 8 * (1 + e) * nf * mpmath.log(2 / d) / (e * e)
    thx = nf * nf * (mpmath.mpf(V) ** 2 + (mpmath.mpf(U) - V) * W) / (mpmath.mpf(W) ** 2) * (Rx / M1x)
    assert abs(rp.theta(nf, U, W, V, Rv, rp.budget_m1(eps, delta, nf)) / thx - 1) < 1e-15


def test_level3_targets():
    """The level-3 rounds run FPRAS to (int64_t)(cum * M1), cum the float64 running sum of 0.01, 0.02, 0.04, 0.08, as
    hv_mc.cu states them.  No GPU case gets past round 1 (oracle/hv_mc_cases.py), so the later targets are pinned here:
    for these budgets they differ from a target formed from each round's own fraction."""
    src = open(os.path.join(os.path.dirname(rp.__file__), "..", "dmosopt_b200", "csrc", "hv_mc.cu")).read()
    assert "const double fractions[4] = {0.01, 0.02, 0.04, 0.08};" in src
    assert "cum += fractions[r];" in src and "run_fpras(ctx, mf, (int64_t)(cum * M1), st)" in src
    for M1 in (665.5, 139738.9, 4.2e6 + 0.5):
        cums = [0.01, 0.01 + 0.02, 0.01 + 0.02 + 0.04, 0.01 + 0.02 + 0.04 + 0.08]
        assert rp.level3_targets(M1) == [(c, int(c * M1)) for c in cums]
        own = [int(f * M1) for f in (0.01, 0.02, 0.04, 0.08)]
        assert all(t != o for (_, t), o in zip(rp.level3_targets(M1)[1:], own[1:]))


def test_r_differs_from_the_power_form_only_by_rounding():
    """oracle/hv_mc.py forms R with eps**2 (1 - eps)**2; the code's product order can differ by an ulp, so the replay
    uses the code's order.  Both stay within a few ulps of the 50-digit value."""
    mpmath.mp.dps = 50
    for eps in np.linspace(0.01, 0.95, 95):
        eps = float(eps)
        Rx = 4 * (1 + mpmath.mpf(eps) * (1 - mpmath.mpf(eps))) * mpmath.log(2 / mpmath.mpf(0.25)) / (mpmath.mpf(eps) ** 2 * (1 - mpmath.mpf(eps)) ** 2)
        a = rp.mcm2rv_rv(eps, 0.25)
        b = (4 * (1 + eps * (1 - eps)) * np.log(2 / 0.25)) / (eps**2 * (1 - eps) ** 2)
        assert abs(a / Rx - 1) < 1e-14 and abs(b / Rx - 1) < 1e-14


# ------------------------------------------------------------------------------------------ the GPU file's claims
@pytest.mark.parametrize("case", cases.CASES, ids=[c.id for c in cases.CASES])
def test_gpu_cases_reach_their_edges(case):
    F, ref = cases.case_input(case)
    _, info = rp.hypervolume_mc(F, ref, **case.args())
    if case.claim:
        case.claim(F, ref, info)


def test_zero_volume_boxes_are_never_chosen_in_the_hybrid_probes():
    F, _, ref = cases.underflow_front()
    _, info = rp.hypervolume_mc(F, ref, "hybrid", 0.15, 0.25, seed=5)
    cases.boxes_nonzero(F, ref, info)
