"""Nine to sixteen objectives on the GPU: rank, distances, survival and selection against the CPU oracle, one generation
of every optimizer plugin, and the Monte-Carlo hypervolume estimators (csrc/hv_mc.cu) against exact volumes."""

import itertools

import numpy as np
import pytest

from oracle import agemoea, dda, indicators, moea
from oracle import hv as ohv

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def sphere(rng, n, M, noise=0.05):
    x = rng.random((n, M)) + 1e-3
    return x / np.linalg.norm(x, axis=1, keepdims=True) * (1 + noise * rng.random((n, 1)))


# ------------------------------------------------------------------------------------------ rank
@pytest.mark.parametrize("M", [9, 10, 12, 15, 16])
@pytest.mark.parametrize("n", [1, 127, 128, 129, 3000])
def test_rank_vs_canonical(L, n, M):
    rng = np.random.default_rng(n * 31 + M)
    Y = sphere(rng, n, M) if n > 129 else rng.random((n, M))
    assert np.array_equal(L.rank_nd(Y), dda.rank_canonical(Y))
    # tied columns and duplicate rows
    T = np.floor(rng.random((n, M)) * 3)
    T[: n // 3] = T[n // 3: 2 * (n // 3)]
    assert np.array_equal(L.rank_nd(T), dda.rank_canonical(T))


@pytest.mark.parametrize("M", [12, 16])
def test_rank_full_size_property(L, M):
    rng = np.random.default_rng(M)
    n = 131072
    Y = rng.random((n, M))
    r = L.rank_nd(Y)
    for i in rng.choice(n, size=200, replace=False):
        dom = np.all(Y <= Y[i], axis=1) & np.any(Y < Y[i], axis=1)
        assert r[i] == ((r[dom].max() + 1) if dom.any() else 0)
    assert len(np.unique(r)) == r.max() + 1


# ------------------------------------------------------------------------------------------ distances, truncation, AGE, EHVI
@pytest.mark.parametrize("M", range(9, 17))
def test_distances_truncation_age_and_ehvi(L, M):
    rng = np.random.default_rng(100 + M)
    n = 400
    Y = sphere(rng, n, M)  # tie-free columns
    assert np.array_equal(L.crowding_distance(Y), indicators.crowding_distance_metric(Y))
    assert np.array_equal(L.euclidean_distance(Y), indicators.euclidean_distance_metric(Y))
    X = rng.random((n, 4))
    for code, metric in ((L.METRIC_CROWDING, indicators.crowding_distance_metric), (L.METRIC_EUCLIDEAN, indicators.euclidean_distance_metric),
                         (L.METRIC_NONE, None)):
        xs, ys, rk, _ = L.remove_worst(X, Y, 150, code)
        xo, yo, rko = moea.remove_worst(X, Y, 150, [metric] if metric else None, rank_fn=dda.rank_canonical)[:3]
        assert np.array_equal(ys, yo) and np.array_equal(xs, xo) and np.array_equal(rk, rko), code
    # AGE-MOEA greedy survival on a front
    fy = sphere(rng, 120, M, noise=0.0)
    ideal = fy.min(axis=0)
    yf = fy - ideal
    ext = agemoea.corner_solutions(yf)
    yn = yf / agemoea.hyperplane_normalization(yf, ext)
    p = agemoea.geometry_p(yn, ext)
    _, _, cd = agemoea.survival_score(fy, ideal)
    np.testing.assert_allclose(L.age_survival(yn, np.linalg.norm(yn, p, axis=1), p, ext), cd, rtol=1e-10)
    # EHVI selection
    front = sphere(rng, 30, M, noise=0.0)
    mu = sphere(rng, 64, M, noise=0.2)
    var = 0.01 + 0.05 * rng.random((64, M))
    ref = np.full(M, 1.3)
    sel, score = L.ehvi_select(front, mu, var, ref, 5, nds=False, return_scores=True)
    osel, oscore = ohv.select_candidates(front, mu, var, ref, 5)
    np.testing.assert_allclose(score, oscore, rtol=1e-9)
    assert np.array_equal(sel, osel)


def test_rank0_filter_above_eight_objectives_keeps_the_exact_route_at_eight(L):
    with pytest.raises(L.DmoError):  # exact hypervolume stays at M <= 8
        L.hypervolume(np.full((3, 9), 0.5), np.ones(9))


# ------------------------------------------------------------------------------------------ plugins
@pytest.mark.parametrize("name,M,mv", [(nm, M, False) for M in (10, 16) for nm in ("NSGA2", "AGEMOEA", "SMPSO", "CMAES", "TRS")] + [("NSGA2", 8, True)])
def test_one_generation_of_each_plugin(L, name, M, mv):
    import dmosopt_b200 as b2

    d, pop = 12, 64
    rng = np.random.default_rng(7)
    f = lambda x: sphere(np.random.default_rng(int(x.sum() * 1e6) % 2**32), len(x), M, noise=0.0) * (1 + x[:, :1])  # noqa: E731
    kw = {"optimize_mean_variance": True} if mv else {}
    opt = getattr(b2, name)(popsize=pop, nInput=d, nOutput=M, model=b2.Model(), **kw)
    x0 = rng.random((5 * pop, d))  # SMPSO seeds its swarm_size (5) swarms from the initial rows
    y0 = f(x0)
    if mv:
        y0 = np.hstack((y0, 0.1 * rng.random(y0.shape)))
    opt.initialize_strategy(x0, y0.astype(np.float32), np.column_stack((np.zeros(d), np.ones(d))), np.random.default_rng(3))
    launches = L.launch_count()
    x_gen, st = opt.generate()
    y_gen = f(np.asarray(x_gen))
    if mv:
        y_gen = np.hstack((y_gen, 0.1 * rng.random(y_gen.shape)))
    if name == "NSGA2":
        parents_x, parents_y = np.array(opt.state.population_parm, dtype=np.float64), np.array(opt.state.population_obj, dtype=np.float64)
        x_gen_h = np.array(x_gen, dtype=np.float64)
    opt.update(x_gen, y_gen, st)
    assert L.launch_count() > launches
    px, py = opt.get_population_strategy()
    assert np.all(np.isfinite(px)) and np.all(np.isfinite(py)) and py.shape[1] == y0.shape[1]
    if name == "NSGA2":
        # survivors: the first popsize rows of the sortMO order of children stacked over parents (NSGA2.py:205-236)
        metrics = opt.y_distance_metrics
        fn = None if metrics is None else {"crowding": indicators.crowding_distance_metric, "euclidean": indicators.euclidean_distance_metric}[metrics[0]]
        xo, yo, rko = moea.remove_worst(np.vstack((x_gen_h, parents_x)), np.vstack((y_gen, parents_y)), pop, [fn] if fn else None,
                                        rank_fn=dda.rank_canonical)[:3]
        assert np.array_equal(py, yo.astype(py.dtype)) and np.array_equal(np.asarray(px, dtype=np.float64), xo.astype(px.dtype).astype(np.float64))
        assert np.array_equal(np.asarray(opt.state.rank), rko)


# ------------------------------------------------------------------------------------------ Monte-Carlo hypervolume
ALGOS = ["hybrid", "fpras", "mcm2rv", "monte_carlo"]


def embedded(L, rng, n, m_low, M):
    """An m_low-objective front embedded into M objectives with constant extra coordinates: the exact volume is the
    m_low-objective one (GPU exact route, m_low <= 8) times the box of the extra coordinates."""
    P = sphere(rng, n, m_low, noise=0.0)
    ref_low = np.full(m_low, 1.1)
    c = 0.2 + 0.5 * rng.random(M - m_low)
    ref = np.concatenate((ref_low, np.full(M - m_low, 1.0)))
    F = np.hstack((P, np.tile(c, (n, 1))))
    return F, ref, L.hypervolume(P, ref_low) * np.prod(1.0 - c)


def inclusion_exclusion(P, ref):
    total = 0.0
    for k in range(1, len(P) + 1):
        for sub in itertools.combinations(range(len(P)), k):
            total += (-1) ** (k + 1) * np.prod(ref - P[list(sub)].max(axis=0))
    return total


def test_single_point_is_exact(L):
    for M in (2, 10, 16):
        p = np.full((1, M), 0.25)
        for a in ("fpras", "hybrid"):
            v, info = L.hypervolume_mc(p, np.ones(M), a, 0.05, 0.25, seed=1)
            assert v == pytest.approx(0.75**M, rel=1e-15), (M, a, info)


@pytest.mark.parametrize("case", [(2, 10, 2000), (3, 12, 500), (6, 16, 300), (8, 10, 200)])
@pytest.mark.parametrize("algo", ALGOS)
def test_estimates_within_epsilon_of_exact(L, case, algo):
    m_low, M, n = case
    F, ref, exact = embedded(L, np.random.default_rng(m_low * M), n, m_low, M)
    v, info = L.hypervolume_mc(F, ref, algo, 0.01, 0.01, n_samples=2_000_000, seed=3)
    tol = 0.01 if algo != "monte_carlo" else 0.005
    assert abs(v - exact) <= tol * exact, (v, exact, info)


@pytest.mark.parametrize("M,n", [(10, 8), (13, 10), (16, 12)])
def test_small_random_fronts_by_inclusion_exclusion(L, M, n):
    rng = np.random.default_rng(M + n)
    P = sphere(rng, n, M, noise=0.3)
    ref = np.full(M, 1.4)
    exact = inclusion_exclusion(P, ref)  # dominated rows change nothing
    for algo in ("hybrid", "fpras", "mcm2rv"):
        v, info = L.hypervolume_mc(P, ref, algo, 0.01, 0.01, seed=5)
        assert abs(v - exact) <= 0.01 * exact, (algo, v, exact, info)


def test_miss_rate_is_at_most_delta(L):
    F, ref, exact = embedded(L, np.random.default_rng(1), 40, 3, 10)
    for algo in ("fpras", "mcm2rv", "hybrid"):
        misses = sum(abs(L.hypervolume_mc(F, ref, algo, 0.05, 0.25, seed=s)[0] - exact) > 0.05 * exact for s in range(200))
        assert misses <= 0.25 * 200, (algo, misses)


@pytest.mark.parametrize("M", [3, 5, 8])
def test_agrees_with_the_exact_route_at_eight_or_fewer(L, M):
    rng = np.random.default_rng(M)
    F = sphere(rng, 60, M)
    ref = np.full(M, 1.2)
    exact = L.hypervolume(F, ref)
    for algo in ("hybrid", "fpras", "mcm2rv"):
        assert abs(L.hypervolume_mc(F, ref, algo, 0.01, 0.01, seed=2)[0] - exact) <= 0.01 * exact, algo


@pytest.mark.parametrize("algo", ALGOS)
def test_determinism_streams_and_filtering(L, algo):
    F, ref, exact = embedded(L, np.random.default_rng(9), 300, 3, 12)
    a = L.hypervolume_mc(F, ref, algo, 0.02, 0.1, n_samples=500_000, seed=11, stream=0)
    b = L.hypervolume_mc(F, ref, algo, 0.02, 0.1, n_samples=500_000, seed=11, stream=0)
    assert a == b
    c = L.hypervolume_mc(F, ref, algo, 0.02, 0.1, n_samples=500_000, seed=11, stream=1)
    assert c[0] != a[0] and abs(c[0] - exact) <= 0.02 * exact
    extra = np.vstack((F, F[:50] + 0.01, np.full((3, 12), 2.0)))  # dominated rows and rows outside ref
    assert L.hypervolume_mc(extra, ref, algo, 0.02, 0.1, n_samples=500_000, seed=11, stream=0) == a


def test_plugin_mirror_and_install_route_to_the_gpu(L):
    from dmosopt_b200 import hv as bhv

    F, ref, exact = embedded(L, np.random.default_rng(4), 200, 3, 10)
    h = bhv.AdaptiveHyperVolume(ref, mc_epsilon=0.02, mc_delta=0.1, seed=8)
    v0, v1 = h.compute_hypervolume(F), h.compute_hypervolume(F)
    assert v0 != v1 and abs(v0 - exact) <= 0.02 * exact and abs(v1 - exact) <= 0.02 * exact
    assert bhv.AdaptiveHyperVolume(ref, mc_epsilon=0.02, mc_delta=0.1, seed=8).compute_hypervolume(F) == v0
    from oracle import reference_build

    path = reference_build.reference_path()
    if path is None:
        pytest.skip("reference package not built (oracle/_ref)")
    import sys

    sys.path.insert(0, path)
    try:
        from dmosopt import hv as rhv

        from dmosopt_b200 import patch

        patch.install()
        try:
            for M in (10, 16):
                F, ref, exact = embedded(L, np.random.default_rng(M), 200, 3, M)
                launches = L.launch_count()
                v = rhv.AdaptiveHyperVolume(ref, mc_epsilon=0.02, mc_delta=0.1).compute_hypervolume(F)
                assert L.launch_count() > launches and abs(v - exact) <= 0.02 * exact
        finally:
            patch.uninstall()
    finally:
        sys.path.remove(path)


@pytest.mark.parametrize("algo", ["fpras", "mcm2rv", "hybrid"])
def test_distributional_parity_with_the_reference_estimators(L, algo):
    """Same random variables and stopping rules as dmosopt/hv_adaptive.py: over 32 runs each on a 30-point, 10-objective
    front at epsilon 0.05, the means of the estimate and of N (num_samples) agree within a few standard errors."""
    from oracle import reference_build
    from oracle.hv_mc import filtered_front

    path = reference_build.reference_path()
    if path is None:
        pytest.skip("reference package not built (oracle/_ref)")
    import contextlib
    import io
    import sys

    sys.path.insert(0, path)
    try:
        from dmosopt import hv_adaptive
    finally:
        sys.path.remove(path)
    rng = np.random.default_rng(30)
    x = rng.random((30, 10)) + 0.2
    F = x / np.linalg.norm(x, axis=1, keepdims=True)
    ref = np.full(10, 1.1)
    assert np.array_equal(filtered_front(F, ref), F)  # the reference's unfiltered front is the GPU's filtered one
    fn = getattr(hv_adaptive, f"compute_hypervolume_{algo}")
    runs = 32
    ref_v, ref_n, gpu_v, gpu_n = [], [], [], []
    np.random.seed(2026)
    for s in range(runs):
        with contextlib.redirect_stdout(io.StringIO()):  # compute_hypervolume_mcm2rv prints every iteration
            r = fn(F, ref, 0.05, 0.25)
        ref_v.append(r.hypervolume)
        ref_n.append(r.num_samples)
        v, info = L.hypervolume_mc(F, ref, algo, 0.05, 0.25, seed=77, stream=s)
        gpu_v.append(v)
        gpu_n.append(info["samples"])
    for a, b, what in ((gpu_v, ref_v, "estimate"), (gpu_n, ref_n, "N")):
        a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
        se = np.sqrt(a.var(ddof=1) / runs + b.var(ddof=1) / runs)
        assert abs(a.mean() - b.mean()) <= 4.0 * se + 1e-12 * abs(b.mean()), (algo, what, a.mean(), b.mean(), se)
