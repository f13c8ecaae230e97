"""The per-generation operator kernels (csrc/variation.cu, csrc/moea_ext.cu, csrc/smpso.cu) against float64 / long-double
replays of the reference's formulas, fed the kernels' own Philox draws recomputed on the host (oracle/philox.py).

Tolerances.  Where a kernel rounds every operation in NumPy's order (``__d*_rn``), the comparison is bit for bit.  Where
CUDA's ``pow`` is involved (polynomial mutation, SBX, the Minkowski distances of AGE-MOEA) the kernel is compared with an
evaluation whose ``pow`` and everything after it run in ``np.longdouble``, under a bound derived operation by operation
(``mutation_ref`` / ``sbx_ref`` below): CUDA documents ``pow`` to 2 ulp, and each later rounding of the kernel adds at most
one ulp of its result on top of the propagated error.  Against a float64 NumPy evaluation (whose ``pow`` is within 1 ulp)
the ``pow`` allowance is 3 ulp.  Where the kernel sums without an ordering guarantee (the MO-CMA-ES matrix-vector
products, possibly FMA-contracted), the tolerance is d * eps * sum|terms|, carried through the formulas that follow.
"""

import numpy as np
import pytest

from oracle import moea, nsga2, philox
from oracle import cmaes as ocm

gpu = pytest.mark.gpu
LD = np.longdouble
EPS = 2.0**-52  # ulp(1): one ulp of |x| is at most EPS * |x|


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def ulp(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)))


def within(got, ref, bound):
    """|got - ref| <= bound elementwise, NaN where the reference is NaN; the differences in long double."""
    got, ref = np.asarray(got), np.asarray(ref)
    nan = np.isnan(ref.astype(np.float64))
    assert np.array_equal(np.isnan(got), nan), "NaN pattern differs"
    err = np.abs(got.astype(LD) - ref.astype(LD))
    ok = (err <= np.asarray(bound, dtype=LD)) | nan
    if not ok.all():
        i = np.flatnonzero(~ok.ravel())[:5]
        raise AssertionError(f"{(~ok).sum()} entries outside the bound, e.g. got {got.ravel()[i]} ref {ref.ravel()[i]} bound {np.ravel(bound)[i] if np.ndim(bound) else bound}")


# ---------------------------------------------------------------------------------------------- references
def mutation_ref(parent, u, di, lb, ub, rate, pow_ulps=2):
    """MOEA.py:191-212.  The operations before ``pow`` are float64 (the kernel and NumPy round them identically), ``pow``
    and what follows run in long double.  Bound on the kernel's error, propagated step by step:
      P = pow(x, e)         dP = pow_ulps ulp(P)
      D = P - 1 | 1 - P     dD = dP + ulp(D)
      Q = (ub - lb) D       dQ = |ub - lb| dD + ulp(Q)      (ub - lb is the same double on both sides)
      S = parent + Q        dS = dQ + ulp(S)
    and the clip is 1-Lipschitz."""
    parent, u = np.asarray(parent, np.float64), np.asarray(u, np.float64)
    e = 1.0 / (np.asarray(di, np.float64) + 1.0)
    lo = u < rate
    x = np.where(lo, 2.0 * u, 2.0 * (1.0 - u))
    P = np.power(x.astype(LD), np.broadcast_to(e, x.shape).astype(LD))
    D = np.where(lo, P - 1, 1 - P)
    W = np.asarray(ub, np.float64) - np.asarray(lb, np.float64)
    Q = W.astype(LD) * D
    S = parent.astype(LD) + Q
    child = np.minimum(np.maximum(S, LD(0) + lb), LD(0) + ub)
    child = np.where(np.isnan(S), S, child)  # np.clip propagates NaN
    bound = (np.abs(W) * (pow_ulps * ulp(P) + ulp(D)) + ulp(Q)) + ulp(S)
    return child, bound


def sbx_ref(p1, p2, u, di, lb, ub, pow_ulps=2):
    """MOEA.py:215-239, evaluated like ``mutation_ref``.  With B = pow(x, e), a = 1 - B, b = 1 + B:
      dB = pow_ulps ulp(B), da = dB + ulp(a), db = dB + ulp(b),
      s1 = a p1 + b p2: ds1 = |p1| da + ulp(a p1) + |p2| db + ulp(b p2) + ulp(s1),  c1 = s1 / 2: dc1 = ds1 / 2 + ulp(c1)
    and the same for c2 = (b p1 + a p2) / 2."""
    p1, p2, u = (np.asarray(v, np.float64) for v in (p1, p2, u))
    e = 1.0 / (np.asarray(di, np.float64) + 1.0)
    lo = u <= 0.5
    with np.errstate(divide="ignore"):
        x = np.where(lo, 2.0 * u, 1.0 / (2.0 * (1.0 - u)))
    B = np.power(x.astype(LD), np.broadcast_to(e, x.shape).astype(LD))
    a, b = 1 - B, 1 + B
    lbl, ubl = LD(0) + lb, LD(0) + ub
    out = []
    for q1, q2, f1, f2 in ((p1, p2, a, b), (p2, p1, a, b)):  # c1 = (a p1 + b p2) / 2, c2 = (b p1 + a p2) / 2
        t1, t2 = f1 * q1.astype(LD), f2 * q2.astype(LD)
        s = t1 + t2
        c = np.minimum(np.maximum(s / 2, lbl), ubl)
        c = np.where(np.isnan(s), s, c)
        dB = pow_ulps * ulp(B)
        ds = np.abs(q1) * (dB + ulp(f1)) + ulp(t1) + np.abs(q2) * (dB + ulp(f2)) + ulp(t2) + ulp(s)
        out += [c, ds / 2 + ulp(s / 2)]
    # the second pass computed (a p2 + b p1) / 2 = c2
    return out[0], out[1], out[2], out[3]


# ---------------------------------------------------------------------------------------------- variation
def edge_uniforms(rate):
    r = float(rate)
    return np.array([0.0, 2.0**-53, r, np.nextafter(r, 0.0), np.nextafter(r, 1.0), 0.5, np.nextafter(0.5, 0.0), np.nextafter(0.5, 1.0),
                     1.0 - 2.0**-53])


def variation_case(n, d, seed, rate):
    rng = np.random.default_rng(seed)
    lb = rng.uniform(-3.0, 0.5, d)
    ub = lb + rng.uniform(0.1, 4.0, d)
    if d >= 3:
        ub[1] = lb[1]  # a column with xlb == xub
        lb[2], ub[2] = -7.5, -0.25  # negative bounds
    P1 = lb + rng.random((n, d)) * (ub - lb)
    P2 = lb + rng.random((n, d)) * (ub - lb)
    U = rng.random((n, d))
    eu = edge_uniforms(rate)
    k = min(n * d, eu.size)
    U.ravel()[:k] = eu[:k]
    U.ravel()[-k:] = eu[::-1][:k]
    if n * d > 4:  # parents on either bound, and equal parents
        P1.ravel()[1 :: 7] = np.broadcast_to(lb, (n, d)).ravel()[1 :: 7]
        P1.ravel()[2 :: 7] = np.broadcast_to(ub, (n, d)).ravel()[2 :: 7]
        P2.ravel()[3 :: 7] = P1.ravel()[3 :: 7]
        P2.ravel()[4 :: 11] = np.broadcast_to(ub, (n, d)).ravel()[4 :: 11]
    di = np.where(np.arange(d) % 3 == 0, 20.0, np.where(np.arange(d) % 3 == 1, 0.0, 1e3))
    return P1, P2, U, di, lb, ub


@gpu
@pytest.mark.parametrize("n,d", [(1, 1), (255, 1), (256, 1), (257, 1), (51, 5), (8, 32), (1, 257), (65536, 30)])
@pytest.mark.parametrize("rate", [0.3, 0.7])
def test_mutation_and_sbx_at_their_edges(L, n, d, rate):
    P1, P2, U, di, lb, ub = variation_case(n, d, n * 31 + d, rate)
    got = L.mutation_u(P1, U, di, lb, ub, rate)
    ref, bound = mutation_ref(P1, U, di, lb, ub, rate)
    within(got, ref, bound)
    c1, c2 = L.sbx_u(P1, P2, U, di, lb, ub)
    r1, b1, r2, b2 = sbx_ref(P1, P2, U, di, lb, ub)
    within(c1, r1, b1)
    within(c2, r2, b2)
    # values on a bound and columns with xlb == xub are exact
    assert np.all((got >= lb) & (got <= ub)) and np.all((c1 >= lb) & (c1 <= ub)) and np.all((c2 >= lb) & (c2 <= ub))
    if d >= 3:
        assert np.all(got[:, 1] == lb[1]) and np.all(c1[:, 1] == lb[1]) and np.all(c2[:, 1] == lb[1])


@gpu
def test_mutation_branch_points_are_taken_on_the_reference_side(L):
    """At u == rate the reference takes the upper branch (u < rate is false), one ulp below it the lower one; with rate
    != 0.5 the two branches give different genes, so a kernel deciding on the wrong side is far outside the bound.
    (SBX's branches meet at u = 0.5, beta = 1, so its decision point cannot be told apart and need not be.)"""
    d = 4
    lb, ub, di = np.zeros(d), np.ones(d), np.full(d, 20.0)
    for rate in (0.25, 0.3, 0.7, 1.0 / 30.0):
        u = np.array([[rate, np.nextafter(rate, 0.0), np.nextafter(rate, 1.0), 0.5]])
        p = np.full((1, d), 0.5)
        got = L.mutation_u(p, u, di, lb, ub, rate)
        ref, bound = mutation_ref(p, u, di, lb, ub, rate)
        within(got, ref, bound)
        lower, _ = mutation_ref(p, u, di, lb, ub, np.nextafter(rate, 1.0))  # what u <= rate would give
        assert abs(float(lower[0, 0]) - got[0, 0]) > 1e3 * bound[0, 0]


@gpu
def test_variation_propagates_nan_like_np_clip(L):
    d = 3
    lb, ub = np.zeros(d), np.ones(d)
    p = np.array([[np.nan, 0.5, 0.25]])
    u = np.array([[0.1, 0.9, 0.5]])
    got = L.mutation_u(p, u, 20.0, lb, ub, 0.5)
    assert np.isnan(got[0, 0]) and np.isfinite(got[0, 1:]).all()
    assert np.isnan(moea.mutation_u(p, u, 20.0, lb, ub, 0.5)[0, 0])
    c1, c2 = L.sbx_u(p, np.full((1, d), 0.5), u, 1.0, lb, ub)
    assert np.isnan(c1[0, 0]) and np.isnan(c2[0, 0]) and np.isfinite(c1[0, 1:]).all()


# ---------------------------------------------------------------------------------------------- NSGA-II generate
def replay_plan(seed, stream, T, poolsize, d):
    """The draws of plan_kernel / children_kernel (variation.cu) recomputed from Philox."""
    t = np.arange(T, dtype=np.uint64)
    a = philox.draws(seed, stream, philox.P_DECIDE, t)
    b = philox.draws(seed, stream, philox.P_PAIR, t)
    c = philox.draws(seed, stream, philox.P_SINGLE, t)
    i1 = np.minimum(np.floor(philox.u01_53(b[0], b[1]) * float(poolsize)).astype(np.int64), poolsize - 1)
    if poolsize > 1:
        i2 = np.minimum(np.floor(philox.u01_53(b[2], b[3]) * float(poolsize - 1)).astype(np.int64), poolsize - 2)
        i2 = i2 + (i2 >= i1)
    else:
        i2 = np.zeros(T, dtype=np.int64)
    g = philox.draws(seed, stream, philox.P_GENES, np.arange(T * d, dtype=np.uint64))
    genes = np.stack([philox.u01_53(g[0], g[1]).reshape(T, d), philox.u01_53(g[2], g[3]).reshape(T, d)], axis=1)
    return {"u_cross": philox.u01_53(a[0], a[1]), "u_mut": philox.u01_53(a[2], a[3]), "pair": np.stack([i1, i2], axis=1),
            "single": np.minimum(np.floor(philox.u01_53(c[0], c[1]) * float(poolsize)).astype(np.int64), poolsize - 1), "u_genes": genes}


@gpu
@pytest.mark.parametrize("pc,pm", [(0.9, 0.1), (1.0, 0.0), (0.0, 1.0), (1.0, 1.0), (0.05, 0.05)])
@pytest.mark.parametrize("npop,poolsize,popsize,d", [(7, 2, 2, 3), (9, 3, 3, 1), (40, 2, 40, 257), (60, 3, 31, 1), (300, 150, 300, 8)])
def test_nsga2_generate_replays_exactly(L, pc, pm, npop, poolsize, popsize, d):
    _nsga2_case(L, pc, pm, npop, poolsize, popsize, d, seed=npop * 7 + d, stream=int(pc * 10) + 100 * int(pm * 10))


@gpu
def test_nsga2_generate_at_the_bench_shape(L):
    _nsga2_case(L, 0.9, 0.1, 65536, 32768, 65536, 30, seed=2024, stream=17)


def _nsga2_case(L, pc, pm, npop, poolsize, popsize, d, seed, stream):
    rng = np.random.default_rng(seed)
    lb, ub = -rng.random(d) - 0.5, 1.0 + rng.random(d)
    pop_x = lb + rng.random((npop, d)) * (ub - lb)
    pop_x[0] = lb
    pop_x[-1] = ub
    pool_idx = rng.permutation(npop)[:poolsize]
    dic, dim = np.full(d, 15.0), np.full(d, 20.0)
    rate = 1.0 / d
    T = int(L.load_library().dmo_nsga2_plan_length(popsize, pc, pm))
    x_gen, kind, dr = L.nsga2_generate(pop_x, pool_idx, popsize, pc, pm, rate, dic, dim, lb, ub, seed=seed, stream_id=stream, return_draws=True)
    rp = replay_plan(seed, stream, T, poolsize, d)
    for k in rp:  # the host restatement of Philox gives the kernel's draws, bit for bit
        assert np.array_equal(rp[k], dr[k]), k
    n_it, kinds, its = nsga2.variation_plan(rp["u_cross"], rp["u_mut"], popsize, pc, pm)
    # the planned iterations are never exhausted (the loop ended at n_it <= T), and T keeps the headroom
    # dmo_nsga2_plan_length claims: 12 standard deviations of the iterations needed for popsize + 1 children,
    # sd = sqrt(var n / e) / e for children per iteration of mean e and variance var (renewal count)
    assert n_it <= T
    e, var, n = 2 * pc + pm, 4 * pc * (1 - pc) + pm * (1 - pm), popsize + 1
    assert T - n / e >= 12 * np.sqrt(var * n / e) / e + 64 or T == 2 * popsize + 64
    P = x_gen.shape[0]
    assert popsize - 1 <= P <= popsize + 1 and P == kinds.size and np.array_equal(kind, kinds)
    pool = pop_x[pool_idx]
    # the oracle loop on the replayed draws (float64, NumPy's pow)
    xo, cidx, midx = nsga2.generate_given_draws(pool, rp["u_cross"], rp["u_mut"], rp["pair"], rp["single"], rp["u_genes"], popsize, dic, dim, lb,
                                                ub, rate, pc, pm)
    assert np.array_equal(np.flatnonzero(kind < 2), cidx) and np.array_equal(np.flatnonzero(kind == 2), midx)
    # every child against the long-double evaluation of its operator
    ref = np.empty((P, d), dtype=LD)
    bnd = np.empty((P, d))
    bnd3 = np.empty((P, d))
    sb = kind == 0
    t = its[sb]
    if t.size:
        r1, b1, r2, b2 = sbx_ref(pool[rp["pair"][t, 0]], pool[rp["pair"][t, 1]], rp["u_genes"][t, 0], dic, lb, ub)
        _, b13, _, b23 = sbx_ref(pool[rp["pair"][t, 0]], pool[rp["pair"][t, 1]], rp["u_genes"][t, 0], dic, lb, ub, pow_ulps=3)
        s2 = np.flatnonzero(sb) + 1
        ref[sb], bnd[sb], bnd3[sb] = r1, b1, b13
        ref[s2], bnd[s2], bnd3[s2] = r2, b2, b23
    mu = kind == 2
    t = its[mu]
    if t.size:
        ref[mu], bnd[mu] = mutation_ref(pool[rp["single"][t]], rp["u_genes"][t, 1], dim, lb, ub, rate)
        bnd3[mu] = mutation_ref(pool[rp["single"][t]], rp["u_genes"][t, 1], dim, lb, ub, rate, pow_ulps=3)[1]
    within(x_gen, ref, bnd)
    within(x_gen, xo, bnd3)


@gpu
def test_nsga2_generate_with_popsize_one_makes_no_children(L):
    """The reference's loop `while count < popsize - 1` does not run for popsize 1."""
    d = 4
    x, kind = L.nsga2_generate(np.random.default_rng(0).random((3, d)), np.arange(3), 1, 0.9, 0.1, 0.25, 1.0, 20.0, np.zeros(d), np.ones(d), 1, 2)
    assert x.shape == (0, d) and kind.shape == (0,)


# ---------------------------------------------------------------------------------------------- tournament
def tournament_uniforms(seed, stream, pop):
    w = philox.draws(seed, stream, philox.P_TOURNAMENT, np.arange(pop, dtype=np.uint64))
    return philox.u01_open(w[0], w[1])


def recovered_order(pool, u):
    """With poolsize == pop the pool is order[top], top depending on the uniforms alone: invert it to read the candidate
    order the kernel sorted."""
    pop = u.shape[0]
    key = np.arange(pop, dtype=np.float64) * np.log(0.5) - np.log(-np.log(u))
    top = np.argsort(-key, kind="stable")
    order = np.empty(pop, dtype=np.int64)
    order[top] = pool
    return order


@gpu
@pytest.mark.parametrize("pop,poolsize", [(1, 1), (2, 2), (5, 1), (300, 300), (2**17 + 3, 2**16), (2**17 + 3, 2**17 + 3)])
def test_tournament_replays_from_philox(L, pop, poolsize):
    rng = np.random.default_rng(pop)
    rank = rng.integers(0, max(1, pop // 50), size=pop)
    crowd = rng.random(pop)
    crowd[rng.random(pop) < 0.1] = np.inf
    seed, stream = 77 + pop, 5
    pool, u = L.tournament(rank, poolsize, seed, stream, crowd=crowd, return_uniforms=True)
    ur = tournament_uniforms(seed, stream, pop)
    assert np.array_equal(u, ur)  # bit for bit
    assert np.array_equal(pool, moea.tournament_selection_gumbel(ur, poolsize, -crowd, rank))
    pool2 = L.tournament(rank, poolsize, seed, stream + 1)
    assert np.array_equal(pool2, moea.tournament_selection_gumbel(tournament_uniforms(seed, stream + 1, pop), poolsize, rank))


@gpu
@pytest.mark.parametrize("case", ["above_pop", "negative", "int32_max", "ties_and_zeros"])
def test_tournament_candidate_order_is_lexsort(L, case):
    rng = np.random.default_rng(3)
    crowd = None
    if case == "above_pop":
        rank = np.array([0, 8, 1, 9])
    elif case == "negative":
        rank = np.array([3, -1, 0, 2, -2**31, 1, -1])
    elif case == "int32_max":
        rank = rng.choice(np.array([0, 1, 2**31 - 1, 2**30, 5000, 2**16]), size=999)
    else:  # many ties, +inf and mixed signed zeros in the crowding key: -0.0 and +0.0 are one key for np.lexsort
        rank = rng.integers(0, 4, size=1000)
        crowd = rng.choice(np.array([0.0, -0.0, np.inf, 1.5, 1.5, 2.0**-1074]), size=1000)
    pop = rank.shape[0]
    pool, u = L.tournament(rank, pop, 11, 3, crowd=crowd, return_uniforms=True)
    expect = np.lexsort((rank,)) if crowd is None else np.lexsort((-crowd, rank))
    assert np.array_equal(recovered_order(pool, u), expect)
    if crowd is not None:  # flipping the sign of every zero changes nothing
        flipped = np.where(crowd == 0, -np.copysign(0.0, crowd), crowd)
        assert np.array_equal(L.tournament(rank, pop, 11, 3, crowd=flipped), pool)


# ---------------------------------------------------------------------------------------------- grouped mutation / SMPSO
def mutate_groups_replay(pop_x, group_size, n_groups, per_group, di, lb, ub, rate, seed, stream, pow_ulps=2, dt=LD):
    d = pop_x.shape[1]
    total = n_groups * per_group
    c = np.arange(total, dtype=np.uint64)
    a = philox.draws(seed, stream, philox.P_MUT_PARENT, c)
    pi = np.minimum(np.floor(philox.u01_53(a[0], a[1]) * float(group_size)).astype(np.int64), group_size - 1)
    prow = (np.arange(total, dtype=np.int64) // per_group) * group_size + pi
    b = philox.draws(seed, stream, philox.P_MUT_GENES, np.arange(total * d, dtype=np.uint64))
    u = philox.u01_53(b[0], b[1]).reshape(total, d)
    if dt is LD:
        ref, bound = mutation_ref(pop_x[prow], u, di, lb, ub, rate, pow_ulps)
    else:  # float64 NumPy (pow within 1 ulp): the kernel may differ by 3 ulp of pow, carried as in mutation_ref
        ref = moea.mutation_u(pop_x[prow], u, di, lb, ub, rate)
        bound = mutation_ref_bound64(pop_x[prow], u, di, lb, ub, rate)
    return prow, ref, bound


def mutation_ref_bound64(parent, u, di, lb, ub, rate):
    e = 1.0 / (np.asarray(di, np.float64) + 1.0)
    lo = u < rate
    P = np.power(np.where(lo, 2.0 * u, 2.0 * (1.0 - u)), e)
    D = np.where(lo, P - 1.0, 1.0 - P)
    W = ub - lb
    Q = W * D
    S = parent + Q
    return (np.abs(W) * (3 * ulp(P) + ulp(D)) + ulp(Q)) + ulp(S)


@gpu
@pytest.mark.parametrize("group_size,n_groups,per_group,d", [(1, 5, 3, 4), (7, 3, 11, 6), (50, 5, 50, 7), (33, 2, 1, 257), (32, 4097, 64, 64)])
def test_mutate_groups_replays_from_philox(L, group_size, n_groups, per_group, d):
    rng = np.random.default_rng(group_size + d)
    lb, ub = -rng.random(d), 1.0 + rng.random(d)
    X = lb + rng.random((group_size * n_groups, d)) * (ub - lb)
    di, rate, seed, stream = rng.uniform(5.0, 30.0, d), 0.3, 123, 9
    out, par = L.mutate_groups(X, group_size, n_groups, per_group, di, lb, ub, rate, seed, stream, return_parents=True)
    big = out.size > 2**24
    prow, ref, bound = mutate_groups_replay(X, group_size, n_groups, per_group, di, lb, ub, rate, seed, stream, dt=np.float64 if big else LD)
    assert np.array_equal(par, prow)
    within(out, ref, bound)


@gpu
@pytest.mark.parametrize("swarms,pop,d", [(1, 1, 1), (3, 17, 5), (5, 64, 30)])
def test_smpso_generate_is_mutate_groups_rounded_to_float32(L, swarms, pop, d):
    rng = np.random.default_rng(swarms * pop)
    lb, ub = -rng.random(d), 1.0 + rng.random(d)
    n = swarms * pop
    parm = (lb + rng.random((n, d)) * (ub - lb)).astype(np.float32).astype(np.float64)
    vel = rng.standard_normal((n, d)) * (ub - lb) * 0.3
    obj = rng.random((n, 2)).astype(np.float32).astype(np.float64)
    sw = L.SmpsoSwarms(parm, obj, vel, swarms, pop)
    di, rate, seed, stream = np.full(d, 20.0), 1.0 / d, 55, 4
    xg = np.asarray(sw.generate(di, lb, ub, rate, seed, stream)).reshape(swarms, 2 * pop, d)
    mut = L.mutate_groups(parm, pop, swarms, pop, di, lb, ub, rate, seed, stream).reshape(swarms, pop, d)
    assert np.array_equal(xg[:, pop:], mut.astype(np.float32).astype(np.float64))  # bit for bit
    moved = np.clip(parm + vel, lb, ub).astype(np.float32).astype(np.float64).reshape(swarms, pop, d)
    assert np.array_equal(xg[:, :pop], moved)


@gpu
@pytest.mark.parametrize("n,d", [(255, 1), (256, 1), (257, 1), (51, 5), (1, 513)])
@pytest.mark.parametrize("f32", [True, False])
def test_smpso_velocity_bit_exact_and_clipped_at_delta(L, n, d, f32):
    rng = np.random.default_rng(n + d)
    lb, ub = -rng.random(d), 1.0 + rng.random(d)
    delta = (ub - lb) / 2
    pos = (lb + rng.random((n, d)) * (ub - lb)).astype(np.float32)
    vel = rng.standard_normal((n, d)) * delta
    # velocities exactly on +-delta, one ulp inside and outside, and far beyond
    edge = np.stack([delta, -delta, np.nextafter(delta, 0), np.nextafter(delta, np.inf), -np.nextafter(delta, np.inf), 3 * delta])
    k = min(n, edge.shape[0])
    vel[:k] = edge[:k]
    l1, l2 = lb + rng.random(d) * (ub - lb), lb + rng.random(d) * (ub - lb)
    if f32:
        l1, l2 = l1.astype(np.float32), l2.astype(np.float32)
    for w, c1, r1, c2, r2, chi in [(1.0, 2.0, 0.0, 2.0, 0.0, 1.0), (0.37, 1.9, 0.61, 2.3, 0.12, 0.8)]:
        out = L.smpso_velocity(pos, vel, l1, l2, w, c1, r1, c2, r2, chi, lb, ub)
        d1 = np.asarray(l1 - pos, dtype=np.float64)  # float32 difference when both are float32 (NumPy promotion)
        d2 = np.asarray(l2 - pos, dtype=np.float64)
        ref = np.clip((w * vel + c1 * r1 * d1 + c2 * r2 * d2) * chi, -delta, delta)
        assert np.array_equal(out.view(np.uint64), ref.view(np.uint64))
        if w == 1.0:  # the pure-velocity case lands on the clip exactly
            assert np.array_equal(out[:k], np.clip(edge[:k], -delta, delta))


# ---------------------------------------------------------------------------------------------- MO-CMA-ES
def exact_pair(rng, n, d):
    """A = D (I + N) with N nonzero only in rows >= h, columns < h (so N^2 = 0) and D a diagonal of powers of two:
    A^-1 = (I - N) D^-1 exactly, every entry a double."""
    h = d // 2
    A, B = np.empty((n, d, d)), np.empty((n, d, d))
    for i in range(n):
        N = np.zeros((d, d))
        N[h:, :h] = np.round(rng.standard_normal((d - h, h)) * 64) / 256
        D = 2.0 ** rng.integers(-1, 2, d)
        A[i] = D[:, None] * (np.eye(d) + N)
        B[i] = (np.eye(d) - N) / D[None, :]
    return A, B


def cholesky_bounds(A, B, pc, z, ps, cc, ccov, pthresh):
    """Long-double update (the oracle's formula on long-double arrays) and a bound on the kernel's float64 result.
    With e_r = (d + 2) eps sum_k |B_rk pc_k| the error of w_r = (Ainv pc)_r (d roundings in any order plus pc's own),
    n2 = sum w^2 is off by dn2 = 2 sum |w| e + d eps n2; b and c are off relatively by dn2 / n2 plus the cancellation in
    root - 1 and 1 - 1/root, 4 eps root / (root - 1); then
      A'_rq    = a A_rq + b pc_r w_q:      3 eps |a A_rq| + |b| (|pc_r| e_q + |w_q| dpc_r + |pc_r w_q| rb) + eps |A'_rq|
      Ainv'_rq = B_rq / a - c w_r wA_q:     3 eps |B_rq / a| + |c| (e_r |wA_q| + |w_r| f_q + |w_r wA_q| rc) + eps |Ainv'_rq|
    with f_q = d eps sum_k |w_k B_kq| + sum_k e_k |B_kq| the error of wA = w Ainv.  The first-order bound is doubled."""
    d = pc.shape[0]
    A2, B2, pc2 = ocm.update_cholesky(A.astype(LD), B.astype(LD), z.astype(LD), ps, pc.astype(LD), cc, ccov, pthresh)
    pcl = np.asarray(pc2, dtype=LD)
    dpc = 3 * EPS * (np.abs((1 - cc) * pc) + np.abs(np.sqrt(cc * (2 - cc)) * z))
    w = (B.astype(LD) @ pcl).astype(np.float64)
    e = (d + 2) * EPS * (np.abs(B) @ np.abs(pcl.astype(np.float64))) + np.abs(B) @ dpc
    if not (w.max() > 1e-20):
        return A2, B2, pc2, 2 * dpc, None, None
    alpha = (1.0 - ccov) if ps < pthresh else (1.0 - ccov) + ccov * cc * (2.0 - cc)
    a = np.sqrt(alpha)
    n2 = float(np.sum(w.astype(LD) ** 2))
    root = np.sqrt(1 + ccov / alpha * n2)
    b = a / n2 * (root - 1)
    c = 1.0 / (a * n2) * (1.0 - 1.0 / root)
    dn2 = 2 * np.sum(np.abs(w) * e) + d * EPS * n2
    rb = dn2 / n2 + 4 * EPS * root / (root - 1) + 4 * EPS
    wA = (w.astype(LD) @ B.astype(LD)).astype(np.float64)
    f = d * EPS * (np.abs(w) @ np.abs(B)) + e @ np.abs(B)
    pcf = pcl.astype(np.float64)
    bA = 3 * EPS * np.abs(a * A) + abs(b) * (np.abs(pcf)[:, None] * e[None, :] + dpc[:, None] * np.abs(w)[None, :] + np.abs(np.outer(pcf, w)) * rb)
    bB = 3 * EPS * np.abs(B / a) + abs(c) * (e[:, None] * np.abs(wA)[None, :] + np.abs(w)[:, None] * f[None, :] + np.abs(np.outer(w, wA)) * rb)
    bA += EPS * np.abs(A2.astype(np.float64))
    bB += EPS * np.abs(B2.astype(np.float64))
    return A2, B2, pc2, 2 * dpc, 2 * bA, 2 * bB


@gpu
@pytest.mark.parametrize("d", [1, 2, 63, 64, 65, 128, 200, 512])
def test_cmaes_update_cholesky_vs_long_double(L, d):
    rng = np.random.default_rng(d)
    n = 4
    A, B = exact_pair(rng, n, d)
    cc, ccov, pthresh = 2.0 / (d + 2), 2.0 / (d * d + 6), 0.44
    pc = rng.standard_normal((n, d)) * 0.3
    z = rng.standard_normal((n, d))
    ps = np.array([0.1, 0.44, 0.9, 0.2])  # both sides of psucc < pthresh, and the threshold itself
    pc[:3], z[:3] = np.abs(pc[:3]), np.abs(z[:3])  # w = Ainv pc has a positive entry (w_k = pc_k / D_k for k < d / 2)
    # individual 3: a w whose entries are all negative (and large): the reference tests w.max(), so nothing moves but pc
    pc[3] = 0.0
    z[3] = -1e3 * (1.0 + rng.random(d))
    A[3], B[3] = np.diag(2.0 ** rng.integers(-1, 2, d)), 0.0
    B[3] = np.diag(1.0 / np.diag(A[3]))
    A2, B2, pc2 = L.cmaes_update_cholesky(A, B, pc, z, ps, cc, ccov, pthresh)
    # device-resident factors give the same bits as host-staged ones
    RA, RB, Rpc = L.resident_rows(A), L.resident_rows(B), L.resident_rows(pc)
    L.cmaes_update_cholesky(RA, RB, Rpc, z, ps, cc, ccov, pthresh)
    assert np.array_equal(np.asarray(RA), A2) and np.array_equal(np.asarray(RB), B2) and np.array_equal(np.asarray(Rpc), pc2)
    for i in range(n):
        rA, rB, rpc, bpc, bA, bB = cholesky_bounds(A[i], B[i], pc[i], z[i], ps[i], cc, ccov, pthresh)
        within(pc2[i], rpc, bpc)
        if bA is None:  # the no-update branch: A and Ainv untouched, bit for bit
            assert i == 3
            assert np.array_equal(A2[i], A[i]) and np.array_equal(B2[i], B[i])
            continue
        assert i != 3
        within(A2[i], rA, bA)
        within(B2[i], rB, bB)
        # invariants in long double, to the first-order effect of the kernel's errors: A' Ainv' = I, and
        # A' A'^T = alpha A A^T + beta pc' pc'^T (A w = pc), off by at most dA |Ainv'| + |A'| dAinv  and  dA |A'^T| + |A'| dA^T
        # (second-order terms dA dAinv and the long-double products' own d 2^-63 |.||.| are added)
        Al, Bl = A2[i].astype(LD), B2[i].astype(LD)
        aA, aB = np.abs(A2[i]), np.abs(B2[i])
        res = np.abs(Al @ Bl - np.eye(d, dtype=LD)).astype(np.float64)
        assert np.all(res <= bA @ aB + aA @ bB + bA @ bB + d * 2.0**-63 * (aA @ aB))
        # with a = sqrt(alpha) rounded to a double and root^2 - 1 = fl(beta / alpha) n2, the exact update gives
        # A' A'^T = a^2 A A^T + a^2 fl(beta / alpha) pc' pc'^T
        alpha = (1.0 - ccov) if ps[i] < pthresh else (1.0 - ccov) + ccov * cc * (2.0 - cc)
        a2 = LD(np.sqrt(alpha)) ** 2
        rhs = a2 * (A[i].astype(LD) @ A[i].T.astype(LD)) + a2 * LD(ccov / alpha) * np.outer(rpc, rpc)
        res = np.abs(Al @ Al.T - rhs).astype(np.float64)
        assert np.all(res <= bA @ aA.T + aA @ bA.T + bA @ bA.T + 2 * d * 2.0**-63 * (aA @ aA.T + np.abs(A[i]) @ np.abs(A[i]).T))
    # pc = 0 with psucc >= pthresh: w = 0, no update either
    pz = np.zeros((1, d))
    A3, B3, pc3 = L.cmaes_update_cholesky(A[:1], B[:1], pz, z[:1], np.array([0.9]), cc, ccov, pthresh)
    assert np.array_equal(A3, A[:1]) and np.array_equal(B3, B[:1]) and np.all(pc3 == 0)


def sample_bound(sg, A, z, pidx):
    """sum_k A_rk z_k in any order, possibly FMA-contracted: d eps sum|terms| on each side (kernel and NumPy); then
    sigma * s and x + sigma s add one ulp each."""
    d = z.shape[1]
    s_abs = np.einsum("ijk,ik->ij", np.abs(A[pidx]), np.abs(z))
    return sg * 2 * d * EPS * s_abs


@gpu
@pytest.mark.parametrize("npar,n,d,cols", [(3, 5, 1, 1), (4, 9, 2, "d"), (7, 300, 65, 1), (5, 64, 512, "d"), (6, 600, 512, 1)])
def test_cmaes_sample_and_generate(L, npar, n, d, cols):
    rng = np.random.default_rng(d + n)
    px = rng.random((npar, d)) - 0.5
    sig = rng.random((npar, d if cols == "d" else 1)) * 0.05 + 0.01
    sig1 = sig if cols == "d" else sig[:, 0]
    A = np.eye(d)[None] + 0.1 * rng.standard_normal((npar, d, d))
    pidx = rng.integers(0, npar, size=n)
    z = rng.standard_normal((n, d))
    z[-1] *= 50.0  # the largest |x| sits in the last row, the end of the grid-stride loop of the abs-max
    sg = sig[pidx] if cols == "d" else sig[pidx][:, :1]
    ind = px[pidx] + sg * np.einsum("ijk,ik->ij", A[pidx], z)
    bound = sample_bound(sg, A, z, pidx) + ulp(sg * np.abs(ind - px[pidx])) + ulp(ind)
    out = L.cmaes_sample(px, sig1, A, pidx, z)
    within(out, ind, bound)
    lb, ub = -1.0 - rng.random(d), 1.0 + rng.random(d)
    x = L.cmaes_generate(px, sig1, L.resident_rows(A), pidx, z, lb, ub)
    # rescale (ind / max|ind|) (ub - lb) + lb, then clip: the max moves by at most max(bound), and each of the three
    # roundings adds one ulp of its result
    mx = np.max(np.abs(ind))
    assert n * d < 4 * L.sm_count() * 256 or np.argmax(np.abs(ind).ravel()) >= 4 * L.sm_count() * 256
    q = ind / mx
    r = q * (ub - lb) + lb
    dq = (bound + np.abs(ind) * np.max(bound) / mx) / mx + ulp(q)
    within(x, np.clip(r, lb, ub), dq * (ub - lb) + ulp(q * (ub - lb)) + ulp(r))


@gpu
def test_scale_rows_with_empty_segments(L):
    rng = np.random.default_rng(4)
    rows = rng.random((6, 5))
    f = rng.uniform(0.5, 2.0, 9)
    seg_row = np.array([0, 2, 3, 5, 1])
    seg_start = np.array([0, 3, 3, 7, 7, 9])  # segments 1 and 3 are empty
    R = L.resident_rows(rows)
    L.scale_rows(R, f, seg_row, seg_start)
    ref = rows.copy()
    for s, r in enumerate(seg_row):
        for e in range(seg_start[s], seg_start[s + 1]):
            ref[r] = ref[r] * f[e]
    assert np.array_equal(np.asarray(R), ref)
    R2 = L.resident_rows(rows)
    L.scale_rows(R2, f[:6])
    assert np.array_equal(np.asarray(R2), rows * f[:6, None])


# ---------------------------------------------------------------------------------------------- AGE-MOEA
def age_rel_bound(M, p):
    """Relative error of one greedy score on each side: the M pow terms 2 eps each, M - 1 additions, then the 1/p-th root
    (which scales the sum's relative error by 1/p, plus 2 eps), the division by nn[s] and the d1 + d2 addition."""
    return (2.0 + (M - 1)) * EPS / p + 4 * EPS


def age_greedy(yn, nn, p, ext, rel):
    """AGEMOEA.py:398-428 in O(m^2): each point keeps its two smallest distances to the selected set.  Asserts that
    every step's maximum is clear of the runner-up by more than both sides' errors, so the selection order is defined."""
    m = yn.shape[0]
    sel = np.zeros(m, dtype=bool)
    crowd = np.zeros(m)
    d1, d2 = np.full(m, np.inf), np.full(m, np.inf)
    q = 1.0 / p

    def update(s):
        nonlocal d1, d2
        dd = np.power(np.power(np.abs(yn - yn[s]), p).sum(axis=1), q) / nn[s]
        d2 = np.where(dd < d1, d1, np.where(dd < d2, dd, d2))
        d1 = np.minimum(d1, dd)

    for s in ext:
        sel[s] = True
        crowd[s] = np.inf
        update(s)
    order = []
    n_sel = len(ext)
    while not sel.all():
        sc = np.where(sel, -np.inf, d1 + d2 if n_sel > 1 else d1)
        j = int(np.argmax(sc))
        if (~sel).sum() > 1:
            runner = np.max(np.delete(sc, j))
            assert sc[j] - runner > 4 * rel * sc[j], "near-tie in the greedy score: choose another front"
        crowd[j] = sc[j]
        sel[j] = True
        order.append(j)
        update(j)
        n_sel += 1
    return crowd, np.array(order, dtype=np.int64)


def age_front(rng, m, M, p):
    yn = rng.random((m, M)) + 0.05
    return yn, np.linalg.norm(yn, p, axis=1)


@pytest.mark.parametrize("m,M", [(40, 2), (120, 3), (200, 5)])
def test_age_greedy_restatement_equals_survival_score(m, M):
    """The O(m^2) greedy the GPU test trusts, against the oracle's O(m^3) survival_score, on the oracle's own
    normalisation of the same front."""
    from oracle import agemoea

    rng = np.random.default_rng(m + M)
    x = rng.random((m, M))
    fy = x / np.linalg.norm(x, axis=1, keepdims=True)
    ideal = fy.min(axis=0)
    yf = fy - ideal
    ext = agemoea.corner_solutions(yf)
    yn = yf / agemoea.hyperplane_normalization(yf, ext)
    p = agemoea.geometry_p(yn, ext)
    rel = age_rel_bound(M, p)
    crowd, _ = age_greedy(yn, np.linalg.norm(yn, p, axis=1), p, ext, rel)
    _, _, cd = agemoea.survival_score(fy, ideal)
    fin = np.isfinite(cd)
    assert np.array_equal(np.isfinite(crowd), fin)
    assert np.all(np.abs(crowd[fin] - cd[fin]) <= 2 * rel * np.abs(cd[fin]))


@gpu
@pytest.mark.parametrize("m,M,p", [(1023, 3, 1.0), (1024, 3, 1.7), (1025, 3, 20.0), (2049, 8, 1.0), (4100, 2, 0.6), (1025, 16, 2.3),
                                   (4100, 16, 1.0), (1025, 2, 20.0), (2049, 3, 1.7)])
def test_age_survival_vs_greedy_past_one_cta(L, m, M, p):
    from oracle import agemoea

    rng = np.random.default_rng(m * 17 + M)
    yn, nn = age_front(rng, m, M, p)
    ext = agemoea.corner_solutions(yn)
    rel = age_rel_bound(M, p)
    ref, _ = age_greedy(yn, nn, p, ext, rel)
    crowd = L.age_survival(yn, nn, p, ext)
    fin = np.isfinite(ref)
    assert np.array_equal(np.isinf(crowd), ~fin)
    # a point selected out of order would carry another step's score: far outside the bound (no near-ties, see above)
    assert np.all(np.abs(crowd[fin] - ref[fin]) <= 2 * rel * ref[fin])


@gpu
@pytest.mark.parametrize("m,M", [(3, 3), (16, 16), (1, 1), (60, 1)])
def test_age_survival_degenerate_fronts(L, m, M):
    rng = np.random.default_rng(m + 100 * M)
    yn, nn = age_front(rng, m, M, 1.0)
    if m == M:  # every row extreme: no greedy step at all
        assert np.all(np.isinf(L.age_survival(yn, nn, 1.0, np.arange(m))))
        return
    ext = np.array([int(np.argmin(yn[:, 0]))])  # a single extreme
    rel = age_rel_bound(M, 1.0)
    ref, _ = age_greedy(yn, nn, 1.0, ext, rel)
    crowd = L.age_survival(yn, nn, 1.0, ext)
    fin = np.isfinite(ref)
    assert np.array_equal(np.isinf(crowd), ~fin)
    assert np.all(np.abs(crowd[fin] - ref[fin]) <= 2 * rel * ref[fin])
