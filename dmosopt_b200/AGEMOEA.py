"""AGE-MOEA optimizer plugin on the GPU path.

Drop-in for ``dmosopt.AGEMOEA.AGEMOEA`` (dmosopt/AGEMOEA.py:24-501), selected by
``optimizer_name="dmosopt_b200.AGEMOEA"``.

Per generation:
  generate_strategy : dmo_tournament on (-crowd_dist, rank) -> dmo_nsga2_generate   (AGEMOEA.py:121-183)
  update_strategy   : vstack(parents, children) -> dmo_get_duplicates -> environmental_selection
                      (AGEMOEA.py:185-229)
environmental_selection (AGEMOEA.py:433-501) keeps the reference's structure; its quadratic parts run on the
GPU -- the non-dominated rank (dmo_rank_nd) and the greedy survival score of the first front
(dmo_age_survival, the m x m distance / m-step arg-max loop of AGEMOEA.py:398-428) -- while the O(m M^2)
bookkeeping (corner solutions, hyperplane intercepts, curvature p, later-front scores) stays in NumPy on the
host exactly as written in the reference.
"""

from typing import Any, Dict, Optional

import numpy as np

from . import _lib
from .MOEA import MOEA, Struct, remove_duplicates
from .NSGA2 import population_diversity


# ---------------------------------------------------------------------------- geometry helpers (host, O(m M^2))
def point_2_line_distance(P, A, B):
    """AGEMOEA.py:342-351, vectorised over the rows of P."""
    pa = P - A
    ba = B - A
    t = (pa @ ba) / np.dot(ba, ba)
    return np.linalg.norm(pa - t[:, None] * ba[None, :], axis=1)


def find_corner_solutions(front):
    """AGEMOEA.py:354-374."""
    m, n = front.shape
    if m <= n:
        return np.arange(m)
    W = 1e-6 + np.eye(n)
    indexes = np.zeros(n, dtype=int)
    selected = np.zeros(m, dtype=bool)
    for i in range(n):
        dists = point_2_line_distance(front, np.zeros(n), W[i, :])
        dists[selected] = np.inf
        index = np.argmin(dists)
        indexes[i] = index
        selected[index] = True
    return indexes


def normalize(front, extreme):
    """AGEMOEA.py:275-315: intercepts of the hyperplane through the extreme points (min-max fallback)."""
    m, n = front.shape
    if len(extreme) != len(np.unique(extreme, axis=0)):
        return np.max(front, axis=0)
    try:
        hyperplane = np.linalg.solve(front[extreme], np.ones(n))
    except Exception:
        hyperplane = np.asarray([np.nan])
    if any(np.isnan(hyperplane)) or any(np.isinf(hyperplane)) or any(hyperplane < 0):
        normalization = np.max(front, axis=0)
    else:
        with np.errstate(divide="ignore"):
            normalization = 1.0 / hyperplane
        if any(np.isnan(normalization)) or any(np.isinf(normalization)):
            normalization = np.max(front, axis=0)
    normalization = np.array(normalization, dtype=np.float64)
    normalization[np.isclose(normalization, 0.0, rtol=1e-4, atol=1e-4)] = 1.0
    return normalization


def get_geometry(front, extreme):
    """AGEMOEA.py:324-339."""
    m, n = front.shape
    d = point_2_line_distance(front, np.zeros(n), np.ones(n))
    d[extreme] = np.inf
    index = np.argmin(d)
    with np.errstate(divide="ignore", invalid="ignore"):
        p = np.log(n) / np.log(1.0 / np.mean(front[index, :]))
    if np.isnan(p) or p <= 0.1:
        p = 1.0
    elif p > 20:
        p = 20.0
    return float(p)


def minkowski_to_point(A, b, p):
    """Row-wise ||A_i - b||_p (AGEMOEA.py:318-321 with a single second point)."""
    return np.power(np.power(np.abs(A - b[None, :]), p).sum(axis=1), 1.0 / p)


def survival_score(y, front, ideal_point):
    """AGEMOEA.py:377-430; the greedy loop runs on the GPU."""
    yfront_raw = y[front, :]
    m, n = yfront_raw.shape
    crowd_dist = np.zeros(m)
    if m < n:
        normalization = np.max(yfront_raw, axis=0).astype(np.float64)
        normalization[np.isclose(normalization, 0.0, rtol=1e-4, atol=1e-4)] = 1.0
        return normalization, 1, crowd_dist
    yfront = yfront_raw - ideal_point
    extreme = find_corner_solutions(yfront)
    normalization = normalize(yfront, extreme)
    ynfront = yfront / normalization
    p = get_geometry(ynfront, extreme)
    nn = np.linalg.norm(ynfront, p, axis=1)
    crowd_dist = _lib.age_survival(ynfront, nn, p, extreme)
    return normalization, p, crowd_dist


def environmental_selection(local_random, population_parm, population_obj, pop, nInput, nOutput, feasibility_model=None, logger=None):
    """AGEMOEA.py:433-501."""
    rank = _lib.rank_nd(population_obj)
    idxr = rank.argsort(kind="stable")  # AGEMOEA.py:267 uses numpy's default (unstable) sort: order inside a front is arbitrary there
    rank = rank[idxr]
    xs = population_parm[idxr, :]
    ys = population_obj[idxr, :]
    rmax = int(np.max(rank))

    yn = np.zeros_like(ys)
    crowd_dist = np.zeros_like(rank).astype(np.float32)
    selected = np.zeros_like(rank).astype(bool)

    # rank is sorted: front r is the contiguous index range [bounds[r], bounds[r + 1]) (= np.argwhere(rank == r))
    bounds = np.searchsorted(rank, np.arange(rmax + 2))
    front_1 = np.arange(bounds[1])
    ideal_point = np.min(ys[front_1, :], axis=0)
    normalization, p, crowd_dist[front_1] = survival_score(ys, front_1, ideal_point)
    yn[front_1, :] = ys[front_1] / normalization

    count = len(front_1)
    if count < pop:
        selected[front_1] = True
        # the reference walks the later fronts one by one (AGEMOEA.py:470-489); their scores are row-wise expressions, so
        # they are evaluated for all later rows at once (rows past the cut keep a score nobody reads)
        rest = slice(int(bounds[1]), len(rank))
        yn[rest] = ys[rest] / normalization
        with np.errstate(divide="ignore"):
            crowd_dist[rest] = 1.0 / minkowski_to_point(yn[rest, :], ideal_point, p)
        for r in range(1, rmax + 1):
            b0, b1 = int(bounds[r]), int(bounds[r + 1])
            if (count + (b1 - b0)) < pop:
                selected[b0:b1] = True
                count += b1 - b0
            else:
                front_r = np.arange(b0, b1)
                sort_keys = []
                if feasibility_model is not None:
                    sort_keys.append(-feasibility_model.rank(xs[front_r]))
                sort_keys.append(-crowd_dist[front_r])
                perm = np.lexsort(sort_keys)
                selected[front_r[perm[: pop - count]]] = True
                break
    else:
        sort_keys = []
        if feasibility_model is not None:
            sort_keys.append(-feasibility_model.rank(xs[front_1]))
        sort_keys.append(-crowd_dist[front_1])
        perm = np.lexsort(sort_keys)
        selected[front_1[perm[:pop]]] = True

    assert np.sum(selected) > 0
    return xs[selected].copy(), ys[selected].copy(), rank[selected].copy(), crowd_dist[selected].copy()


class AGEMOEA(MOEA):
    def __init__(
        self,
        popsize: int,
        nInput: int,
        nOutput: int,
        model: Optional[Any] = None,
        distance_metric: Optional[Any] = None,
        optimize_mean_variance: bool = False,
        feasibility_model: Optional[Any] = None,
        logger=None,
        **kwargs,
    ):
        super().__init__(name="AGEMOEA", popsize=popsize, nInput=nInput, nOutput=nOutput, optimize_mean_variance=optimize_mean_variance, **kwargs)
        self.model = model
        self.logger = logger
        self.feasibility_model = feasibility_model
        self.x_distance_metrics = None
        if feasibility_model is not None:
            self.x_distance_metrics = [feasibility_model.rank]
        p = self.opt_params
        if np.isscalar(p.di_crossover):
            p.di_crossover = np.asarray([p.di_crossover] * nInput)
        if np.isscalar(p.di_mutation):
            p.di_mutation = np.asarray([p.di_mutation] * nInput)
        if p.mutation_rate is None:
            p.mutation_rate = 1.0 / float(nInput)
        p.poolsize = int(round(popsize / 2.0))
        self.optimize_mean_variance = optimize_mean_variance

    @property
    def default_parameters(self) -> Dict[str, Any]:
        """AGEMOEA.py:70-84."""
        return {
            "crossover_prob": 0.9,
            "mutation_prob": 0.1,
            "mutation_rate": None,
            "nchildren": 1,
            "di_crossover": 1.0,
            "di_mutation": 20.0,
            "max_population_size": 2000,
            "min_population_size": 100,
            "adaptive_population_size": False,
        }

    def initialize_state(self, x, y, bounds, local_random=None, **params):
        """AGEMOEA.py:86-119.  As in the reference, the rank / crowd_dist of the selected individuals are kept but
        the stored rows are the first ``popsize`` rows of the raw input (AGEMOEA.py:103-106; SURVEY appendix A)."""
        n = self.opt_params.popsize
        _, _, rank, crowd_dist = environmental_selection(local_random, np.asarray(x), np.asarray(y), n, self.nInput, self.nOutput, logger=self.logger)
        return Struct(bounds=bounds, population_parm=x[:n], population_obj=y[:n], rank=rank[:n], crowd_dist=crowd_dist[:n])

    def generate_strategy(self, **params):
        """AGEMOEA.py:121-183."""
        p, st = self.opt_params, self.state
        xlb, xub = st.bounds[:, 0], st.bounds[:, 1]
        seed = self._rng_seed()
        # tournament_selection(local_random, n, poolsize, -crowd_dist, rank)  (AGEMOEA.py:136-142)
        pool_idxs = _lib.tournament(st.rank, p.poolsize, seed, self._next_stream(), crowd=np.asarray(st.crowd_dist, dtype=np.float64))
        x_gen, kind = _lib.nsga2_generate(
            st.population_parm, pool_idxs, p.popsize, p.crossover_prob, p.mutation_prob, p.mutation_rate,
            p.di_crossover, p.di_mutation, xlb, xub, seed, self._next_stream(),
        )
        return x_gen, {}

    def update_strategy(self, x_gen, y_gen, state, **params):
        """AGEMOEA.py:185-229."""
        st = self.state
        popsize = self.opt_params.popsize
        population_parm = np.vstack((st.population_parm, x_gen))
        population_obj = np.vstack((st.population_obj, y_gen))
        _lib.mirror_drop(x_gen)  # consumed (stacked above): release the HBM copy of the offspring matrix
        population_parm, population_obj = remove_duplicates(population_parm, population_obj)
        population_parm, population_obj, rank, crowd_dist = environmental_selection(
            self.local_random, population_parm, population_obj, popsize, self.nInput, self.nOutput, logger=self.logger
        )
        if self.opt_params.adaptive_population_size:
            st.population_parm, st.population_obj, st.rank, st.crowd_dist = population_parm, population_obj, rank, crowd_dist
            self.update_population_size()
        else:
            st.population_parm[:] = population_parm
            st.population_obj[:] = population_obj
            st.rank[:] = rank
            st.crowd_dist[:] = crowd_dist

    def get_population_strategy(self):
        return self.state.population_parm.copy(), self.state.population_obj.copy()

    def update_population_size(self):
        """AGEMOEA.py:237-258."""
        p = self.opt_params
        diversity, cd_spread = population_diversity(self.state.rank, self.state.population_obj)
        if diversity < 0.5 and cd_spread < 2.0:
            new_size = min(p.max_population_size, int(p.popsize * 1.2))
        elif diversity > 0.9 or cd_spread > 1.0:
            new_size = max(p.min_population_size, int(p.popsize * 0.9))
        else:
            new_size = p.popsize
        p.popsize = new_size
        p.poolsize = int(round(p.popsize / 2.0))
