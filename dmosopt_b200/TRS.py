"""Trust-region search optimizer plugin on the GPU path (SURVEY.md section 8f row N4).

Drop-in for ``dmosopt.TRS.TRS`` (dmosopt/TRS.py:36-322), selected by ``optimizer_name="dmosopt_b200.TRS"``.

  generate_strategy  : Sobol perturbations inside per-individual trust regions (scipy's scrambled Sobol sampler driven by
                       the caller's generator, exactly as dmosopt.sampling.sobol; TRS.py:107-153) -- host, O(pop * d)
  select_candidates  : non-dominated rank of offspring + population (dmo_order_mo), whole fronts first, the overflowing
                       front split by the hypervolume-improvement score (dmo_ehvi_select; TRS.py:200-266) -- GPU
  update_state       : success-window driven growth / shrinkage of the trust region (TRS.py:268-291) -- host scalars
"""

from dataclasses import dataclass, field
from typing import Any, Dict, Optional

import numpy as np

from .MOEA import MOEA, Struct, orderMO, remove_duplicates
from .NSGA2 import population_diversity
from .indicators import HypervolumeImprovement


def sobol(n, s, local_random):
    """dmosopt.sampling.SobolDesign (dmosopt/sampling.py:11-22): first n points of a scrambled base-2 Sobol block."""
    from scipy.stats import qmc

    sampler = qmc.Sobol(d=s, scramble=True, seed=local_random)
    m = 10
    while pow(2, m) < n:
        m = m + 1
    return sampler.random_base2(m)[:n]


class SlidingWindow(list):
    """indicators.SlidingWindow (dmosopt/indicators.py:129-142)."""

    def __init__(self, size=None) -> None:
        super().__init__()
        self.size = size

    def append(self, entry):
        super().append(entry)
        if self.size is not None:
            while len(self) > self.size:
                self.pop(0)

    def is_full(self):
        return self.size == len(self)


@dataclass
class TrState:
    """TRS.py:19-33."""

    dim: int
    is_constrained: bool = False
    length: float = 0.05
    length_init: float = 0.1
    length_min: float = 0.00001
    length_max: float = 1.0
    failure_tolerance: int = float("nan")  # post-initialised
    success_tolerance: int = 0.51
    Y_best: np.ndarray = field(default_factory=lambda: np.asarray([np.inf]))
    constraint_violation = float("inf")
    restart: bool = False

    def __post_init__(self):
        self.failure_tolerance = min(1 / self.dim, self.success_tolerance / 2.0)
        self.Y_best = np.asarray([np.inf] * self.dim).reshape((1, -1))


class TRS(MOEA):
    def __init__(self, popsize: int, nInput: int, nOutput: int, model: Optional[Any], optimize_mean_variance: bool = False, **kwargs):
        kwargs.pop("distance_metric", None)  # MOASMO.epoch passes distance_metric=None to every optimizer (MOASMO.py:365-373)
        super().__init__(name="TRS", popsize=popsize, nInput=nInput, nOutput=nOutput, optimize_mean_variance=optimize_mean_variance, **kwargs)
        self.model = model
        self.x_distance_metrics = None
        if getattr(self.model, "feasibility", None) is not None:
            self.x_distance_metrics = [self.model.feasibility.rank]
        self.indicator = HypervolumeImprovement
        self.optimize_mean_variance = optimize_mean_variance

    @property
    def default_parameters(self) -> Dict[str, Any]:
        """TRS.py:65-76."""
        return {
            "nchildren": 1,
            "success_window_size": 64,
            "max_population_size": 600,
            "min_population_size": 100,
            "adaptive_population_size": False,
        }

    def initialize_state(self, x, y, bounds, local_random=None, **params):
        """TRS.py:78-105."""
        n = self.opt_params.popsize
        order, rank, _ = orderMO(x, y, x_distance_metrics=self.x_distance_metrics)
        return Struct(bounds=bounds, population_parm=x[order][:n], population_obj=y[order][:n], rank=rank[:n], tr=TrState(dim=self.nInput),
                      success_window=SlidingWindow(self.opt_params.success_window_size))

    def generate_strategy(self, **params):
        """TRS.py:107-153."""
        popsize = self.opt_params.popsize
        rng = self.local_random
        st = self.state
        xlb, xub = st.bounds[:, 0], st.bounds[:, 1]
        population_parm, population_obj = remove_duplicates(st.population_parm, st.population_obj)
        x_centers = population_parm
        weights = xub - xlb
        weights = weights / np.mean(weights)
        weights = weights / np.prod(np.power(weights, 1.0 / len(weights)))
        tr_lb = np.clip(x_centers - weights * st.tr.length / 2.0, xlb, xub)
        tr_ub = np.clip(x_centers + weights * st.tr.length / 2.0, xlb, xub)
        pert = sobol(x_centers.shape[0], self.nInput, rng)
        pert = tr_lb + (tr_ub - tr_lb) * pert
        prob_perturb = min(20.0 / st.tr.dim, 1.0)
        perturb_mask = rng.random((st.tr.dim,)) <= prob_perturb
        X_cand = x_centers.copy()
        X_cand[:, perturb_mask] = pert[:, perturb_mask]
        if X_cand.shape[0] < popsize:
            sample = sobol(popsize - X_cand.shape[0], self.nInput, rng)
            X_cand = np.vstack((X_cand, xlb + (xub - xlb) * sample))
        return X_cand, {}

    def update_strategy(self, x_gen, y_gen, state, **params):
        """TRS.py:155-192."""
        st = self.state
        candidates_x = np.vstack((x_gen, st.population_parm))
        candidates_y = np.vstack((y_gen, st.population_obj))
        C, P = x_gen.shape[0], st.population_parm.shape[0]
        is_off = np.concatenate((np.ones(C, dtype=bool), np.zeros(P, dtype=bool)))
        population_parm, population_obj, rank = self.update_state(candidates_x, candidates_y, is_off)
        if self.opt_params.adaptive_population_size:
            st.population_parm, st.population_obj, st.rank = population_parm, population_obj, rank
            self.update_population_size()
        else:
            st.population_parm[:] = population_parm
            st.population_obj[:] = population_obj
            st.rank[:] = rank

    def get_population_strategy(self):
        return self.state.population_parm.copy(), self.state.population_obj.copy()

    def select_candidates(self, candidates_x, candidates_y):
        """TRS.py:200-266: rank on the GPU, fronts filled in rank order, the split front by HV improvement.  (The early
        return of the reference has two values where its caller unpacks three, TRS.py:205-208; three are returned here.)"""
        popsize = self.opt_params.popsize
        n = candidates_x.shape[0]
        order, rank, _ = orderMO(candidates_x, candidates_y, x_distance_metrics=self.x_distance_metrics)
        if n <= popsize:
            full_rank = np.empty(n, dtype=rank.dtype)
            full_rank[order] = rank
            return np.ones(n, dtype=bool), np.zeros(n, dtype=bool), full_rank
        # NB orderMO returns rank[perm] (ranks in sorted order) and the reference indexes candidates with the positions of
        # ``rank == r`` in that array mapped through argsort(order) (TRS.py:213, 226): reproduced as written
        order_inv = np.empty(n, dtype=np.intp)  # np.argsort(order): the inverse permutation
        order_inv[order] = np.arange(n)
        chosen = np.zeros(n, dtype=bool)
        not_chosen = np.zeros(n, dtype=bool)
        mid_front = None
        full = False
        chosen_count = 0
        bounds_r = np.searchsorted(rank, np.arange(int(np.max(rank)) + 2))  # rank is ascending here (orderMO returns rank[perm])
        for r in range(int(np.max(rank)) + 1):
            front_r = order_inv[bounds_r[r] : bounds_r[r + 1]]  # order_inv[np.argwhere(rank == r)], TRS.py:226 (sic)
            if chosen_count + len(front_r) <= popsize and not full:
                chosen[front_r] = True
                chosen_count += len(front_r)
            elif mid_front is None and chosen_count < popsize:
                mid_front = front_r.copy()
                full = True
            else:
                not_chosen[front_r] = True
        k = popsize - chosen_count
        if k > 0:
            ref = np.max(candidates_y, axis=0) + 1
            indicator = self.indicator(ref_point=ref, nds=True)
            assert len(mid_front) > 0
            if chosen_count > 0:
                selected = indicator.do(candidates_y[chosen], candidates_y[mid_front], np.ones_like(candidates_y[mid_front, :]), k)
            else:
                selected = np.arange(k)
            assert len(selected) == k
            chosen[mid_front[selected]] = True
            mask = np.ones(len(mid_front), bool)
            mask[selected] = False
            not_chosen[mid_front[mask]] = True
        return chosen, not_chosen, rank[chosen]

    def update_state(self, X_next, Y_next, is_offspring):
        """TRS.py:268-291."""
        tr = self.state.tr
        if tr.restart:
            self.restart_state()
        chosen, not_chosen, chosen_rank = self.select_candidates(X_next, Y_next)
        success_counter = np.count_nonzero(np.logical_and(is_offspring, chosen))
        self.state.success_window.append(success_counter)
        success_mean = np.mean(self.state.success_window[:])
        success_frac = min(1.0, success_mean / self.opt_params.popsize)
        if success_frac > tr.success_tolerance:
            tr.length = min((1.0 + (success_frac - tr.success_tolerance)) * tr.length, tr.length_max)
            tr.success_counter = 0
        elif success_frac <= tr.failure_tolerance:
            tr.length /= 2.0
            tr.success_counter = 0
        if tr.length < tr.length_min:
            tr.restart = True
        return X_next[chosen], Y_next[chosen], chosen_rank

    def restart_state(self):
        """TRS.py:293-299."""
        tr = self.state.tr
        tr.failure_counter = 0
        tr.length = tr.length_init
        tr.Y_best = np.asarray([np.inf] * tr.dim).reshape((1, -1))
        tr.restart = False
        self.state.success_window = SlidingWindow(self.opt_params.success_window_size)

    def update_population_size(self):
        """TRS.py:301-322."""
        p = self.opt_params
        diversity, cd_spread = population_diversity(self.state.rank, self.state.population_obj)
        if diversity < 0.1 or cd_spread < 2.0:
            new_size = min(p.max_population_size, int(p.popsize * 1.1))
        elif diversity > 0.4 and cd_spread > 1.0:
            new_size = max(p.min_population_size, int(p.popsize * 0.9))
        else:
            new_size = p.popsize
        p.popsize = new_size
