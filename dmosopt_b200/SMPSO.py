"""SMPSO optimizer plugin on the GPU path.

Drop-in for ``dmosopt.SMPSO.SMPSO`` (dmosopt/SMPSO.py:19-348), selected by
``optimizer_name="dmosopt_b200.SMPSO"``.  ``swarm_size`` independent swarms of ``popsize`` particles:

  generate_strategy : positions clip(x + v) of every particle, then ``popsize`` polynomial mutants per swarm
                      (dmo_mutate_groups; SMPSO.py:143-185)
  update_strategy   : per swarm -- crowding of the swarm's slice of y_gen (dmo_crowding_distance), velocity update
                      (dmo_smpso_velocity; SMPSO.py:316-348), then remove_worst of vstack(children, particles)
                      (dmo_remove_worst; SMPSO.py:187-238)

Reference behaviour that is reproduced deliberately (SURVEY.md section 8a row A12): ``x_gen`` is laid out swarm-major
with 2*popsize rows per swarm, but ``update_strategy`` consumes it with the popsize-wide slices
``range(p*popsize, (p+1)*popsize)`` -- swarm p therefore sees rows p*popsize..(p+1)*popsize of the 10*popsize-row
array and the second half of x_gen is evaluated but never used.  The scalar draws of velocity_vector (r1, r2, w,
c1, c2 and the two leader indices) are taken from the caller's NumPy generator in the reference's order, so the
velocity update is reproduced exactly for a given generator state.
"""

from typing import Any, Dict, Optional

import numpy as np

from . import _lib
from .MOEA import MOEA, Struct, remove_duplicates, remove_worst, sortMO
from .NSGA2 import population_diversity


def update_position(parameters, velocity, xlb, xub):
    """SMPSO.py:311-313."""
    return np.clip(parameters + velocity, xlb, xub)


def velocity_vector(local_random, position, velocity, archive, crowding, xlb, xub):
    """SMPSO.py:316-348: scalar draws on the host (reference order), arithmetic on the GPU."""
    r1 = local_random.uniform(low=0.0, high=1.0, size=1)[0]
    r2 = local_random.uniform(low=0.0, high=1.0, size=1)[0]
    w = local_random.uniform(low=0.1, high=0.5, size=1)[0]
    c1 = local_random.uniform(low=1.5, high=2.5, size=1)[0]
    c2 = local_random.uniform(low=1.5, high=2.5, size=1)[0]
    phi = c1 + c2 if c1 + c2 > 4 else 0
    chi = 2 / (2 - phi - ((phi**2) - 4 * phi) ** (1 / 2))
    if archive.shape[0] > 2:
        ind_1, ind_2 = local_random.integers(low=0, high=archive.shape[0], size=2)
        if crowding[ind_1] < crowding[ind_2]:
            ind_1, ind_2 = ind_2, ind_1
    else:
        ind_1 = ind_2 = 0
    return _lib.smpso_velocity(position, velocity, archive[ind_1], archive[ind_2], w, c1, r1, c2, r2, chi, xlb, xub)


class SMPSO(MOEA):
    def __init__(
        self,
        popsize: int,
        nInput: int,
        nOutput: int,
        model: Optional[Any],
        distance_metric: Optional[Any] = None,
        optimize_mean_variance: bool = False,
        **kwargs,
    ):
        swarm_size = kwargs.get("swarm_size", self.default_parameters["swarm_size"])
        kwargs["initial_size"] = popsize * swarm_size  # SMPSO.py:36
        super().__init__(name="SMPSO", popsize=popsize, nInput=nInput, nOutput=nOutput, optimize_mean_variance=optimize_mean_variance, **kwargs)
        self.pop_slices = [range(p * popsize, (p + 1) * popsize) for p in range(swarm_size)]
        self.model = model
        self.distance_metric = distance_metric
        self.y_distance_metrics = None if distance_metric is None else [distance_metric]
        # NB the reference assigns the feasibility metric to a local and leaves this None (SMPSO.py:56-58)
        self.x_distance_metrics = None
        p = self.opt_params
        if np.isscalar(p.di_mutation):
            p.di_mutation = np.asarray([p.di_mutation] * nInput)
        if p.mutation_rate is None:
            p.mutation_rate = 1.0 / float(nInput)
        self.optimize_mean_variance = optimize_mean_variance

    @property
    def default_parameters(self) -> Dict[str, Any]:
        """SMPSO.py:68-83."""
        return {
            "mutation_rate": None,
            "nchildren": 1,
            "swarm_size": 5,
            "di_mutation": 20.0,
            "max_population_size": 2000,
            "min_population_size": 100,
            "min_success_rate": 0.2,
            "max_success_rate": 0.75,
            "adaptive_population_size": False,
            "adaptive_operator_rates": False,
        }

    def initialize_state(self, x, y, bounds, local_random=None, **params):
        """SMPSO.py:87-141."""
        popsize, swarm_size = self.opt_params.popsize, self.opt_params.swarm_size
        xlb, xub = bounds[:, 0], bounds[:, 1]
        population_parm = np.zeros((swarm_size * popsize, self.nInput), dtype=np.float32)
        population_obj = np.zeros((swarm_size * popsize, self.nOutput), dtype=np.float32)
        velocity = local_random.uniform(size=(swarm_size * popsize, self.nInput)) * (xub - xlb) + xlb
        ranks = []
        for sl in self.pop_slices:
            xs, ys, rank_p, _ = sortMO(
                x[sl].astype(np.float32), y[sl].astype(np.float32),
                x_distance_metrics=self.x_distance_metrics, y_distance_metrics=self.y_distance_metrics,
            )
            population_parm[sl] = xs[:popsize]
            population_obj[sl] = ys[:popsize]
            ranks.append(rank_p)
        self._swarms = None  # device-resident copy of (population_parm, population_obj, velocity), built on first use
        # page-locked state arrays (same dtypes / values): the per-generation state read-back is a DMA, not a staged copy
        population_parm, population_obj, velocity = _lib.pinned_like(population_parm), _lib.pinned_like(population_obj), _lib.pinned_like(velocity)
        return Struct(bounds=bounds, population_parm=population_parm, population_obj=population_obj, ranks=ranks,
                      velocity=velocity, successful_children=0)

    # ---- resident swarm state (csrc/smpso.cu).  The NumPy state arrays stay the interface (dmosopt reads and saves
    # them); the device copy is rebuilt whenever the caller has replaced or resized them.
    def _resident(self):
        st, p = self.state, self.opt_params
        if p.adaptive_population_size or getattr(_lib, "SmpsoSwarms", None) is None or self.x_distance_metrics is not None:
            return None
        if self.y_distance_metrics is not None and self.y_distance_metrics[0] not in ("crowding", "euclidean"):
            return None
        sw = getattr(self, "_swarms", None)
        key = (id(st.population_parm), id(st.population_obj), id(st.velocity), st.population_parm.shape)
        if sw is None or getattr(self, "_swarms_key", None) != key:
            sw = self._swarms = _lib.SmpsoSwarms(st.population_parm, st.population_obj, st.velocity, p.swarm_size, p.popsize)
            self._swarms_key = key
        return sw

    def generate_strategy(self, **params):
        """SMPSO.py:143-185."""
        p, st = self.opt_params, self.state
        popsize, swarm_size = p.popsize, p.swarm_size
        xlb, xub = st.bounds[:, 0], st.bounds[:, 1]
        seed = self._rng_seed()
        sw = self._resident()
        if sw is not None:  # one kernel: moved positions and mutants of every swarm, float32 out
            return sw.generate(p.di_mutation, xlb, xub, p.mutation_rate, seed, self._next_stream()), {}
        mutants = _lib.mutate_groups(st.population_parm, popsize, swarm_size, popsize, p.di_mutation, xlb, xub,
                                     p.mutation_rate, seed, self._next_stream())
        blocks = []
        for k, sl in enumerate(self.pop_slices):
            blocks.append(update_position(st.population_parm[sl], st.velocity[sl], xlb, xub))
            blocks.append(mutants[k * popsize : (k + 1) * popsize])
        return np.vstack(blocks).astype(np.float32), {}

    def update_strategy(self, x_gen, y_gen, state, **params):
        """SMPSO.py:187-238."""
        st = self.state
        popsize = self.opt_params.popsize
        xlb, xub = st.bounds[:, 0], st.bounds[:, 1]
        sw = self._resident()
        if sw is not None:
            self._update_resident(sw, x_gen, y_gen, xlb, xub)
            if self.opt_params.adaptive_operator_rates:
                self.update_operator_rates()
            return
        for sl in self.pop_slices:
            D = _lib.crowding_distance(y_gen[sl])
            st.velocity[sl] = velocity_vector(self.local_random, st.population_parm[sl], st.velocity[sl], x_gen[sl], D, xlb, xub)
        total_children = x_gen.shape[0]
        for k, sl in enumerate(self.pop_slices):
            parm_p = np.vstack((x_gen[sl], st.population_parm[sl]))
            obj_p = np.vstack((y_gen[sl], st.population_obj[sl]))
            st.population_parm[sl], st.population_obj[sl], st.ranks[k], perm = remove_worst(
                parm_p, obj_p, popsize, x_distance_metrics=self.x_distance_metrics,
                y_distance_metrics=self.y_distance_metrics, return_perm=True,
            )
            surviving = np.isin(np.arange(total_children), perm, assume_unique=True)
            st.successful_children += np.count_nonzero(surviving)
        if self.opt_params.adaptive_population_size:
            self.update_population_size()
        if self.opt_params.adaptive_operator_rates:
            self.update_operator_rates()

    def _update_resident(self, sw, x_gen, y_gen, xlb, xub):
        """update_strategy with the swarm state in HBM: the scalar draws of velocity_vector are taken from the caller's
        generator in the reference's order (SMPSO.py:317-331, one swarm after the other), everything else is one call."""
        st, p = self.state, self.opt_params
        S, popsize = p.swarm_size, p.popsize
        rng = self.local_random
        sc = np.zeros((S, 8))
        for k in range(S):
            r1 = rng.uniform(low=0.0, high=1.0, size=1)[0]
            r2 = rng.uniform(low=0.0, high=1.0, size=1)[0]
            w = rng.uniform(low=0.1, high=0.5, size=1)[0]
            c1 = rng.uniform(low=1.5, high=2.5, size=1)[0]
            c2 = rng.uniform(low=1.5, high=2.5, size=1)[0]
            phi = c1 + c2 if c1 + c2 > 4 else 0
            chi = 2 / (2 - phi - ((phi**2) - 4 * phi) ** (1 / 2))
            if popsize > 2:
                ind_1, ind_2 = rng.integers(low=0, high=popsize, size=2)
            else:
                ind_1 = ind_2 = -1
            sc[k] = (w, c1, r1, c2, r2, chi, ind_1, ind_2)
        code = {None: _lib.METRIC_NONE, "crowding": _lib.METRIC_CROWDING, "euclidean": _lib.METRIC_EUCLIDEAN}[
            None if self.y_distance_metrics is None else self.y_distance_metrics[0]]
        ranks, perm = sw.update(x_gen, y_gen, sc, xlb, xub, code, st.population_parm, st.population_obj)
        sw.velocity_into(st.velocity)
        _lib.mirror_drop(x_gen)  # consumed: the HBM copy of the offspring matrix is released
        total_children = np.asarray(x_gen).shape[0]
        for k in range(S):
            st.ranks[k] = ranks[k]
            # np.isin(arange(total_children), perm): how many of the kept rows are indices below total_children -- all of them
            # (perm indexes the swarm's 2 * popsize stacked rows and total_children = 2 * swarm_size * popsize), as in SMPSO.py:231-233
            st.successful_children += int(np.count_nonzero(np.isin(np.arange(total_children), perm[k], assume_unique=True)))

    def get_population_strategy(self):
        """SMPSO.py:240-258 (the reference returns the de-duplicated population, not the truncated one)."""
        pop_parm, pop_obj = remove_duplicates(self.state.population_parm.copy(), self.state.population_obj.copy())
        return pop_parm, pop_obj

    def update_population_size(self):
        """SMPSO.py:260-287."""
        p = self.opt_params
        ranks = np.concatenate(self.state.ranks)
        diversity, cd_spread = population_diversity(ranks, self.state.population_obj)
        if diversity < 0.5 and cd_spread < 2.0:
            new_size = min(p.max_population_size, int(p.popsize * 1.2))
        elif diversity > 0.9 or cd_spread > 1.0:
            new_size = max(p.min_population_size, int(p.popsize * 0.9))
        else:
            new_size = p.popsize
        p.popsize = new_size
        self.pop_slices = [range(k * new_size, (k + 1) * new_size) for k in range(p.swarm_size)]

    def update_operator_rates(self):
        """SMPSO.py:289-308."""
        p, st = self.opt_params, self.state
        rate = st.successful_children / (p.popsize * p.swarm_size)
        if rate < p.min_success_rate:
            p.di_mutation = np.maximum(1.0, p.di_mutation * 0.9)
            p.mutation_rate = np.minimum(0.95, p.mutation_rate * 1.1)
        elif rate > p.max_success_rate:
            p.di_mutation = np.minimum(100.0, p.di_mutation * 1.1)
            p.mutation_rate = np.maximum(0.05 / self.nInput, p.mutation_rate * 0.9)
        st.successful_children = 0
