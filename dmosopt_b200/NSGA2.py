"""NSGA-II optimizer plugin on the GPU path.

Drop-in for ``dmosopt.NSGA2.NSGA2`` (dmosopt/NSGA2.py:18-316): same constructor, parameters, state
fields and ``generate / update`` contract, selected in dmosopt by
``optimizer_name="dmosopt_b200.NSGA2"`` (dmosopt/config.py:5-11, dmosopt/MOASMO.py:256-259).

Per generation (MOASMO.optimize, dmosopt/MOASMO.py:105-116):
  generate_strategy : dmo_tournament -> dmo_nsga2_generate   (NSGA2.py:116-185)
  update_strategy   : dmo_remove_worst on vstack(children, parents)  (NSGA2.py:187-236)
The state lives in NumPy arrays exactly as in the reference (so dmosopt's HDF5 save / restart keeps
working); survivors are written back in place, which rounds the objectives to the state dtype
(float32 inside MOASMO.optimize) just as NSGA2.py:228-230 does.
"""

from typing import Any, Dict, Optional

import numpy as np

from . import _lib
from .MOEA import MOEA, Struct, remove_worst, sortMO


def population_diversity(rank, Y):
    """indicators.PopulationDiversity._do (dmosopt/indicators.py:316-335)."""
    rank = np.asarray(rank).ravel()
    front0 = np.flatnonzero(rank == 0)
    diversity = len(front0) / len(rank)
    D = _lib.crowding_distance(Y)
    if len(front0) > 1:
        cd = D[front0]
        cd_spread = np.std(cd) / np.mean(cd)
    else:
        cd_spread = 0
    return diversity, cd_spread


class NSGA2(MOEA):
    def __init__(
        self,
        popsize: int,
        nInput: int,
        nOutput: int,
        model: Optional[Any],
        distance_metric: Optional[Any] = "crowding",
        optimize_mean_variance: bool = False,
        **kwargs,
    ):
        super().__init__(name="NSGA2", popsize=popsize, nInput=nInput, nOutput=nOutput, optimize_mean_variance=optimize_mean_variance, **kwargs)
        self.model = model
        self.distance_metric = distance_metric
        self.optimize_mean_variance = optimize_mean_variance
        self.y_distance_metrics = None if distance_metric is None else [distance_metric]
        self.x_distance_metrics = None
        if getattr(self.model, "feasibility", None) is not None:
            self.x_distance_metrics = [self.model.feasibility.rank]

        p = self.opt_params
        if np.isscalar(p.di_crossover):
            p.di_crossover = np.asarray([p.di_crossover] * nInput)
        if np.isscalar(p.di_mutation):
            p.di_mutation = np.asarray([p.di_mutation] * nInput)
        if p.mutation_rate is None:
            p.mutation_rate = 1.0 / float(nInput)
        p.poolsize = int(round(p.popsize / 2.0))

    @property
    def default_parameters(self) -> Dict[str, Any]:
        """NSGA2.py:65-82."""
        return {
            "crossover_prob": 0.9,
            "mutation_prob": 0.1,
            "mutation_rate": None,
            "nchildren": 1,
            "di_crossover": 1.0,
            "di_mutation": 20.0,
            "max_population_size": 2000,
            "min_population_size": 100,
            "min_success_rate": 0.2,
            "max_success_rate": 0.75,
            "adaptive_population_size": False,
            "adaptive_operator_rates": False,
        }

    def initialize_state(self, x, y, bounds, local_random=None, **params):
        """NSGA2.py:84-114."""
        x, y, rank, _ = sortMO(x, y, x_distance_metrics=self.x_distance_metrics, y_distance_metrics=self.y_distance_metrics)
        n = self.opt_params.popsize
        # same values / dtypes as the reference's slices.  The parameter matrix is exposed as a read-only view of a
        # page-locked array with a device mirror: generate / update then read and write it in HBM and only the
        # survivors cross the PCIe bus (once, device -> host).  Replacing state.population_parm with an ordinary
        # array simply turns the mirror off.
        px, self._pop_base = _lib.mirrored_readonly(x[:n])
        return Struct(
            bounds=bounds,
            population_parm=px,
            population_obj=y[:n],
            rank=rank[:n],
            successful_crossovers=0,
            total_crossovers=0,
            successful_mutations=0,
            total_mutations=0,
        )

    def generate_strategy(self, **params):
        """NSGA2.py:116-185 (tournament pool, then the crossover / mutation loop planned on the GPU)."""
        p = self.opt_params
        st = self.state
        xlb, xub = st.bounds[:, 0], st.bounds[:, 1]
        seed = self._rng_seed()
        pool_idxs = _lib.tournament(st.rank, p.poolsize, seed, self._next_stream())
        x_gen, kind = _lib.nsga2_generate(
            st.population_parm, pool_idxs, p.popsize, p.crossover_prob, p.mutation_prob, p.mutation_rate,
            p.di_crossover, p.di_mutation, xlb, xub, seed, self._next_stream(),
        )
        crossover_indices = np.flatnonzero(kind < 2)
        mutation_indices = np.flatnonzero(kind == 2)
        st.total_crossovers += len(crossover_indices) // 2
        st.total_mutations += len(mutation_indices)
        return x_gen, {
            "crossover_indices": crossover_indices.astype(int),
            "mutation_indices": mutation_indices.astype(int),
        }

    def update_strategy(self, x_gen, y_gen, state, **params):
        """NSGA2.py:187-236."""
        st = self.state
        popsize = self.opt_params.popsize
        builtin = self.x_distance_metrics is None and (self.y_distance_metrics is None or self.y_distance_metrics[0] in ("crowding", "euclidean"))
        if builtin and not self.opt_params.adaptive_population_size:
            # children stacked over parents (NSGA2.py:205-206) on the device; survivors land directly in the state array
            code = {None: _lib.METRIC_NONE, "crowding": _lib.METRIC_CROWDING, "euclidean": _lib.METRIC_EUCLIDEAN}[
                None if self.y_distance_metrics is None else self.y_distance_metrics[0]]
            base = getattr(self, "_pop_base", None)
            if base is not None and (st.population_parm.ctypes.data != base.ctypes.data or st.population_parm.shape != base.shape):
                base = self._pop_base = None  # the caller replaced the state array
            out_x = base
            if out_x is None and st.population_parm.flags.writeable and st.population_parm.dtype == np.float64 and st.population_parm.shape[0] == popsize:
                out_x = st.population_parm
            population_parm, population_obj, rank, perm = _lib.remove_worst_pair(
                x_gen, y_gen, st.population_parm, st.population_obj, popsize, code, out_X=out_x)
            if population_parm is base:
                population_parm = st.population_parm  # survivors are already in the (mirrored) state array
        else:
            population_parm = np.vstack((x_gen, st.population_parm))
            population_obj = np.vstack((y_gen, st.population_obj))
            population_parm, population_obj, rank, perm = remove_worst(
                population_parm, population_obj, popsize,
                x_distance_metrics=self.x_distance_metrics, y_distance_metrics=self.y_distance_metrics, return_perm=True,
            )
        _lib.mirror_drop(x_gen)  # consumed: the caller may keep the host array, the HBM copy is released
        st.successful_crossovers += np.count_nonzero(np.isin(state["crossover_indices"], perm, assume_unique=True)) / 2
        st.successful_mutations += np.count_nonzero(np.isin(state["mutation_indices"], perm, assume_unique=True))
        if self.opt_params.adaptive_population_size:
            st.population_parm, st.population_obj, st.rank = population_parm, population_obj, rank
            self.update_population_size()
        else:
            if population_parm is not st.population_parm:
                self._store_population(population_parm)
            st.population_obj[:] = population_obj
            st.rank[:] = rank
        if self.opt_params.adaptive_operator_rates:
            self.update_operator_rates()

    def _store_population(self, new):
        """Write a new parameter matrix into the state, keeping the device mirror (if any) coherent."""
        st = self.state
        base = getattr(self, "_pop_base", None)
        if base is not None and st.population_parm.ctypes.data == base.ctypes.data and base.shape == new.shape:
            base[...] = new
            _lib.mirror_upload(base)
        elif st.population_parm.flags.writeable and st.population_parm.shape == new.shape:
            st.population_parm[:] = new
        else:
            st.population_parm = np.array(new, dtype=st.population_parm.dtype)

    def get_population_strategy(self):
        """NSGA2.py:238-242: copies, as in the reference.  The parameter matrix is copied into a recycled page-locked
        buffer (no first-touch page faults on 8*pop*d bytes every generation); the result is an ordinary writable array."""
        return _lib.copy_into_pooled(self.state.population_parm), self.state.population_obj.copy()

    def update_population_size(self):
        """NSGA2.py:244-266."""
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

    def update_operator_rates(self):
        """NSGA2.py:268-316: success-rate driven adaptation of the operator parameters."""
        p, st = self.opt_params, self.state
        if st.total_crossovers > 0:
            rate = st.successful_crossovers / st.total_crossovers
            if rate < p.min_success_rate:
                p.di_crossover = np.maximum(1.0, p.di_crossover * 0.9)
                p.crossover_prob = np.minimum(0.95, p.crossover_prob * 1.1)
            elif rate > p.max_success_rate:
                p.di_crossover = np.minimum(100.0, p.di_crossover * 1.1)
                p.crossover_prob = np.maximum(0.5, p.crossover_prob * 0.9)
        if st.total_mutations > 0:
            rate = st.successful_mutations / st.total_mutations
            if rate < p.min_success_rate:
                p.di_mutation = np.maximum(1.0, p.di_mutation * 0.9)
                p.mutation_prob = np.minimum(1.0 - p.crossover_prob, p.mutation_prob * 1.05)
                p.mutation_rate = np.minimum(0.95, p.mutation_rate * 1.1)
            elif rate > p.max_success_rate:
                p.di_mutation = np.minimum(100.0, p.di_mutation * 1.1)
                p.mutation_prob = np.maximum(0.1, p.mutation_prob * 0.9)
                p.mutation_rate = np.maximum(0.05 / self.nInput, p.mutation_rate * 0.9)
        st.successful_crossovers = st.total_crossovers = 0
        st.successful_mutations = st.total_mutations = 0
