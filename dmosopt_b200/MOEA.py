"""Host-side mirror of dmosopt's MOEA plugin surface, backed by the CUDA library.

Mirrors ``dmosopt/MOEA.py`` (reference @ 5cd63e4c):
  * ``Struct``                       MOEA.py:26-52
  * ``MOEA`` base class              MOEA.py:55-188   (same constructor / method contract, so the
                                     subclasses here are drop-in ``optimizer_name`` targets for
                                     MOASMO.epoch, dmosopt/MOASMO.py:256-259, 365-373)
  * ``sortMO / orderMO / remove_worst``  MOEA.py:242-347, 398-423  -> dmo_order_mo / dmo_remove_worst
  * ``tournament_selection``         MOEA.py:375-395  -> dmo_tournament (log-space, scales past pop 2150)
  * ``mutation / crossover_sbx``     MOEA.py:191-239  -> dmo_mutation_u / dmo_sbx_u
  * ``get_duplicates / remove_duplicates``  MOEA.py:426-442 -> dmo_get_duplicates
  * ``EpsilonSort``                  MOEA.py:470-595  -> dmo_epsilon_sort (rows buffered, resolved in one call)

All numerical work happens on the GPU through ``_lib``; this module only adapts shapes, dtypes and
the reference's calling conventions.
"""

import math
from typing import Any, Dict, Optional, Tuple

import numpy as np

from . import _lib



def crowding_distance_metric(Y):
    """indicators.crowding_distance_metric (dmosopt/indicators.py:12-51), re-exported like the reference's MOEA module does."""
    return _lib.crowding_distance(Y)


def euclidean_distance_metric(Y):
    """indicators.euclidean_distance_metric (dmosopt/indicators.py:54-62)."""
    return _lib.euclidean_distance(Y)


MAX_OBJECTIVES = 16  # dmo_rank_nd / dmo_crowding_distance / dmo_age_survival / dmo_ehvi_select (exact hypervolume: 8, _lib.HV_MAX_OBJECTIVES)

_METRIC_CODES = {None: _lib.METRIC_NONE, "crowding": _lib.METRIC_CROWDING, "euclidean": _lib.METRIC_EUCLIDEAN}


class Struct(object):
    """Attribute bag used for optimizer parameters and state (MOEA.py:26-52)."""

    def __init__(self, **items):
        self.__dict__.update(items)

    def update(self, items):
        self.__dict__.update(items)

    def items(self):
        return self.__dict__.items()

    def __call__(self):
        return self.__dict__

    def __getitem__(self, key):
        return self.__dict__[key]

    def __setitem__(self, key, val):
        self.__dict__[key] = val

    def __contains__(self, k):
        return k in self.__dict__

    def __repr__(self):
        return f"Struct({self.__dict__})"

    def __str__(self):
        return "<Struct>"


def _initial_design(n, d, local_random, method=None):
    """Latin-hypercube (default) or Sobol initial design in [0,1]^d (MOEA.generate_initial, MOEA.py:118-143).

    The reference delegates to dmosopt.sampling.lh / sobol (scipy.stats.qmc); the same scipy samplers
    are used here.  This runs once per epoch and is not part of the accelerated path.
    """
    from scipy.stats import qmc

    if method == "sobol":
        return qmc.Sobol(d=d, scramble=True, seed=local_random).random(n)
    return qmc.LatinHypercube(d=d, seed=local_random).random(n)


class MOEA(object):
    """Base class of the GPU optimizer plugins; same contract as dmosopt.MOEA.MOEA (MOEA.py:55-188)."""

    def __init__(self, name: str, popsize: int, nInput: int, nOutput: int, **kwargs):
        doubled = bool(kwargs.pop("optimize_mean_variance", False))  # not an optimizer parameter: only sizes the check below
        self.name = name
        self.popsize = popsize
        self.nInput = nInput
        self.nOutput = nOutput
        self.opt_params = Struct(**self.default_parameters)
        self.opt_params.update(
            {
                "popsize": popsize,
                "nInput": nInput,
                "nOutput": nOutput,
                "initial_size": popsize,
                "initial_sampling_method": None,
                "initial_sampling_method_params": None,
            }
        )
        for k, v in kwargs.items():
            if k not in self.opt_params or v is not None:
                self.opt_params[k] = v
        self.local_random = None
        self.state = None
        # limits of the kernels, checked before an epoch starts rather than at the first sortMO (csrc/rank.cu, sortmo.cu:
        # records and per-objective tables are sized for at most 16 objectives; optimize_mean_variance doubles the count)
        n_sorted = nOutput * (2 if doubled else 1)
        if n_sorted > MAX_OBJECTIVES:
            raise ValueError(f"dmosopt_b200.{name}: {n_sorted} objectives to sort (nOutput={nOutput}"
                             f"{', doubled by optimize_mean_variance' if n_sorted != nOutput else ''}); the rank / crowding kernels take at most {MAX_OBJECTIVES}")

    @property
    def default_parameters(self) -> Dict[str, Any]:
        return {}

    @property
    def opt_parameters(self) -> Dict[str, Any]:
        return self.opt_params()

    @property
    def population_objectives(self) -> Tuple[np.ndarray, np.ndarray]:
        return self.get_population_strategy()

    def get_population_strategy(self):
        raise NotImplementedError

    def initialize_strategy(self, x, y, bounds, local_random: Optional[np.random.Generator] = None, **params):
        self.bounds = bounds
        self.local_random = local_random
        self.state = self.initialize_state(x, y, bounds, local_random)
        return self.state

    def generate_initial(self, bounds, local_random):
        xlb, xub = bounds[:, 0], bounds[:, 1]
        n = self.opt_params.initial_size
        method = self.opt_params.initial_sampling_method
        params = self.opt_params.initial_sampling_method_params
        if method is None or method == "sobol":
            return _initial_design(n, self.nInput, local_random, method) * (xub - xlb) + xlb
        if callable(method):
            if params is None:
                return method(local_random, n, self.nInput, xlb, xub)
            return method(local_random, **params)
        raise RuntimeError(f"Unknown sampling method {method}")

    def generate(self, **params):
        x, state = self.generate_strategy(**params)
        lb, ub = self.bounds[:, 0], self.bounds[:, 1]
        if isinstance(x, np.ndarray) and not x.flags.writeable and _lib.mirror_ptr(x) is not None:
            # offspring produced by the variation kernels are already clamped to these bounds on the device
            # (variation.cu, same [xlb, xub] as MOEA.py:155); the read-only array keeps its device mirror
            return x, state
        if isinstance(x, np.ndarray) and x.dtype == np.float64 and x.flags.writeable:
            return np.clip(x, lb, ub, out=x), state  # same values as MOEA.py:155, without a second 8*P*d byte buffer
        return np.clip(x, lb, ub), state

    def update(self, x, y, state, **params):
        self.update_strategy(x, y, state, **params)
        return self.state

    def initialize_state(self, *args, **params):
        raise NotImplementedError

    def generate_strategy(self, **params):
        raise NotImplementedError

    def update_strategy(self, x, y, state, **params):
        raise NotImplementedError

    # ---- Philox stream bookkeeping: the seed is drawn once from the caller's NumPy generator
    # (MOASMO.py:51-52 owns it), so a run stays reproducible from dmosopt's ``random_seed``.
    def _rng_seed(self):
        if getattr(self, "_philox_seed", None) is None:
            rng = self.local_random if self.local_random is not None else np.random.default_rng()
            self._philox_seed = int(rng.integers(0, 2**63 - 1))
            self._philox_stream = 0
        return self._philox_seed

    def _next_stream(self):
        self._rng_seed()
        self._philox_stream += 1
        return self._philox_stream


# ----------------------------------------------------------------------------- metric plumbing
def _split_metrics(y_distance_metrics, y):
    """Built-in string metrics run on the GPU; callables are evaluated on the host and passed as keys."""
    code = _lib.METRIC_NONE
    host_keys = []
    if y_distance_metrics is not None:
        assert len(y_distance_metrics) > 0
        for m in y_distance_metrics:
            if callable(m):
                host_keys.append(np.asarray(m(y), dtype=np.float64))
            elif m in ("crowding", "euclidean"):
                if code != _lib.METRIC_NONE or host_keys:
                    # several y metrics: evaluate the extra built-in ones through the GPU functions, keep order
                    host_keys.append(_lib.crowding_distance(y) if m == "crowding" else _lib.euclidean_distance(y))
                else:
                    code = _METRIC_CODES[m]
            else:
                raise RuntimeError(f"sortMO: unknown distance metric {m}")
    return code, host_keys


def orderMO(x, y, x_distance_metrics=None, y_distance_metrics=None):
    """MOEA.orderMO (MOEA.py:300-347): (perm, rank[perm], y_dists[perm])."""
    y = np.asarray(y)
    code, ykeys = _split_metrics(y_distance_metrics, y)
    xkeys = []
    if x_distance_metrics is not None:
        for m in x_distance_metrics:
            if not callable(m):
                raise RuntimeError(f"sortMO: unknown distance metric {m}")
            xkeys.append(np.asarray(m(x), dtype=np.float64))
    if ykeys:
        # lexsort order: x metrics (least significant), then y metrics in list order, then rank.
        # The single GPU metric slot sits between the extras and the rank, so with host-evaluated
        # y metrics present everything is passed as extra keys.
        if code != _lib.METRIC_NONE:
            first = _lib.crowding_distance(y) if code == _lib.METRIC_CROWDING else _lib.euclidean_distance(y)
            ykeys = [first] + ykeys
            code = _lib.METRIC_NONE
        perm, rank, _ = _lib.order_mo(y, _lib.METRIC_NONE, xkeys + ykeys)
        return perm, rank, tuple(k[perm] for k in ykeys)
    perm, rank, dist = _lib.order_mo(y, code, xkeys)
    return perm, rank, (() if dist is None else (dist,))


def sortMO(x, y, return_perm=False, x_distance_metrics=None, y_distance_metrics=None):
    """MOEA.sortMO (MOEA.py:242-297)."""
    x = np.asarray(x)
    y = np.asarray(y)
    perm, rank, dists = orderMO(x, y, x_distance_metrics, y_distance_metrics)
    if return_perm:
        return x[perm], y[perm], rank, dists, perm
    return x[perm], y[perm], rank, dists


def remove_worst(population_parm, population_obj, pop, x_distance_metrics=None, y_distance_metrics=None, return_perm=False):
    """MOEA.remove_worst (MOEA.py:398-423): the first ``pop`` rows of the sortMO order."""
    x = np.asarray(population_parm)
    y = np.asarray(population_obj)
    code, ykeys = _split_metrics(y_distance_metrics, y)
    if ykeys or x_distance_metrics is not None:
        perm, rank, _ = orderMO(x, y, x_distance_metrics, y_distance_metrics)
        perm = perm[:pop]
        res = (x[perm], y[perm], rank[:pop])
        return res + (perm,) if return_perm else res
    xs, ys, rank, perm = _lib.remove_worst(x, y, pop, code)
    # the gathered rows keep the callers' dtypes (the reference indexes the stacked arrays)
    xs = xs.astype(x.dtype, copy=False)
    ys = ys.astype(y.dtype, copy=False)
    return (xs, ys, rank, perm) if return_perm else (xs, ys, rank)


def tournament_selection(local_random, pop, poolsize, *metrics, seed=None, stream_id=0):
    """MOEA.tournament_selection (MOEA.py:375-395).

    ``metrics`` are lexsort keys, last one primary: ``(rank,)`` for NSGA-II, ``(-crowd_dist, rank)``
    for AGE-MOEA.  The Philox seed is drawn from ``local_random`` unless given.
    """
    if seed is None:
        seed = int(local_random.integers(0, 2**63 - 1))
    rank = np.asarray(metrics[-1])
    crowd = None
    if len(metrics) == 2:
        crowd = -np.asarray(metrics[0], dtype=np.float64)  # the reference passes -crowd_dist
    elif len(metrics) != 1:
        raise RuntimeError("tournament_selection: expected (rank,) or (-crowd_dist, rank)")
    return _lib.tournament(rank, poolsize, seed, stream_id, crowd=crowd)


def mutation(local_random, parent, di_mutation, xlb, xub, mutation_rate=0.5, nchildren=1):
    """MOEA.mutation (MOEA.py:191-212); the uniforms come from ``local_random`` exactly as in the reference."""
    parent = np.asarray(parent, dtype=np.float64)
    n = parent.shape[0]
    u = np.vstack([local_random.random(n) for _ in range(nchildren)])
    return _lib.mutation_u(np.broadcast_to(parent, (nchildren, n)), u, di_mutation, xlb, xub, mutation_rate)


def crossover_sbx(local_random, parent1, parent2, di_crossover, xlb, xub, nchildren=1):
    """MOEA.crossover_sbx (MOEA.py:215-239)."""
    p1 = np.asarray(parent1, dtype=np.float64)
    p2 = np.asarray(parent2, dtype=np.float64)
    n = p1.shape[0]
    u = np.vstack([local_random.random(n) for _ in range(nchildren)])
    return _lib.sbx_u(np.broadcast_to(p1, (nchildren, n)), np.broadcast_to(p2, (nchildren, n)), u, di_crossover, xlb, xub)


def get_duplicates(X, Y=None, eps=1e-16):
    """MOEA.get_duplicates (MOEA.py:426-437): the self-comparison the optimizers use (AGEMOEA.py:203-205) and the
    two-set form of MOASMO's resample step (MOASMO.py:442): row i of X is a duplicate when a row j < i of Y is within
    eps (the reference masks the upper triangle of cdist(X, Y) including the diagonal)."""
    if Y is None or Y is X:
        return _lib.get_duplicates(X, eps)
    return _lib.get_duplicates(X, eps, Y=Y)


def remove_duplicates(population_parm, population_obj, eps=1e-16):
    """MOEA.remove_duplicates (MOEA.py:440-442)."""
    dup = get_duplicates(population_parm, eps=eps)
    return population_parm[~dup, :], population_obj[~dup, :]


class EpsilonSort:
    """MOEA.EpsilonSort (MOEA.py:470-595): an archive of epsilon-nondominated solutions with tag-along data.

    Same interface (``epsilons``, ``itobj``, ``archive``, ``tagalongs``, ``boxes``, ``add``, ``remove``, ``sortinto``), at
    most ``_lib.EPSILON_MAX_OBJECTIVES`` objectives.  ``sortinto`` only buffers its row (it still raises OverflowError
    at once where the reference's would); reading ``archive`` / ``tagalongs`` / ``boxes``, or calling ``add`` /
    ``remove``, sorts the buffered rows together with the current archive in one ``dmo_epsilon_sort`` call.  That gives
    the archive of one-by-one insertion: a row that left the archive loses again to whatever displaced it.
    """

    def __init__(self, epsilons):
        if len(epsilons) > _lib.EPSILON_MAX_OBJECTIVES:
            raise ValueError(f"dmosopt_b200.EpsilonSort: {len(epsilons)} objectives; dmo_epsilon_sort takes at most {_lib.EPSILON_MAX_OBJECTIVES}")
        self.epsilons = [e if e != 0 and not np.isnan(e) else 1e-8 for e in epsilons]
        self.itobj = range(len(epsilons))
        self._eps = np.array(self.epsilons, dtype=np.float64)
        self._archive, self._tagalongs, self._boxes = [], [], []
        self._pending = []  # (objectives, tagalong) not yet sorted in

    @property
    def archive(self):
        self._resolve()
        return self._archive

    @property
    def tagalongs(self):
        self._resolve()
        return self._tagalongs

    @property
    def boxes(self):
        self._resolve()
        return self._boxes

    def add(self, objectives, tagalong, ebox):
        """add a solution to the archive, plus auxiliary information"""
        self._resolve()
        self._archive.append(objectives)
        self._tagalongs.append(tagalong)
        self._boxes.append(ebox)

    def remove(self, index):
        """remove a solution from the archive"""
        self._resolve()
        self._archive.pop(index)
        self._tagalongs.pop(index)
        self._boxes.pop(index)

    def sortinto(self, objectives, tagalong=None):
        """Sort a solution into the archive (minimisation); ``tagalong`` is kept with it while it stays."""
        objectives = np.nan_to_num(objectives)
        with np.errstate(over="ignore"):
            if np.isinf(np.asarray(objectives[: len(self._eps)], dtype=np.float64) / self._eps).any():
                raise OverflowError("cannot convert float infinity to integer")
        self._pending.append((objectives, tagalong))

    def _resolve(self):
        if not self._pending:
            return
        rows = self._archive + [o for o, _ in self._pending]
        tags = self._tagalongs + [t for _, t in self._pending]
        self._pending = []
        M = len(self._eps)
        Y = np.array([np.asarray(r, dtype=np.float64)[:M] for r in rows])
        keep = _lib.epsilon_sort(Y, self._eps)
        self._archive = [rows[i] for i in keep]
        self._tagalongs = [tags[i] for i in keep]
        self._boxes = [[math.floor(v) for v in b] for b in np.floor(Y[keep] / self._eps)]
