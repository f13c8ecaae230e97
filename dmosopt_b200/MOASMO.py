"""Host-side mirror of dmosopt's MOASMO helpers, backed by the CUDA library.

  * ``optimize``           MOASMO.py:21-131, the surrogate epoch: a drop-in with the same signature and generator
                           protocol.  An eligible epoch (``resident_eligible``) keeps the population in HBM and runs
                           each generation as one ``dmo_nsga2_step_record`` call (GPR_Matern, GPR_RBF) or one
                           ``dmo_nsga2_step_record_posterior`` call (EGP, the variational and the deep-GP surrogates); any
                           other runs the reference's per-generation plugin loop (``optimize_per_generation``).  Both
                           return the same results.
  * ``epsilon_get_best``   MOASMO.py:703-758 -> MOEA.get_duplicates (dmo_get_duplicates) + dmo_epsilon_sort
"""

import itertools
from collections import namedtuple

import numpy as np
from numpy.random import default_rng
from scipy import stats

from . import MOEA, _lib
from .driver import EpochResults as _EpochResults

_OptHistory = namedtuple("OptHistory", ["n_gen", "n_eval", "x", "y", "c"])  # dmosopt/datatypes.py


def _datatypes():
    """(OptHistory, EpochResults): dmosopt's own when it is importable, the same named tuples otherwise."""
    try:
        from dmosopt.datatypes import EpochResults, OptHistory
    except ImportError:
        return _OptHistory, _EpochResults
    return OptHistory, EpochResults


def _posterior_types():
    """The surrogate types whose epochs step on ``dmo_nsga2_step_record_posterior`` (by exact type)."""
    from .model_gpflow import CRV_Matern, SIV_Matern, SPV_Matern, SVGP_Matern, VGP_Matern
    from .model_gpytorch import EGP_Matern, MDGP_Matern, MDSPP_Matern

    return (EGP_Matern, SVGP_Matern, VGP_Matern, SIV_Matern, SPV_Matern, CRV_Matern, MDSPP_Matern, MDGP_Matern)


def resident_eligible(optimizer, model, optimize_mean_variance=False):
    """True when ``optimize`` runs this epoch on the resident generation step: the optimizer is exactly
    ``dmosopt_b200.NSGA2``, the surrogate exactly ``GPR_Matern``, ``GPR_RBF``, ``EGP_Matern``, one of the five
    variational classes or one of the two deep GPs, with its device posterior and returning the mean only, no
    mean-variance objectives, no adaptive population size, a y-metric of None, "crowding" or "euclidean", and an x-metric
    of None or the rank of a GPU ``LogisticFeasibilityModel``."""
    from .model import GPR_Matern, GPR_RBF
    from .NSGA2 import NSGA2, _device_feasibility_key

    sm = getattr(model, "objective", None)
    if type(optimizer) is not NSGA2:
        return False
    if type(sm) in (GPR_Matern, GPR_RBF):
        if getattr(sm, "_gp", None) is None:
            return False
    elif type(sm) not in _posterior_types() or sm.resident_posterior()[1] is None:
        return False
    if optimize_mean_variance or optimizer.optimize_mean_variance or sm.return_mean_variance:
        return False
    if optimizer.opt_params.adaptive_population_size:
        return False
    ym = optimizer.y_distance_metrics
    if ym is not None and (len(ym) != 1 or not isinstance(ym[0], str) or ym[0] not in ("crowding", "euclidean")):
        return False
    return optimizer.x_distance_metrics is None or _device_feasibility_key(optimizer.x_distance_metrics) is not None


def _state_fits(optimizer, model):
    """The initialized state has the shapes and dtypes of the resident step: pop (>= 2) rows of float64 parameters,
    float32 or float64 objectives, ranks."""
    st, sm = optimizer.state, model.objective
    x, y, r = st.population_parm, st.population_obj, np.asarray(st.rank)
    pop = optimizer.opt_params.popsize
    return (isinstance(x, np.ndarray) and isinstance(y, np.ndarray) and x.dtype == np.float64 and y.dtype in (np.float32, np.float64)
            and pop >= 2 and x.shape == (pop, sm.nInput) and y.shape == (pop, sm.nOutput) and r.shape == (pop,))


def optimize(num_generations, optimizer, model, nInput, nOutput, xlb, xub, popsize=100, initial=None, termination=None,
             local_random=None, logger=None, optimize_mean_variance=False, **kwargs):
    """dmosopt.MOASMO.optimize (MOASMO.py:21-131): a generator that returns the EpochResults through StopIteration.

    Eligible epochs (``resident_eligible``) never yield: the host steps before the loop are the reference's, then each
    generation is one ``dmo_nsga2_step_record`` (or, for EGP, the variational and the deep-GP surrogates,
    ``dmo_nsga2_step_record_posterior``) call on the population kept in HBM, with the same Philox streams,
    results and optimizer state as the per-generation loop.  The host waits only for the offspring count of each
    generation; with ``termination`` it also reads the population back before every ``has_terminated``, and with
    ``adaptive_operator_rates`` the operator counts before every ``update_operator_rates``.  The offspring and their
    mean are recorded in page-locked memory, G * (pop + 1) * (d + M) * 8 bytes for G generations.  Other epochs run
    ``optimize_per_generation``."""
    return _optimize(True, num_generations, optimizer, model, nInput, nOutput, xlb, xub, popsize, initial, termination,
                     local_random, logger, optimize_mean_variance, kwargs)


def optimize_per_generation(num_generations, optimizer, model, nInput, nOutput, xlb, xub, popsize=100, initial=None,
                            termination=None, local_random=None, logger=None, optimize_mean_variance=False, **kwargs):
    """The reference's loop (MOASMO.py:21-131) as it stands: ``optimizer.generate``, ``model.objective.evaluate`` and
    ``optimizer.update`` once per generation (or, without a surrogate, the values sent back for each yielded x)."""
    return _optimize(False, num_generations, optimizer, model, nInput, nOutput, xlb, xub, popsize, initial, termination,
                     local_random, logger, optimize_mean_variance, kwargs)


def _optimize(resident, num_generations, optimizer, model, nInput, nOutput, xlb, xub, popsize, initial, termination,
              local_random, logger, optimize_mean_variance, optimizer_kwargs):
    OptHistory, EpochResults = _datatypes()
    if local_random is None:
        local_random = default_rng()
    bounds = np.column_stack((xlb, xub))

    x = optimizer.generate_initial(bounds, local_random)
    if model.objective is None:
        y = yield x
    else:
        if optimize_mean_variance:
            y_mean, y_variance = model.objective.evaluate(x)
            y = np.column_stack((y_mean, np.round(y_variance, 6))).astype(np.float32)
        else:
            y = model.objective.evaluate(x).astype(np.float32)

    x_initial = y_initial = None
    if initial is not None:
        x_initial, y_initial = initial
    if x_initial is not None:
        x = np.vstack((x_initial.astype(np.float32), x))
    if y_initial is not None:
        y = np.vstack((y_initial.astype(np.float32), y))

    optimizer.initialize_strategy(x, y, bounds, local_random, **optimizer_kwargs)
    if logger is not None:
        logger.info(f"{optimizer.name}: optimizer parameters are {repr(optimizer.opt_params)}")

    gen_indexes = [np.zeros((x.shape[0],), dtype=np.uint32)]
    x_new, y_new = [], []
    if (resident and model.objective is not None and resident_eligible(optimizer, model, optimize_mean_variance)
            and _state_fits(optimizer, model)):
        for i, x_gen, y_gen in _resident_generations(num_generations, optimizer, model, termination, logger, OptHistory):
            x_new.append(x_gen)
            y_new.append(y_gen)
            gen_indexes.append(np.ones((x_gen.shape[0],), dtype=np.uint32) * i)
    else:
        n_eval = 0
        it = range(1, num_generations + 1) if termination is None else itertools.count(1)
        for i in it:
            if termination is not None:
                pop_x, pop_y = optimizer.population_objectives
                if termination.has_terminated(OptHistory(i, n_eval, pop_x, pop_y, None)):
                    break
            _log_generation(logger, optimizer, i, num_generations, termination)
            x_gen, state_gen = optimizer.generate()
            if model.objective is None:
                y_gen = yield x_gen
            elif optimize_mean_variance:
                y_gen_mean, y_gen_variance = model.objective.evaluate(x_gen)
                y_gen = np.column_stack((y_gen_mean, np.round(y_gen_variance, 6)))
            else:
                y_gen = model.objective.evaluate(x_gen)
            optimizer.update(x_gen, y_gen, state_gen)
            n_eval += x_gen.shape[0]
            x_new.append(x_gen)
            y_new.append(y_gen)
            gen_indexes.append(np.ones((x_gen.shape[0],), dtype=np.uint32) * i)

    gen_index = np.concatenate(gen_indexes)
    x = np.vstack([x] + x_new)
    y = np.vstack([y] + y_new)
    bestx, besty = optimizer.population_objectives
    return EpochResults(bestx, besty, gen_index, x, y, optimizer)


def _log_generation(logger, optimizer, i, num_generations, termination):
    if logger is not None:
        if termination is not None:
            logger.info(f"{optimizer.name}: generation {i}...")
        else:
            logger.info(f"{optimizer.name}: generation {i} of {num_generations}...")


class _History:
    """Page-locked rows the resident generations are recorded into: (pop + 1) offspring rows, their means and four
    operator counts per generation, allocated in blocks of ``per_block`` generations as the epoch goes (its length is
    open with a termination criterion; page-locked blocks of a bounded size are also recycled by the pool)."""

    def __init__(self, pop, d, M, per_block):
        self.pop, self.d, self.M, self.per_block = pop, d, M, max(int(per_block), 1)
        self.blocks = []
        self.n = 0

    def next(self):
        k, j = divmod(self.n, self.per_block)
        if k == len(self.blocks):
            b = self.per_block
            self.blocks.append((_lib.pinned_empty((b, self.pop + 1, self.d)), _lib.pinned_empty((b, self.pop + 1, self.M)),
                                _lib.pinned_empty((b, 4), np.int64)))
        self.n += 1
        xb, yb, cb = self.blocks[k]
        return xb[j], yb[j], cb[j]


def _resident_generations(num_generations, optimizer, model, termination, logger, OptHistory):
    """The generations of an eligible epoch on the resident step; yields (i, x_gen, y_gen) once the epoch is done (the
    rows are views of the page-locked record) and leaves the optimizer's state as the per-generation loop leaves it."""
    from .NSGA2 import _device_feasibility_key

    from .model import GPR_Matern, GPR_RBF

    p, st, sm = optimizer.opt_params, optimizer.state, model.objective
    # (kind, handle, precision, mean dtype) of the surrogates that step on dmo_nsga2_step_record_posterior
    post = None if type(sm) in (GPR_Matern, GPR_RBF) else sm.resident_posterior()
    pop, d = st.population_parm.shape
    M = st.population_obj.shape[1]
    key = _device_feasibility_key(optimizer.x_distance_metrics)
    ym = optimizer.y_distance_metrics
    metric = {None: _lib.METRIC_NONE, "crowding": _lib.METRIC_CROWDING, "euclidean": _lib.METRIC_EUCLIDEAN}[None if ym is None else ym[0]]
    round_f32 = st.population_obj.dtype == np.float32
    xlb, xub = st.bounds[:, 0], st.bounds[:, 1]

    # the population in HBM: the state's own device mirror when it has one (NSGA2.initialize_state), else a copy
    base = getattr(optimizer, "_pop_base", None)
    if base is not None and (st.population_parm.ctypes.data != base.ctypes.data or st.population_parm.shape != base.shape):
        base = None
    dev_x = _lib.mirror_array(base) if base is not None else None
    if dev_x is None:
        base = None
        dev_x = _lib.DeviceArray((pop, d), np.float64).upload(st.population_parm)
    dev_y = _lib.DeviceArray((pop, M), np.float64).upload(np.asarray(st.population_obj, dtype=np.float64))
    dev_r = _lib.DeviceArray((pop,), np.int32).upload(np.asarray(st.rank, dtype=np.int32))

    def sync_state():
        if base is not None:
            _lib.memcpy(base, dev_x.ptr, base.nbytes)  # the read-only state view shows the survivors
        else:
            optimizer._store_population(dev_x.download())
        st.population_obj[:] = dev_y.download()
        st.rank[:] = dev_r.download()

    pending = []  # operator counts of generations not yet added to the success counters

    def add_counts():
        _lib.synchronize()
        for c in pending:
            # with the plugin's types: len() of the index arrays, np.count_nonzero (an np.intp) of the survivors
            st.total_crossovers += int(c[0]) // 2  # NSGA2.py:159, 176
            st.total_mutations += int(c[1])
            st.successful_crossovers += np.intp(c[2]) / 2  # NSGA2.py:216-222
            st.successful_mutations += np.intp(c[3])
        pending.clear()

    hist = _History(pop, d, M, 8)
    done = []
    n_eval = 0
    it = range(1, num_generations + 1) if termination is None else itertools.count(1)
    for i in it:
        if termination is not None:
            add_counts()
            sync_state()
            pop_x, pop_y = optimizer.population_objectives
            if termination.has_terminated(OptHistory(i, n_eval, pop_x, pop_y, None)):
                break
        _log_generation(logger, optimizer, i, num_generations, termination)
        seed = optimizer._rng_seed()
        stream = optimizer._next_stream()  # the tournament's stream; the variation takes the next one
        optimizer._next_stream()
        x_gen, y_gen, counts = hist.next()
        if post is None:
            P = _lib.nsga2_step_record(sm._gp, dev_x, dev_y, dev_r, p.crossover_prob, p.mutation_prob, p.mutation_rate, p.di_crossover,
                                       p.di_mutation, xlb, xub, seed, stream, sm.precision, metric, round_f32, x_gen, y_gen, counts, key=key)
        else:
            kind, handle, precision, mean_dtype = post
            # a deep GP draws its key as each predict does: MDGP's call counter advances once per generation, in order
            draw = sm._draw_key() if kind == _lib.POSTERIOR_DGP else (0, 0)
            P = _lib.nsga2_step_record_posterior(kind, handle, draw, dev_x, dev_y, dev_r, p.crossover_prob, p.mutation_prob, p.mutation_rate,
                                                 p.di_crossover, p.di_mutation, xlb, xub, seed, stream, precision, metric,
                                                 mean_dtype == np.float32, round_f32, x_gen, y_gen, counts, key=key)
        pending.append(counts)
        n_eval += P
        done.append((i, x_gen[:P], y_gen[:P]))
        if p.adaptive_operator_rates:
            add_counts()  # the rates of the next generation depend on this one's counts
            optimizer.update_operator_rates()
    add_counts()
    sync_state()
    if post is not None and post[3] == np.float32:
        # evaluate's float32 means (the record holds them exactly); read once the copies have landed (add_counts synchronised)
        done = [(i, x, y.astype(np.float32)) for i, x, y in done]
    yield from done


def epsilon_get_best(x, y, f, c, feasible=True, delete_duplicates=True, epsilons=None):
    """The epsilon-nondominated rows of a run's evaluations: (x[m], y[m], f[m], c[m], epsilons).

    As the reference: infeasible rows (some c <= 0) are dropped only when some row is feasible, then duplicate rows of
    y; ``epsilons`` is None (1e-9 per objective), a number, a sequence or "auto" (5 % of the inter-quartile range of the
    remaining y); an empty set returns early.  The archive is one ``dmo_epsilon_sort`` call over every row in order.
    Unlike the reference under NumPy 2 (``epsilons == "auto"`` raises ValueError on an array of several epsilons), a
    NumPy array is accepted like a list.
    """
    if feasible and c is not None:
        feasible = np.argwhere(np.all(c > 0.0, axis=1)).ravel()
        if len(feasible) > 0:
            x = x[feasible, :]
            y = y[feasible, :]
            if f is not None:
                f = f[feasible]
            c = c[feasible, :]

    if delete_duplicates:
        is_duplicate = MOEA.get_duplicates(y)
        x = x[~is_duplicate]
        y = y[~is_duplicate]
        if f is not None:
            f = f[~is_duplicate]
        if c is not None:
            c = c[~is_duplicate]

    if epsilons is None:
        epsilons = [1e-9] * y.shape[1]
    elif isinstance(epsilons, (int, float)):
        epsilons = [float(epsilons)] * y.shape[1]
    elif isinstance(epsilons, str) and epsilons == "auto":
        epsilons = 0.05 * stats.iqr(y, axis=0)

    if y.shape[0] == 0:
        return x, y, f, c, epsilons

    m = _lib.epsilon_sort(y, epsilons)
    return x[m], y[m], (None if f is None else f[m]), (None if c is None else c[m]), epsilons
