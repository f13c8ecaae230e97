"""Host-side mirror of dmosopt's MOASMO helpers, backed by the CUDA library.

  * ``optimize``           MOASMO.py:21-131, the surrogate epoch: a drop-in with the same signature and generator
                           protocol.  An eligible epoch (``resident_eligible``) keeps the population in HBM and runs
                           each generation as one C call: for NSGA2, ``dmo_nsga2_step_record`` (GPR_Matern, GPR_RBF) or
                           ``dmo_nsga2_step_record_posterior`` (EGP, the variational and the deep-GP surrogates); for
                           SMPSO, ``dmo_smpso_step_record`` on the resident swarms (every one of those surrogates); for
                           CMAES, ``dmo_cmaes_step_record`` and ``dmo_cmaes_step_apply`` on the resident parent state.
                           Any other epoch runs the reference's per-generation plugin loop (``optimize_per_generation``).
                           Both return the same results.
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
    """True when ``optimize`` runs this epoch on a resident generation step: the optimizer is exactly
    ``dmosopt_b200.NSGA2``, ``dmosopt_b200.SMPSO`` or ``dmosopt_b200.CMAES``, the surrogate exactly ``GPR_Matern``,
    ``GPR_RBF``, ``EGP_Matern``, one of the five variational classes or one of the two deep GPs, with its device posterior
    and returning the mean only, no mean-variance objectives, no adaptive population size, and
      NSGA2: a y-metric of None, "crowding" or "euclidean", an x-metric of None or the rank of a GPU
             ``LogisticFeasibilityModel``;
      SMPSO: the same y-metrics and its resident swarm state (``SMPSO._resident``);
      CMAES: no x-metric (no ``model.feasibility``); its sortMO never reads the y-metric."""
    from .CMAES import CMAES
    from .model import GPR_Matern, GPR_RBF
    from .NSGA2 import NSGA2, _device_feasibility_key
    from .SMPSO import SMPSO

    sm = getattr(model, "objective", None)
    if type(optimizer) not in (NSGA2, SMPSO, CMAES):
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
    if type(optimizer) is CMAES:
        return optimizer.x_distance_metrics is None
    ym = optimizer.y_distance_metrics
    if ym is not None and (len(ym) != 1 or not isinstance(ym[0], str) or ym[0] not in ("crowding", "euclidean")):
        return False
    if type(optimizer) is SMPSO:
        return optimizer._resident_available()
    return optimizer.x_distance_metrics is None or _device_feasibility_key(optimizer.x_distance_metrics) is not None


def _state_fits(optimizer, model):
    """The initialized state has the shapes and dtypes of the resident step.  NSGA2: pop (>= 2) rows of float64
    parameters, float32 or float64 objectives, ranks.  SMPSO: swarm_size * pop rows of float32 positions, float32
    objectives and float64 velocities, one rank array per swarm.  CMAES: pop (>= 2) resident rows of parameters, step
    sizes (one or d per row), Cholesky factors, their inverses and paths, float32 or float64 objectives, success rates
    and ranks, and at least one offspring per generation."""
    from .CMAES import CMAES
    from .SMPSO import SMPSO

    st, sm = optimizer.state, model.objective
    pop = optimizer.opt_params.popsize
    if type(optimizer) is CMAES:
        p, d, M = optimizer.opt_params, sm.nInput, sm.nOutput
        rows = (st.parents_x, st.sigmas, st.A, st.Ainv, st.pc)
        y, ps, r = st.parents_y, st.psucc, np.asarray(st.rank)
        return (all(isinstance(a, _lib.ResidentRows) for a in rows) and st.parents_x.shape == (pop, d) and st.sigmas.shape in ((pop,), (pop, d))
                and st.A.shape == (pop, d, d) and st.Ainv.shape == (pop, d, d) and st.pc.shape == (pop, d) and isinstance(y, np.ndarray)
                and y.dtype in (np.float32, np.float64) and y.shape == (pop, M) and isinstance(ps, np.ndarray) and ps.dtype == np.float64
                and ps.shape == (pop,) and r.shape == (pop,) and pop >= 2 and int(p.mu) >= 1 and int(p.lambda_) >= 1 and d <= 512 and M <= 16)
    if type(optimizer) is SMPSO:
        n = optimizer.opt_params.swarm_size * pop
        x, y, v = st.population_parm, st.population_obj, st.velocity
        return (all(isinstance(a, np.ndarray) for a in (x, y, v)) and x.dtype == np.float32 and y.dtype == np.float32
                and v.dtype == np.float64 and x.shape == (n, sm.nInput) and y.shape == (n, sm.nOutput) and v.shape == (n, sm.nInput)
                and len(st.ranks) == optimizer.opt_params.swarm_size and optimizer._resident() is not None)
    x, y, r = st.population_parm, st.population_obj, np.asarray(st.rank)
    return (isinstance(x, np.ndarray) and isinstance(y, np.ndarray) and x.dtype == np.float64 and y.dtype in (np.float32, np.float64)
            and pop >= 2 and x.shape == (pop, sm.nInput) and y.shape == (pop, sm.nOutput) and r.shape == (pop,))


def optimize(num_generations, optimizer, model, nInput, nOutput, xlb, xub, popsize=100, initial=None, termination=None,
             local_random=None, logger=None, optimize_mean_variance=False, **kwargs):
    """dmosopt.MOASMO.optimize (MOASMO.py:21-131): a generator that returns the EpochResults through StopIteration.

    Eligible epochs (``resident_eligible``) never yield: the host steps before the loop are the reference's, then each
    generation is one C call on the population kept in HBM, with the same Philox streams, host draws, results and
    optimizer state as the per-generation loop.  NSGA2 steps on ``dmo_nsga2_step_record`` (or, for EGP, the variational
    and the deep-GP surrogates, ``dmo_nsga2_step_record_posterior``); the host waits for the offspring count of each
    generation, and with ``adaptive_operator_rates`` reads the operator counts before every ``update_operator_rates``.
    SMPSO steps on ``dmo_smpso_step_record`` with the swarms' velocity draws taken on the host; its success counter and
    operator rates need nothing from the device, and the host waits only inside the predict and the swarm truncations.
    CMAES steps on ``dmo_cmaes_step_record`` (with the normals and parent draws taken on the host first), one wait for
    the candidates' selection and the offspring's parents, its success rates and step-size factors on the host
    (``CMAES._strategy_scalars``), then ``dmo_cmaes_step_apply``.
    With ``termination`` the state is read back before every ``has_terminated``.  The offspring and their mean are
    recorded in page-locked memory, G * R * (d + M) * 8 bytes for G generations of R offspring rows (NSGA2: pop + 1,
    SMPSO: 2 * swarm_size * pop, CMAES: lambda_ * mu).  Other epochs run ``optimize_per_generation``."""
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
    """Page-locked rows the resident generations are recorded into: ``rows`` offspring rows, their means and
    ``n_counts`` operator counts per generation, allocated in blocks of ``per_block`` generations as the epoch goes (its
    length is open with a termination criterion; page-locked blocks of a bounded size are also recycled by the pool)."""

    def __init__(self, rows, d, M, per_block, n_counts):
        self.rows, self.d, self.M, self.per_block, self.n_counts = rows, d, M, max(int(per_block), 1), n_counts
        self.blocks = []
        self.n = 0

    def next(self):
        k, j = divmod(self.n, self.per_block)
        if k == len(self.blocks):
            b = self.per_block
            self.blocks.append((_lib.pinned_empty((b, self.rows, self.d)), _lib.pinned_empty((b, self.rows, self.M)),
                                _lib.pinned_empty((b, self.n_counts), np.int64) if self.n_counts else None))
        self.n += 1
        xb, yb, cb = self.blocks[k]
        return xb[j], yb[j], None if cb is None else cb[j]


def _resident_posterior(sm):
    """(kind, handle, precision, mean dtype, var_route_mean) of the surrogate's device posterior: the exact GP's mean-only
    predict for GPR_Matern / GPR_RBF, else the mean of the predict with variance (``resident_posterior``)."""
    from .model import GPR_Matern, GPR_RBF

    if type(sm) in (GPR_Matern, GPR_RBF):
        return _lib.POSTERIOR_GP, sm._gp, sm.precision, np.float64, False
    return tuple(sm.resident_posterior()) + (True,)


class _Nsga2Step:
    """NSGA2's generation on the population in HBM: ``dmo_nsga2_step_record`` (GPR_Matern, GPR_RBF) or
    ``dmo_nsga2_step_record_posterior``; the operator counts are added to the success counters once read."""

    n_counts = 4

    def __init__(self, optimizer, model, post):
        from .NSGA2 import _device_feasibility_key

        self.opt, self.sm, self.post = optimizer, model.objective, post
        st = optimizer.state
        pop, d = st.population_parm.shape
        M = st.population_obj.shape[1]
        self.rows = pop + 1
        self.key = _device_feasibility_key(optimizer.x_distance_metrics)
        ym = optimizer.y_distance_metrics
        self.metric = {None: _lib.METRIC_NONE, "crowding": _lib.METRIC_CROWDING, "euclidean": _lib.METRIC_EUCLIDEAN}[None if ym is None else ym[0]]
        self.round_f32 = st.population_obj.dtype == np.float32
        # the population in HBM: the state's own device mirror when it has one (NSGA2.initialize_state), else a copy
        base = getattr(optimizer, "_pop_base", None)
        if base is not None and (st.population_parm.ctypes.data != base.ctypes.data or st.population_parm.shape != base.shape):
            base = None
        self.dev_x = _lib.mirror_array(base) if base is not None else None
        if self.dev_x is None:
            base = None
            self.dev_x = _lib.DeviceArray((pop, d), np.float64).upload(st.population_parm)
        self.base = base
        self.dev_y = _lib.DeviceArray((pop, M), np.float64).upload(np.asarray(st.population_obj, dtype=np.float64))
        self.dev_r = _lib.DeviceArray((pop,), np.int32).upload(np.asarray(st.rank, dtype=np.int32))
        self.pending = []  # operator counts of generations not yet added to the success counters

    def __call__(self, x_gen, y_gen, counts, draw):
        opt, p, st = self.opt, self.opt.opt_params, self.opt.state
        xlb, xub = st.bounds[:, 0], st.bounds[:, 1]
        seed = opt._rng_seed()
        stream = opt._next_stream()  # the tournament's stream; the variation takes the next one
        opt._next_stream()
        kind, handle, precision, mean_dtype, var_route_mean = self.post
        if not var_route_mean:
            P = _lib.nsga2_step_record(handle, self.dev_x, self.dev_y, self.dev_r, p.crossover_prob, p.mutation_prob, p.mutation_rate,
                                       p.di_crossover, p.di_mutation, xlb, xub, seed, stream, precision, self.metric, self.round_f32, x_gen,
                                       y_gen, counts, key=self.key)
        else:
            P = _lib.nsga2_step_record_posterior(kind, handle, draw, self.dev_x, self.dev_y, self.dev_r, p.crossover_prob, p.mutation_prob,
                                                 p.mutation_rate, p.di_crossover, p.di_mutation, xlb, xub, seed, stream, precision,
                                                 self.metric, mean_dtype == np.float32, self.round_f32, x_gen, y_gen, counts, key=self.key)
        self.pending.append(counts)
        if p.adaptive_operator_rates:
            self._add_counts()  # the rates of the next generation depend on this one's counts
            opt.update_operator_rates()
        return P

    def _add_counts(self):
        _lib.synchronize()
        st = self.opt.state
        for c in self.pending:
            # with the plugin's types: len() of the index arrays, np.count_nonzero (an np.intp) of the survivors
            st.total_crossovers += int(c[0]) // 2  # NSGA2.py:159, 176
            st.total_mutations += int(c[1])
            st.successful_crossovers += np.intp(c[2]) / 2  # NSGA2.py:216-222
            st.successful_mutations += np.intp(c[3])
        self.pending.clear()

    def sync(self):
        """The host state as the plugin loop leaves it; every recorded row has landed."""
        self._add_counts()
        st = self.opt.state
        if self.base is not None:
            _lib.memcpy(self.base, self.dev_x.ptr, self.base.nbytes)  # the read-only state view shows the survivors
        else:
            self.opt._store_population(self.dev_x.download())
        st.population_obj[:] = self.dev_y.download()
        st.rank[:] = self.dev_r.download()


class _SmpsoStep:
    """SMPSO's generation on its resident swarms (``SMPSO._resident``): ``dmo_smpso_step_record`` with the velocity
    scalars drawn on the host.  Every swarm keeps pop of its 2 * pop stacked rows, all of them offspring indices below
    2 * swarm_size * pop, so the plugin's success count (np.isin over the survivors' indices) is swarm_size * pop per
    generation, known without the device."""

    n_counts = 0

    def __init__(self, optimizer, model, post):
        self.opt, self.post = optimizer, post
        self.sw = optimizer._resident()
        p = optimizer.opt_params
        self.n = p.swarm_size * p.popsize
        self.rows = 2 * self.n
        self.metric = optimizer._metric_code()
        self.dev_r = _lib.DeviceArray((self.n,), np.int32)  # written by every step; read only once one has run
        self.stepped = False

    def __call__(self, x_gen, y_gen, counts, draw):
        opt, p, st = self.opt, self.opt.opt_params, self.opt.state
        xlb, xub = st.bounds[:, 0], st.bounds[:, 1]
        seed = opt._rng_seed()  # generate_strategy's order: the seed, then the stream
        stream = opt._next_stream()
        sc = opt._velocity_scalars()  # update_strategy's draws
        kind, handle, precision, mean_dtype, var_route_mean = self.post
        self.sw.step_record(kind, handle, draw, var_route_mean, p.di_mutation, xlb, xub, p.mutation_rate, seed, stream, precision,
                            mean_dtype == np.float32, self.metric, sc, self.dev_r, x_gen, y_gen)
        self.stepped = True
        st.successful_children += self.n
        if p.adaptive_operator_rates:
            opt.update_operator_rates()
        return self.rows

    def sync(self):
        """The host state as the plugin loop leaves it, written into the state's own arrays (so the resident copy stays
        keyed to them); every recorded row has landed.  Before the first step the host state is already the plugin's."""
        _lib.synchronize()
        if not self.stepped:
            return
        st, sw = self.opt.state, self.sw
        st.population_parm[...] = sw.parm.download()  # float32 values: the casts are exact
        st.population_obj[...] = sw.obj.download()
        sw.velocity_into(st.velocity)
        r = self.dev_r.download().astype(np.intp).reshape(self.opt.opt_params.swarm_size, -1)
        for k in range(r.shape[0]):
            st.ranks[k] = r[k]


class _CmaesStep:
    """CMAES's generation on its resident parent state (``_lib.CmaesResident``): the normals and parent draws of
    generate_strategy from ``local_random`` in its order, ``dmo_cmaes_step_record``, one wait, the host arithmetic of
    update_strategy (``CMAES._strategy_scalars``), ``dmo_cmaes_step_apply``."""

    n_counts = 0

    def __init__(self, optimizer, model, post):
        self.opt, self.post = optimizer, post
        st, p = optimizer.state, optimizer.opt_params
        self.mu, self.lambda_ = int(p.mu), int(p.lambda_)
        self.rows = self.lambda_ * self.mu
        # vstack((y_gen, parents_y)) stays float32 only when both are
        self.cand_f32 = post[3] == np.float32 and st.parents_y.dtype == np.float32
        self.res = _lib.CmaesResident(st.parents_x, st.sigmas, st.A, st.Ainv, st.pc, st.parents_y, self.rows)
        self.psucc = st.psucc
        self.stepped = False

    def __call__(self, x_gen, y_gen, counts, draw):
        from .CMAES import _strategy_scalars

        opt, p, res = self.opt, self.opt.opt_params, self.res
        rng = opt.local_random
        xlb, xub = opt.bounds[:, 0], opt.bounds[:, 1]
        arz = rng.normal(size=(self.rows, res.d))  # generate_strategy's draws, in its order
        js = rng.choice(min(self.mu, res.pop), size=self.rows)
        kind, handle, precision, mean_dtype, var_route_mean = self.post
        res.step_record(kind, handle, draw, var_route_mean, precision, mean_dtype == np.float32, self.cand_f32, arz, js, self.mu, xlb, xub,
                        x_gen, y_gen)
        _lib.synchronize()
        chosen = res.codes.astype(bool)
        pidx = np.concatenate((res.p_idx, np.arange(res.pop, dtype=np.int_)))
        h = _strategy_scalars(p, self.psucc, pidx, self.rows, chosen, ~chosen)
        res.step_apply(h, xlb, xub, p.cc, p.ccov, p.pthresh)
        self.psucc = h.psucc
        self.stepped = True
        return self.rows

    def sync(self):
        """The host state as the plugin loop leaves it: the current half of the double buffer becomes the state's
        ResidentRows.  Before the first step the host state is already the plugin's."""
        _lib.synchronize()
        if not self.stepped:
            return
        st = self.opt.state
        st.parents_x, st.sigmas, st.A, st.Ainv, st.pc, py, rank = self.res.state
        st.parents_y = py.download().astype(np.float32 if self.cand_f32 else np.float64)
        st.rank = rank.download().astype(np.intp)
        st.psucc = self.psucc


def _resident_generations(num_generations, optimizer, model, termination, logger, OptHistory):
    """The generations of an eligible epoch on the resident step; yields (i, x_gen, y_gen) once the epoch is done (the
    rows are views of the page-locked record) and leaves the optimizer's state as the per-generation loop leaves it."""
    from .CMAES import CMAES
    from .SMPSO import SMPSO

    sm = model.objective
    post = _resident_posterior(sm)
    step = {SMPSO: _SmpsoStep, CMAES: _CmaesStep}.get(type(optimizer), _Nsga2Step)(optimizer, model, post)
    # blocks of 8 generations, or of the whole epoch when it is shorter and its length is known
    per_block = 8 if termination is not None else min(8, num_generations)
    hist = _History(step.rows, sm.nInput, sm.nOutput, per_block, step.n_counts)
    done = []
    n_eval = 0
    it = range(1, num_generations + 1) if termination is None else itertools.count(1)
    for i in it:
        if termination is not None:
            step.sync()
            pop_x, pop_y = optimizer.population_objectives
            if termination.has_terminated(OptHistory(i, n_eval, pop_x, pop_y, None)):
                break
        _log_generation(logger, optimizer, i, num_generations, termination)
        x_gen, y_gen, counts = hist.next()
        # a deep GP draws its key as each predict does: MDGP's call counter advances once per generation, in order
        draw = sm._draw_key() if post[0] == _lib.POSTERIOR_DGP else (0, 0)
        P = step(x_gen, y_gen, counts, draw)
        n_eval += P
        done.append((i, x_gen[:P], y_gen[:P]))
    step.sync()
    if post[3] == np.float32:
        # evaluate's float32 means (the record holds them exactly); read once the copies have landed (sync synchronised)
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
