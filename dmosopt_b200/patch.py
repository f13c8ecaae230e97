"""Opt-in routing of the reference controller's own helpers to the GPU library (SURVEY.md section 8f rows N2 / N3).

The optimizer and surrogate plugins are reached by import path and need no patching.  A few hot helpers, however, are
called by the reference's controller code directly on its own modules, so swapping the plugins does not reach them:

  * resample step of ``MOASMO.epoch``     ``MOEA.get_duplicates(best_x, x_0)`` + ``MOEA.crowding_distance_metric``
                                          (dmosopt/MOASMO.py:441-448)
  * ``MOASMO.get_best``                   ``MOEA.get_duplicates(y)`` + ``MOEA.sortMO`` (dmosopt/MOASMO.py:581-639)
  * per-generation termination            ``dmosopt.hv.AdaptiveHyperVolume.compute_hypervolume`` of the whole
                                          population (dmosopt/hv_termination.py:1093-1134 via the multi-fidelity
                                          tracker; dmosopt/hv.py:123-241): 'box' exactly for 1 .. 8 objectives, the
                                          Monte-Carlo branches for 2 .. 16 objectives (hv.HV_MC_DEFAULT_SEED,
                                          consecutive calls on consecutive streams); the rest stays with the reference
  * the rank function of every ``sortMO`` ``dmosopt.dda.dda_ens`` (dmosopt/dda.py:97-152)
  * ``MOASMO.epsilon_get_best``           ``MOEA.get_duplicates(y)`` + ``MOEA.EpsilonSort`` (dmosopt/MOASMO.py:703-758,
                                          dmosopt/MOEA.py:470-595): ``MOEA.EpsilonSort`` becomes a factory that builds
                                          this package's lazy archive for up to 16 objectives and the reference's own
                                          class for wider archives

``install()`` rebinds exactly those module attributes of an already importable ``dmosopt`` package to the functions of
this package (same signatures, same results: see tests/test_gpu_reference_loop.py) and ``uninstall()`` restores them.
``install(resident_epoch=True)`` also rebinds ``MOASMO.optimize``, the surrogate epoch of ``MOASMO.epoch``: an epoch
that ``dmosopt_b200.MOASMO.resident_eligible`` accepts (this package's NSGA2 or SMPSO with one of its GPU surrogates)
runs on the resident generation step, with the per-generation loop's results; every other epoch runs the reference's own
``optimize`` unchanged, including the yield / send protocol of an epoch without a surrogate.
Nothing is patched implicitly; importing dmosopt_b200 never touches dmosopt.
"""

import importlib
import inspect

import numpy as np

from . import MOEA as _MOEA
from . import _lib
from . import hv as _hv
from . import indicators as _ind

_saved = []


def _set(obj, name, new):
    _saved.append((obj, name, getattr(obj, name)))
    setattr(obj, name, new)


def _dda_ens(Y, return_dom=False):
    if return_dom:
        raise NotImplementedError("dmosopt_b200: the dense dominance matrix is never materialised (dda.py:40-41 needs O(n^2) memory)")
    return _lib.rank_nd(np.asarray(Y, dtype=np.float64))


def install(package="dmosopt", resident_epoch=False):
    """Route the helpers listed in the module docstring to the GPU (and, with ``resident_epoch``, eligible surrogate
    epochs to the resident generation step).  Returns the list of patched names."""
    if not _saved:
        _install_helpers(package)
    if resident_epoch and not any(name == "optimize" for _, name, _ in _saved):
        _install_resident_epoch(package)
    return [f"{getattr(o, '__name__', o)}.{n}" for o, n, _ in _saved]


def _install_resident_epoch(package):
    from . import MOASMO as _moasmo

    moasmo = importlib.import_module(f"{package}.MOASMO")
    original = moasmo.optimize
    signature = inspect.signature(original)

    def optimize(*args, **kwargs):
        a = signature.bind(*args, **kwargs)
        a.apply_defaults()
        if _moasmo.resident_eligible(a.arguments["optimizer"], a.arguments["model"], a.arguments["optimize_mean_variance"]):
            return (yield from _moasmo.optimize(*args, **kwargs))
        return (yield from original(*args, **kwargs))

    optimize.__doc__ = original.__doc__
    _set(moasmo, "optimize", optimize)


def _install_helpers(package):
    moea = importlib.import_module(f"{package}.MOEA")
    ind = importlib.import_module(f"{package}.indicators")
    dda = importlib.import_module(f"{package}.dda")
    hv = importlib.import_module(f"{package}.hv")
    for name in ("get_duplicates", "remove_duplicates", "sortMO", "orderMO", "remove_worst"):
        _set(moea, name, getattr(_MOEA, name))
    for mod in (moea, ind):
        for name in ("crowding_distance_metric", "euclidean_distance_metric"):
            if hasattr(mod, name):
                _set(mod, name, getattr(_ind, name))
    _set(dda, "dda_ens", _dda_ens)
    if hasattr(moea, "EpsilonSort"):
        reference_epsilon_sort = moea.EpsilonSort

        def EpsilonSort(epsilons):
            if len(epsilons) > _lib.EPSILON_MAX_OBJECTIVES:
                return reference_epsilon_sort(epsilons)
            return _MOEA.EpsilonSort(epsilons)

        _set(moea, "EpsilonSort", EpsilonSort)
    if hasattr(moea, "dda_ens"):
        _set(moea, "dda_ens", _dda_ens)

    original = hv.AdaptiveHyperVolume.compute_hypervolume
    mc_seed = _hv.HV_MC_DEFAULT_SEED
    mc_calls = [0]

    def compute_hypervolume(self, pareto_front, algorithm=None, verbose=False):
        auto = algorithm in (None, "auto")
        exact = algorithm == "box" or (auto and self.n_objectives < self.dimension_threshold_exact)
        if exact and 1 <= self.n_objectives <= _lib.HV_MAX_OBJECTIVES:
            pf = np.asarray(pareto_front, dtype=np.float64)
            if len(pf) == 0:
                return 0.0
            return _lib.hypervolume(pf, self.ref_point)  # points not strictly inside ref are ignored, as hv.py:159 does
        if not exact and 2 <= self.n_objectives <= _lib.HVMC_MAX_OBJECTIVES:
            # the Monte-Carlo branches; the reference's defaults for attributes a subclass or stand-in may lack
            if auto:
                algorithm = "hybrid" if getattr(self, "use_adaptive_mc", True) else "monte_carlo"
            if algorithm in _lib.HVMC_ALGORITHMS:
                pf = np.asarray(pareto_front, dtype=np.float64)
                if len(pf) == 0:
                    return 0.0
                value, _ = _lib.hypervolume_mc(pf, self.ref_point, algorithm, getattr(self, "mc_epsilon", 0.01), getattr(self, "mc_delta", 0.25),
                                               getattr(self, "monte_carlo_samples", 100000), seed=mc_seed, stream=mc_calls[0] % (1 << 24))
                mc_calls[0] += 1
                return value
        return original(self, pareto_front, algorithm, verbose)

    _set(hv.AdaptiveHyperVolume, "compute_hypervolume", compute_hypervolume)


def uninstall():
    while _saved:
        obj, name, old = _saved.pop()
        setattr(obj, name, old)
