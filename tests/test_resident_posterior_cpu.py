"""Which surrogates step on dmo_nsga2_step_record_posterior (no GPU): MOASMO.resident_eligible accepts EGP_Matern, the
five variational classes and the two deep GPs by exact type, with a device posterior and without mean-variance
objectives; not their subclasses, and not MEGP_Matern."""

import numpy as np

CLASSES = {  # class name: (module, handle attribute, posterior kind, mean dtype)
    "EGP_Matern": ("model_gpytorch", "_gp", 0, np.float32),
    "SVGP_Matern": ("model_gpflow", "_h", 1, np.float32),
    "VGP_Matern": ("model_gpflow", "_h", 1, np.float32),
    "SIV_Matern": ("model_gpflow", "_h", 1, np.float32),
    "SPV_Matern": ("model_gpflow", "_h", 1, np.float32),
    "CRV_Matern": ("model_gpflow", "_h", 1, np.float32),
    "MDSPP_Matern": ("model_gpytorch", "_gp", 2, np.float64),
    "MDGP_Matern": ("model_gpytorch", "_gp", 2, np.float64),
}


class _Handle:
    pass


def _surrogate(cls, attr, mean_variance=False, handle=True):
    sm = cls.__new__(cls)
    sm.return_mean_variance, sm.precision = mean_variance, 1
    if handle:
        setattr(sm, attr, _Handle())
    return sm


def _nsga2(model, **kw):
    import dmosopt_b200 as b2

    return b2.NSGA2(popsize=10, nInput=3, nOutput=2, model=model, **kw)


def test_the_eight_classes_are_eligible_by_exact_type():
    import importlib

    import dmosopt_b200 as b2
    from dmosopt_b200 import _lib
    from dmosopt_b200.MOASMO import resident_eligible

    assert (_lib.POSTERIOR_GP, _lib.POSTERIOR_SVGP, _lib.POSTERIOR_DGP) == (0, 1, 2)
    for name, (mod, attr, kind, dtype) in CLASSES.items():
        cls = getattr(importlib.import_module(f"dmosopt_b200.{mod}"), name)
        sm = _surrogate(cls, attr)
        assert sm.resident_posterior() == (kind, getattr(sm, attr), 1, dtype), name
        m = b2.Model(objective=sm)
        assert resident_eligible(_nsga2(m), m), name
        assert resident_eligible(_nsga2(m, distance_metric="crowding"), m), name
        assert resident_eligible(_nsga2(m, adaptive_operator_rates=True), m), name
        assert not resident_eligible(_nsga2(m), m, optimize_mean_variance=True), name
        assert not resident_eligible(_nsga2(m, adaptive_population_size=True), m), name
        assert not resident_eligible(b2.AGEMOEA(popsize=10, nInput=3, nOutput=2, model=m), m), name

        sub = type("Sub" + name, (cls,), {})
        for other in (_surrogate(sub, attr), _surrogate(cls, attr, mean_variance=True), _surrogate(cls, attr, handle=False)):
            mm = b2.Model(objective=other)
            assert not resident_eligible(_nsga2(mm), mm), (name, type(other).__name__)
        none = _surrogate(cls, attr)
        setattr(none, attr, None)
        mm = b2.Model(objective=none)
        assert not resident_eligible(_nsga2(mm), mm), name


def test_megp_stays_on_the_plugin_loop():
    import dmosopt_b200 as b2
    from dmosopt_b200.model_gpytorch import MEGP_Matern
    from dmosopt_b200.MOASMO import resident_eligible

    sm = _surrogate(MEGP_Matern, "_gp")
    m = b2.Model(objective=sm)
    assert not resident_eligible(_nsga2(m), m)
