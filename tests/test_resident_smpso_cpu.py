"""Host logic of the resident SMPSO surrogate epoch (dmosopt_b200.MOASMO.optimize on dmo_smpso_step_record) without a GPU:
which SMPSO epochs are eligible, the velocity scalars drawn in the plugin's order, and the generator protocol of an epoch
without a surrogate."""

import numpy as np
import pytest

import fake_backend


class _FakeGP:
    pass


def _gp(mean_variance=False, handle=True):
    import dmosopt_b200 as b2

    sm = b2.GPR_Matern.__new__(b2.GPR_Matern)
    sm._gp, sm.return_mean_variance = (_FakeGP() if handle else None), mean_variance
    return sm


def _smpso(model, cls=None, **kw):
    import dmosopt_b200 as b2

    return (cls or b2.SMPSO)(popsize=10, nInput=3, nOutput=2, model=model, swarm_size=2, **kw)


def test_eligibility(monkeypatch):
    import dmosopt_b200 as b2
    from dmosopt_b200 import _lib
    from dmosopt_b200.MOASMO import resident_eligible

    class _Sub(b2.SMPSO):
        pass

    m = b2.Model(objective=_gp())
    for metric in (None, "crowding", "euclidean"):
        assert resident_eligible(_smpso(m, distance_metric=metric), m)
    assert resident_eligible(_smpso(m, adaptive_operator_rates=True), m)

    assert not resident_eligible(_smpso(m, cls=_Sub), m)
    assert not resident_eligible(_smpso(m, adaptive_population_size=True), m)
    assert not resident_eligible(_smpso(m, distance_metric=lambda y: y[:, 0]), m)
    assert not resident_eligible(_smpso(m), m, optimize_mean_variance=True)
    for sm in (_gp(mean_variance=True), _gp(handle=False), None):
        mm = b2.Model(objective=sm)
        assert not resident_eligible(_smpso(mm), mm)
    # a library without the resident swarm state
    monkeypatch.setattr(_lib, "SmpsoSwarms", None)
    assert not resident_eligible(_smpso(m), m)


def _plugin_draws(rng, swarms, popsize):
    """The draws of SMPSO.velocity_vector (SMPSO.py:317-331), one swarm after the other, as the resident update passes them."""
    out = []
    for _ in range(swarms):
        r1 = rng.uniform(low=0.0, high=1.0, size=1)[0]
        r2 = rng.uniform(low=0.0, high=1.0, size=1)[0]
        w = rng.uniform(low=0.1, high=0.5, size=1)[0]
        c1 = rng.uniform(low=1.5, high=2.5, size=1)[0]
        c2 = rng.uniform(low=1.5, high=2.5, size=1)[0]
        phi = c1 + c2 if c1 + c2 > 4 else 0
        chi = 2 / (2 - phi - ((phi**2) - 4 * phi) ** (1 / 2))
        ind = rng.integers(low=0, high=popsize, size=2) if popsize > 2 else (-1, -1)
        out.append((w, c1, r1, c2, r2, chi, ind[0], ind[1]))
    return np.array(out, dtype=np.float64)


@pytest.mark.parametrize("swarms,popsize", [(1, 2), (2, 3), (5, 24)])
def test_velocity_scalars_are_the_plugin_draws(swarms, popsize):
    import dmosopt_b200 as b2

    opt = b2.SMPSO(popsize=popsize, nInput=3, nOutput=2, model=b2.Model(), swarm_size=swarms)
    opt.local_random = np.random.default_rng(5)
    ref_rng = np.random.default_rng(5)
    for _ in range(3):
        got = opt._velocity_scalars()
        want = _plugin_draws(ref_rng, swarms, popsize)
        assert got.dtype == np.float64 and got.shape == (swarms, 8) and np.array_equal(got, want)
    assert opt.local_random.random() == ref_rng.random()


def _dtlz2(X, M):
    g = ((X[:, M - 1 :] - 0.5) ** 2).sum(axis=1)
    Y = np.ones((X.shape[0], M)) * (1.0 + g)[:, None]
    for i in range(M):
        for j in range(M - 1 - i):
            Y[:, i] *= np.cos(0.5 * np.pi * X[:, j])
        if i > 0:
            Y[:, i] *= np.sin(0.5 * np.pi * X[:, M - 1 - i])
    return Y


def test_epoch_without_surrogate_still_yields(monkeypatch):
    """With model.objective None the SMPSO epoch yields x and takes y back (MOASMO.py:57-58, 107-108)."""
    import dmosopt_b200 as b2
    from dmosopt_b200 import MOASMO

    fake_backend.install(monkeypatch)
    d, M, pop, S = 4, 2, 6, 2
    xlb, xub = np.zeros(d), np.ones(d)
    opt = b2.SMPSO(popsize=pop, nInput=d, nOutput=M, model=b2.Model(), swarm_size=S)
    gen = MOASMO.optimize(2, opt, b2.Model(), d, M, xlb, xub, popsize=pop, local_random=np.random.default_rng(1))
    x = next(gen)
    n = 0
    try:
        while True:
            x = gen.send(_dtlz2(np.asarray(x, dtype=np.float64), M))
            n += 1
    except StopIteration as ex:
        res = ex.value
    assert n == 2
    assert res.gen_index.max() == 2 and res.x.shape[0] == res.y.shape[0] == S * pop + 2 * (2 * S * pop)
