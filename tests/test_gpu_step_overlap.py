"""dmo_nsga2_step runs its truncation on a stream of its own, beside the GP's variance contraction (which runs on a
higher-priority stream, its grid keeping DMO_GP_VAR_RESERVE more SMs free), unless DMO_STEP_OVERLAP=0 keeps the serial
order.  From the same population and Philox streams, every setting must give bit-identical population, objectives,
ranks, offspring count and hypervolume, with the same number of host waits: the order of the work changes, not the work."""

import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SETTINGS = [("0", None), ("1", "0"), ("1", "8"), ("1", "100000")]  # (DMO_STEP_OVERLAP, DMO_GP_VAR_RESERVE); the last: one CTA


def _dtlz2(X, M):
    g = ((X[:, M - 1 :] - 0.5) ** 2).sum(axis=1)
    Y = np.ones((X.shape[0], M)) * (1.0 + g)[:, None]
    for i in range(M):
        for j in range(M - 1 - i):
            Y[:, i] *= np.cos(0.5 * np.pi * X[:, j])
        if i > 0:
            Y[:, i] *= np.sin(0.5 * np.pi * X[:, M - 1 - i])
    return Y


# name: (d, N_train, pop, objectives, metric)
CASES = {
    "peel": (30, 1024, 16384, "dtlz2", 0),
    # offspring next to the training inputs: AUTO refines rows and the step truncates again after the lane has joined
    "refined": (30, 4096, 4096, "dtlz2_on_training", 0),
    # merged set below the peel threshold (n < 8192): the truncation ranks through the chain kernel on the lane
    "chain_crowding": (30, 1024, 4095, "dtlz2", 1),
}


@pytest.mark.parametrize("case", list(CASES))
def test_overlap_settings_give_the_same_bits_and_waits(monkeypatch, case):
    import dmosopt_b200 as b2
    from dmosopt_b200 import _lib as L

    L.context()
    d, N, pop, kind, metric = CASES[case]
    M = 3
    rng = np.random.default_rng(77 + len(case))
    xlb, xub = np.zeros(d), np.ones(d)
    Xtr = rng.random((N, d))
    Ytr = _dtlz2(Xtr, M)
    sm = b2.GPR_Matern(Xtr, Ytr, d, M, xlb, xub, optimizer=None)
    gp = sm._gp
    gp.predict(rng.random((64, d)), return_var=True, precision=L.GP_AUTO)
    assert gp.auto_info()["var_tensor"], case
    x0 = Xtr[:pop].copy() if kind == "dtlz2_on_training" else rng.random((pop, d))
    y0 = sm.evaluate(x0).astype(np.float32).astype(np.float64)
    r0 = L.rank_nd(y0).astype(np.int32)
    ref = y0.max(axis=0) + 0.1 * (y0.max(axis=0) - y0.min(axis=0))
    lib, ctx = L.load_library(), L.context()
    DA = L.DeviceArray
    dic, dim = DA((d,)).upload(np.full(d, 1.0)), DA((d,)).upload(np.full(d, 20.0))
    dlb, dub = DA((d,)).upload(xlb), DA((d,)).upload(xub)

    runs = []
    for overlap, reserve in SETTINGS:
        monkeypatch.setenv("DMO_STEP_OVERLAP", overlap)
        if reserve is None:
            monkeypatch.delenv("DMO_GP_VAR_RESERVE", raising=False)
        else:
            monkeypatch.setenv("DMO_GP_VAR_RESERVE", reserve)
        fx, fy, fr = DA((pop, d)).upload(x0), DA((pop, M)).upload(y0), DA((pop,), np.int32).upload(r0)
        nch = np.zeros(1, dtype=np.int64)
        gens = []
        for gen in range(2):
            hv = ctypes.c_double(0.0)
            w0 = L.wait_count()
            L._check(lib.dmo_nsga2_step(ctx, gp._h, fx.ptr, fy.ptr, fr.ptr, pop, d, M, 0.9, 0.1, 1.0 / d, dic.ptr, dim.ptr, dlb.ptr,
                                        dub.ptr, 99, 2 * gen + 1, L.GP_AUTO, metric, 1, 1, ref.ctypes.data, nch.ctypes.data,
                                        ctypes.byref(hv)), "nsga2_step")
            gens.append((L.wait_count() - w0, int(nch[0]), hv.value, gp.auto_info()["last_refined"]))
        runs.append((gens, fx.download(), fy.download(), fr.download()))

    base = runs[0]
    for (overlap, reserve), run in zip(SETTINGS[1:], runs[1:]):
        msg = (case, overlap, reserve)
        assert run[0] == base[0], (msg, run[0], base[0])  # waits, offspring count, hypervolume, rows refined
        for a, b in zip(run[1:], base[1:]):
            assert np.array_equal(a, b), msg
    if case == "refined":
        assert max(g[3] for g in base[0]) > 0, base[0]
