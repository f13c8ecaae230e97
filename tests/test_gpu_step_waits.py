"""dmo_nsga2_step composes the device bodies of the entry points it uses, without their trailing host waits, and on the
tensor route truncates on a stream of its own beside the GP's variance contraction.  For several generations the fused
step runs beside the same generation composed serially from the public entry points on device buffers (as bench.py's
multi-GPU branch composes it), from the same population and Philox streams: population, objectives, ranks,
offspring count and hypervolume must be bit-identical, and the fused step must wait on the host only where it needs a
value (the offspring count, one read-back after the GP, one per peeled front and the hypervolume's route and value), i.e.
exactly the composed calls' waits minus the trailing wait of each of the four wrappers (plus a second truncation's when
AUTO refines rows: the fused step truncates before it reads the GP back, and again on the refined rows)."""

import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def _dtlz2(X, M):
    g = ((X[:, M - 1 :] - 0.5) ** 2).sum(axis=1)
    Y = np.ones((X.shape[0], M)) * (1.0 + g)[:, None]
    for i in range(M):
        for j in range(M - 1 - i):
            Y[:, i] *= np.cos(0.5 * np.pi * X[:, j])
        if i > 0:
            Y[:, i] *= np.sin(0.5 * np.pi * X[:, M - 1 - i])
    return Y


# name: (d, N_train, pop, objectives, metric, rank route expected in the truncation)
CASES = {
    # bench.py's shape (DTLZ2, d 30, M 3) at a reduced training set: the merged set is peeled front by front
    "bench_peel": (30, 1024, 65536, "dtlz2", 0, "peel"),
    # objectives = the first three inputs: a uniform cloud, the probe or the forecast hands the rank to the chain
    "uniform_chain": (6, 512, 8192, "cube", 0, "chain"),
    # the population starts on the training inputs: offspring that mutation barely moves have a variance near 0, which AUTO
    # recomputes in float64 (n_ref > 0)
    "refined": (30, 4096, 4096, "dtlz2_on_training", 0, None),
    "crowding": (30, 1024, 8192, "dtlz2", 1, None),
    "euclidean": (30, 1024, 8192, "dtlz2", 2, None),
    "odd_pop": (30, 1024, 8193, "dtlz2", 0, None),
    # merged set below the peel threshold (n < 8192): the chain, no peel
    "small_chain": (30, 1024, 4095, "dtlz2", 0, "chain_only"),
    # the same with crowding: the chain and the crowding distance on the lane beside the variance contraction
    "chain_crowding": (30, 1024, 4095, "dtlz2", 1, "chain_only"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_fused_step_equals_composed_entry_points_with_fewer_waits(L, case):
    import dmosopt_b200 as b2

    d, N, pop, kind, metric, route = CASES[case]
    M = 3
    rng = np.random.default_rng(2026 + len(case))
    xlb, xub = np.zeros(d), np.ones(d)
    Xtr = rng.random((N, d))
    Ytr = Xtr[:, :M].copy() if kind == "cube" else _dtlz2(Xtr, M)
    sm = b2.GPR_Matern(Xtr, Ytr, d, M, xlb, xub, optimizer=None)
    gp = sm._gp
    gp.predict(rng.random((64, d)), return_var=True, precision=L.GP_AUTO)  # calibration and tensor set-up: once per model
    tensor = gp.auto_info()["var_tensor"]
    x0 = Xtr[:pop].copy() if kind == "dtlz2_on_training" else rng.random((pop, d))
    y0 = sm.evaluate(x0).astype(np.float32).astype(np.float64)
    r0 = L.rank_nd(y0).astype(np.int32)
    ref = y0.max(axis=0) + 0.1 * (y0.max(axis=0) - y0.min(axis=0))
    lib, ctx = L.load_library(), L.context()
    DA = L.DeviceArray
    dic, dim = DA((d,)).upload(np.full(d, 1.0)), DA((d,)).upload(np.full(d, 20.0))
    dlb, dub = DA((d,)).upload(xlb), DA((d,)).upload(xub)
    poolsize = pop // 2  # int(round(pop / 2.0)): halves round to even
    if (pop & 1) and (poolsize & 1):
        poolsize += 1
    cap = pop + 1
    fx, fy, fr = DA((pop, d)).upload(x0), DA((pop, M)).upload(y0), DA((pop,), np.int32).upload(r0)
    cx, cy, cr = DA((pop, d)).upload(x0), DA((pop, M)).upload(y0), DA((pop,), np.int32).upload(r0)
    pool, perm, kind_d = DA((poolsize,), np.int64), DA((pop,), np.int64), DA((cap,), np.int32)
    Xs, Ys, var = DA((cap + pop, d)), DA((cap + pop, M)), DA((cap, M))
    nch_f, nch_c = np.zeros(1, dtype=np.int64), np.zeros(1, dtype=np.int64)
    seed, stream = 4242, 10

    def waits_of(fn):
        w0 = L.wait_count()
        fn()
        return L.wait_count() - w0

    refined = []
    for gen in range(3):
        L.profile_enable(True)
        hv_f = ctypes.c_double(0.0)
        w_fused = waits_of(lambda: L._check(lib.dmo_nsga2_step(ctx, gp._h, fx.ptr, fy.ptr, fr.ptr, pop, d, M, 0.9, 0.1, 1.0 / d, dic.ptr, dim.ptr,
                                                                dlb.ptr, dub.ptr, seed, stream + 1, L.GP_AUTO, metric, 1, 1, ref.ctypes.data,
                                                                nch_f.ctypes.data, ctypes.byref(hv_f)), "nsga2_step"))
        refined.append(gp.auto_info()["last_refined"])
        prof = L.profile_report()
        L.profile_enable(False)

        hv_c = ctypes.c_double(0.0)
        w = {}
        w["tournament"] = waits_of(lambda: L._check(lib.dmo_tournament(ctx, cr.ptr, None, pop, poolsize, seed, stream + 1, pool.ptr, None), "tournament"))
        w["generate"] = waits_of(lambda: L._check(lib.dmo_nsga2_generate(ctx, cx.ptr, pop, d, pool.ptr, poolsize, pop, 0.9, 0.1, 1.0 / d, dic.ptr, dim.ptr,
                                                                          dlb.ptr, dub.ptr, seed, stream + 2, Xs.ptr, kind_d.ptr, nch_c.ctypes.data,
                                                                          None), "generate"))
        P = int(nch_c[0])
        w["gp"] = waits_of(lambda: L._check(lib.dmo_gp_predict(ctx, gp._h, Xs.ptr, P, Ys.ptr, var.ptr, L.GP_AUTO), "gp_predict"))
        assert gp.auto_info()["last_refined"] == refined[-1]
        L.memcpy(Xs.offset(P * d), cx.ptr, pop * d * 8)
        L.memcpy(Ys.offset(P * M), cy.ptr, pop * M * 8)
        w["truncate"] = waits_of(lambda: L._check(lib.dmo_remove_worst(ctx, Xs.ptr, Ys.ptr, P + pop, d, M, metric, None, 0, pop, cx.ptr, cy.ptr, cr.ptr,
                                                                       perm.ptr), "remove_worst"))
        L.round_f32(cy.ptr, pop * M)
        w["hv"] = waits_of(lambda: L._check(lib.dmo_hypervolume_ranked(ctx, cy.ptr, pop, M, ref.ctypes.data, cr.ptr, ctypes.byref(hv_c)), "hypervolume"))
        stream += 2

        msg = (case, gen)
        assert int(nch_f[0]) == P, msg
        assert np.array_equal(fx.download(), cx.download()), msg
        assert np.array_equal(fy.download(), cy.download()), msg
        assert np.array_equal(fr.download(), cr.download()), msg
        assert hv_f.value == hv_c.value and hv_f.value > 0.0, (msg, hv_f.value, hv_c.value)

        # composed: tournament 1 (trailing), generate 2 (count + trailing), AUTO predict on the tensor route 2 (one read-back
        # after the contraction + trailing), on the float64 route 1
        assert w["tournament"] == 1 and w["generate"] == 2 and w["gp"] == (2 if tensor else 1), (msg, w)
        # the fused step enqueues the truncation before it reads the GP back; when AUTO then refines rows, it truncates again
        redo = w["truncate"] - 1 if tensor and refined[-1] > 0 else 0
        assert w_fused == sum(w.values()) - 4 + redo, (msg, w_fused, w, refined[-1])
        if route == "peel" and gen == 2:  # the random initial population may still be spread over many fronts
            assert "rank_peel" in prof and "rank_chain" not in prof, (msg, sorted(prof))
            # count + GP + probe + the fronts (at least two) + the hypervolume's route and value
            assert w_fused >= 1 + 1 + 1 + 2 + 2, (msg, w_fused)
        elif route == "chain" and gen == 0:  # the survivors of a generation no longer form a uniform cloud
            assert "rank_chain" in prof, (msg, sorted(prof))
        elif route == "chain_only":
            assert "rank_chain" in prof and "rank_peel" not in prof, (msg, sorted(prof))
    if case == "refined":
        assert tensor and max(refined) > 0, refined
    elif case in ("bench_peel", "crowding", "euclidean", "odd_pop", "chain_crowding"):
        assert tensor, case
