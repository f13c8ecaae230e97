"""Sensitivity analysis on the GPU against a NumPy-only host build of the same designs and statistics.

    python scripts/sa_sweep.py [--N 10000] [--ntrain 4096]

For d in {30, 90} and M in {3, 8} outputs: the three kernels on their own (CUDA events of the library's profile timers),
the NumPy restatement of each step (oracle/sa.py: designs, DGSM statistics with the same 100 bootstrap replicates), and
SA_DGSM.analyze / SA_FAST.analyze end to end against a GPR_Matern surrogate trained on N_train points, next to the same
analysis with the designs and statistics built on the host.  GPR_Matern's predict takes at most 64 inputs, so the
end-to-end rows at d 90 are not measured.  Prints the card name and power limit first.
"""

import argparse
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dmosopt_b200 import _lib as L  # noqa: E402
from oracle import sa as osa  # noqa: E402


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return f"device: {torch.cuda.get_device_properties(0).name}; nvidia-smi: {q.stdout.strip() or q.stderr.strip()}"


def kernel_ms(name, fn, reps=3):
    """Least CUDA-event time of the kernel ``name`` over ``reps`` calls (after one warm-up call)."""
    fn()
    best = math.inf
    for _ in range(reps):
        L.profile_enable(True)
        fn()
        L.synchronize()
        best = min(best, L.profile_report()[name][0])
        L.profile_enable(False)
    return best


def wall_s(fn, reps=2, warm=True):
    if warm:
        fn()
    best = math.inf
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        best = min(best, time.perf_counter() - t)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=10000)
    ap.add_argument("--ntrain", type=int, default=4096)
    ap.add_argument("--dims", type=int, nargs="+", default=[30, 90])
    ap.add_argument("--outputs", type=int, nargs="+", default=[3, 8])
    a = ap.parse_args()
    L.context()
    print(card(), flush=True)
    N, R = a.N, 100
    rng = np.random.default_rng(0)
    for d in a.dims:
        lb, ub = np.zeros(d), np.ones(d)
        B = osa.dgsm_base(N, d)
        w = osa.fast_frequencies(N, d)
        phi = 2 * math.pi * rng.random(d)
        rows_dg, rows_fa = N * (d + 1), N * d
        dev = L.DeviceArray((rows_dg, d))
        lib = L.load_library()
        t_dg = kernel_ms("dgsm_design_kernel", lambda: L._check(lib.dmo_sa_dgsm_design(L.context(), B.ctypes.data, N, d, lb.ctypes.data, ub.ctypes.data, 0.01, dev.ptr), "design"))
        t_fa = kernel_ms("fast_design_kernel", lambda: L._check(lib.dmo_sa_fast_design(L.context(), N, d, w.ctypes.data, phi.ctypes.data, lb.ctypes.data, ub.ctypes.data, dev.ptr), "design"))
        dev.free()
        h_dg = wall_s(lambda: osa.dgsm_design(B, lb, ub), reps=1, warm=False)
        h_fa = wall_s(lambda: osa.fast_design(N, w, phi, lb, ub), reps=1, warm=False)
        print(f"d {d} N {N}: dgsm_design {rows_dg}x{d} ({rows_dg * d * 8 / 1e6:.0f} MB written) kernel {t_dg:.3f} ms "
              f"({rows_dg * d * 8 / t_dg / 1e6:.0f} GB/s) | numpy {h_dg * 1e3:.0f} ms", flush=True)
        print(f"d {d} N {N}: fast_design {rows_fa}x{d} ({rows_fa * d * 8 / 1e6:.0f} MB written) kernel {t_fa:.3f} ms "
              f"({rows_fa * d * 8 / t_fa / 1e6:.0f} GB/s) | numpy {h_fa * 1e3:.0f} ms", flush=True)
        X = L.sa_dgsm_design(B, lb, ub)
        for M in a.outputs:
            Y = np.column_stack([np.sin((k + 1) * X[:, k % d]) + X[:, (k + 1) % d] * X[:, (2 * k + 3) % d] for k in range(M)])
            idx = rng.integers(0, N, size=(R, N), dtype=np.int32)
            Yd = L.DeviceArray(Y.shape).upload(Y)
            t_st = kernel_ms("dgsm_stats_kernel", lambda: L.sa_dgsm_stats(X, Yd, lb, ub, idx))
            g = L.sa_dgsm_stats(X, Y, lb, ub, idx)
            t0 = time.perf_counter()
            o = osa.dgsm_stats(X, Y, lb, ub, idx)
            h_st = time.perf_counter() - t0
            err = max(np.max(np.abs(g[k] - o[k]) / np.maximum(np.abs(o[k]), 1e-300)) for k in ("vi", "dgsm", "conf"))
            print(f"d {d} M {M} N {N} R {R}: dgsm_stats kernel {t_st:.3f} ms | numpy {h_st * 1e3:.0f} ms | max rel. diff {err:.1e}", flush=True)
            Yd.free()
        del X
        for M in a.outputs:
            if d > L.GP_PREDICT_MAX_D:
                print(f"d {d} M {M}: analyze end to end not measured (GPR_Matern predicts at most {L.GP_PREDICT_MAX_D} inputs)", flush=True)
                continue
            e2e(d, M, N, a.ntrain, rng)


def e2e(d, M, N, ntrain, rng):
    import dmosopt_b200 as b2
    from dmosopt_b200.sa import SA_DGSM, SA_FAST

    lb, ub = np.zeros(d), np.ones(d)
    Xt = rng.random((ntrain, d))
    Yt = np.column_stack([np.sin(3 * Xt[:, k % d]) + Xt[:, (k + 1) % d] ** 2 + 0.1 * Xt.sum(axis=1) for k in range(M)])
    sm = b2.GPR_Matern(Xt, Yt, d, M, lb, ub, optimizer=None)
    names, outs = [f"x{i}" for i in range(d)], [f"f{k}" for k in range(M)]
    t_dg = wall_s(lambda: SA_DGSM(lb, ub, names, outs, seed=1).analyze(sm, N))
    t_fa = wall_s(lambda: SA_FAST(lb, ub, names, outs, seed=1).analyze(sm, N))
    # the same analyses with the designs and statistics built on the host (the surrogate still predicts on the GPU)
    idx = np.random.default_rng(1).integers(0, N, size=(100, N), dtype=np.int32)

    def host_dgsm():
        X = osa.dgsm_design(osa.dgsm_base(N, d), lb, ub)
        return osa.dgsm_stats(X, sm.evaluate(X), lb, ub, idx)

    def host_fast():
        X = osa.fast_design(N, osa.fast_frequencies(N, d), 2 * math.pi * np.random.default_rng(1).random(d), lb, ub)
        return osa.fast_indices(sm.evaluate(X), N, d)

    h_dg = wall_s(host_dgsm, reps=1, warm=False)
    h_fa = wall_s(host_fast, reps=1, warm=False)
    print(f"d {d} M {M} N {N} N_train {ntrain}: SA_DGSM.analyze {t_dg * 1e3:.0f} ms (host-built {h_dg * 1e3:.0f} ms) | "
          f"SA_FAST.analyze {t_fa * 1e3:.0f} ms (host-built {h_fa * 1e3:.0f} ms)", flush=True)


if __name__ == "__main__":
    main()
