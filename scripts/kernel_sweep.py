"""GPU micro-timings of the individual hot-path kernels (CUDA events through the library's profile timers)."""
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dmosopt_b200 import _lib as L  # noqa: E402


def timed(fn, reps=3):
    fn()
    L.synchronize()
    best = 1e9
    for _ in range(reps):
        L.timer_begin()
        fn()
        best = min(best, L.timer_end())
    return best


def main():
    L.context()
    rng = np.random.default_rng(0)
    what = sys.argv[1] if len(sys.argv) > 1 else "rank"
    if what == "rank":
        for n, M, kind in [(131072, 3, "uniform"), (131072, 3, "sphere"), (131072, 2, "uniform"), (16384, 2, "uniform"), (65536, 5, "uniform")]:
            Y = rng.random((n, M))
            if kind == "sphere":
                Y = Y / np.linalg.norm(Y, axis=1, keepdims=True) * (1 + 0.01 * rng.random((n, 1)))
            d = L.DeviceArray((n, M)).upload(Y)
            r = L.DeviceArray((n,), np.int32)
            lib, ctx = L.load_library(), L.context()
            L.profile_enable(True)
            ms = timed(lambda: L._check(lib.dmo_rank_nd(ctx, d.ptr, n, M, r.ptr), "rank"))
            rep = L.profile_report()
            L.profile_enable(False)
            rk = r.download()
            print(f"rank n={n} M={M} {kind}: total {ms:.3f} ms, chain {rep['rank_chain'][0] / rep['rank_chain'][1]:.3f} ms, fronts {rk.max() + 1}, OCC={os.environ.get('DMO_RANK_OCC', 'default')}", flush=True)


def gp_sweep():
    """GP posterior at the BASELINE shape: fp64 vs tensor path, accuracy and time, for two models: the reference's
    fixed initial theta for every objective (one shared covariance, as bench.py's model) and three distinct constants
    (1.0, 1.5, 2.0: three covariances).  The executed rate of the variance contraction counts the MMAs issued:
    2 N^2 G flop per candidate for G covariances, times 1.59 for the split-fp16 products over the lower triangle plus the
    diagonal blocks (DESIGN 4.1)."""
    L.context()
    rng = np.random.default_rng(1)
    N, d, M, P = 4096, 30, 3, 65536
    from oracle import gp as ogp

    Xtr = rng.random((N, d))
    Ytr = np.column_stack([np.sin(3 * Xtr[:, :4].sum(axis=1) + k) + Xtr[:, 4 + k] ** 2 for k in range(M)])
    X = rng.random((P, d))
    Xd = L.DeviceArray((P, d)).upload(X)
    md, vd = L.DeviceArray((P, M)), L.DeviceArray((P, M))
    lib, ctx = L.load_library(), L.context()
    print(device_line(), flush=True)
    for label, consts in (("shared theta", [1.0] * M), ("distinct constants", [1.0, 1.5, 2.0])):
        st = ogp.fit_fixed(Xtr, Ytr, np.zeros(d), np.ones(d), consts, 0.5, 1e-6)
        h = L.GPHandle(st.X_train, np.stack([o.alpha for o in st.objectives]), np.stack([o.L for o in st.objectives]), [o.constant for o in st.objectives],
                       [np.full(d, 0.5)] * M, [o.noise for o in st.objectives], [o.y_mean for o in st.objectives], [o.y_std for o in st.objectives],
                       np.zeros(d), np.ones(d))
        G, group_of = h.covariance_groups()
        print(f"== model: {label}, constants {consts}: covariance_groups() = ({G}, {group_of})", flush=True)
        prior = np.array([(o.constant + o.noise) * o.y_std**2 for o in st.objectives])
        ref = None
        for name, prec in (("fp64", L.GP_FP64), ("tensor", L.GP_TENSOR)):
            L.profile_enable(True)
            ms = timed(lambda: L._check(lib.dmo_gp_predict(ctx, h._h, Xd.ptr, P, md.ptr, vd.ptr, prec), "gp"), reps=2)
            rep = L.profile_report()
            L.profile_enable(False)
            mean, var = md.download(), vd.download()
            if ref is None:
                ref = (mean, var)
                err = ""
            else:
                tv = rep["gp_var"][0] / rep["gp_var"][1]
                flop = 2.0 * N * N * G * P * 1.59
                err = (f" | vs fp64: var err/prior {np.max(np.abs(var - ref[1]) / prior):.2e}, mean err {np.max(np.abs(mean - ref[0])):.2e}"
                       f" | contraction executes {flop:.3e} flop: {flop / tv / 1e9:.0f} TFLOP/s")
            parts = ", ".join(f"{k} {v[0] / v[1]:.3f}" for k, v in rep.items())
            print(f"gp {name}: total {ms:.3f} ms [{parts}]{err}", flush=True)
        kstar_sweep(lib, ctx, h, Xd, md, vd, P, N, G)
        h.close()


def device_line():
    import subprocess

    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return f"device: {torch.cuda.get_device_properties(0).name}; nvidia-smi: {q.stdout.strip() or q.stderr.strip()}"


def write_floor_ms(nbytes, reps=5):
    """A write-only floor for `nbytes`: one plain store kernel (torch's fill over a contiguous byte buffer), CUDA events."""
    import torch

    buf = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    buf.fill_(1)
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        buf.fill_(0)
        e1.record()
        e1.synchronize()
        best = min(best, e0.elapsed_time(e1))
    del buf
    torch.cuda.empty_cache()
    return best


def kstar_sweep(lib, ctx, h, Xd, md, vd, P, N, G):
    """K_* producer of the tensor predict, both routes (DMO_GP_FUSED=1: K_* and the mean from one kernel; 0: K_* kernel
    then the mean read back from K_*): time, bytes of K_* written (fp16 hi + lo, one plane of Pcpad x Npad per covariance:
    4 G Pcpad Npad bytes) and the achieved rate, next to a write-only floor over the same bytes measured in the same
    process."""
    Npad = -(-N // 256) * 256
    Pcpad = -(-P // 256) * 256
    kbytes = 4 * G * Pcpad * Npad
    floor = write_floor_ms(kbytes)
    print(f"write-only floor (one store kernel over {kbytes / 1e9:.3f} GB): {floor:.3f} ms = {kbytes / floor / 1e6:.0f} GB/s", flush=True)
    saved = os.environ.get("DMO_GP_FUSED")
    outs = {}
    for fused in ("1", "0"):
        os.environ["DMO_GP_FUSED"] = fused
        L.profile_enable(True)
        ms = timed(lambda: L._check(lib.dmo_gp_predict(ctx, h._h, Xd.ptr, P, md.ptr, vd.ptr, L.GP_TENSOR), "gp"), reps=3)
        rep = L.profile_report()
        L.profile_enable(False)
        outs[fused] = (md.download(), vd.download())
        ks = rep["gp_kstar"][0] / rep["gp_kstar"][1]
        mean = f", gp_mean {rep['gp_mean'][0] / rep['gp_mean'][1]:.3f} ms" if "gp_mean" in rep else ""
        print(f"tensor predict DMO_GP_FUSED={fused}: total {ms:.3f} ms; gp_kstar {ks:.3f} ms{mean}; K_* written {kbytes / 1e9:.3f} GB "
              f"-> {kbytes / ks / 1e6:.0f} GB/s ({floor / ks:.2f} of the write-only floor's rate)", flush=True)
    if saved is None:
        del os.environ["DMO_GP_FUSED"]
    else:
        os.environ["DMO_GP_FUSED"] = saved
    (m1, v1), (m0, v0) = outs["1"], outs["0"]
    print(f"routes agree: var bit-identical {np.array_equal(v1, v0)}, max |mean difference| {np.max(np.abs(m1 - m0)):.2e}", flush=True)


def mtgp_sweep():
    """MEGP_Matern's multitask posterior (dmo_mtgp_predict, tensor and fp64) next to GPR_Matern's tensor predict at the
    same shape (P = 65536, N = 4096, M = 3, d = 30), with the K_* bytes each writes per predict."""
    import torch

    L.context()
    rng = np.random.default_rng(3)
    N, d, M, P = 4096, 30, 3, 65536
    Npad = -(-N // 256) * 256
    Xtr = rng.random((N, d))
    Ytr = np.column_stack([np.sin(3 * Xtr[:, :4].sum(axis=1) + k) + Xtr[:, 4 + k] ** 2 for k in range(M)])
    yn = (Ytr - Ytr.mean(0)) / Ytr.std(0)
    ls = np.full(d, 0.5)
    # GPR_Matern: M independent GPs (fitted on the GPU for fixed hyper-parameters)
    Lf, alpha, _ = L.gp_fit(Xtr, yn.T, [1.0] * M, [ls] * M, [1e-3] * M, jitter=0.0)
    gpr = L.GPHandle(Xtr, alpha, Lf, [1.0] * M, [ls] * M, [1e-3] * M, Ytr.mean(0), Ytr.std(0), np.zeros(d), np.ones(d))
    # MEGP_Matern: one multitask GP, rank-1 task covariance plus diagonal
    F = np.array([[0.8], [0.5], [-0.4]])
    B = F @ F.T + np.diag([0.3, 0.4, 0.5])
    mt = L.MTGPHandle(Xtr, yn, ls, B, np.full(M, 2e-3), np.zeros((M, d)), np.zeros(M), Ytr.mean(0), Ytr.std(0), np.zeros(d), np.ones(d))
    X = rng.random((P, d))
    Xd = L.DeviceArray((P, d)).upload(X)
    md, vd = L.DeviceArray((P, M)), L.DeviceArray((P, M))
    lib, ctx = L.load_library(), L.context()
    import subprocess

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"device: {torch.cuda.get_device_properties(0).name}; nvidia-smi: {q.stdout.strip() or q.stderr.strip()}", flush=True)
    out = {}
    G = gpr.covariance_groups()[0]  # one K_* plane per distinct covariance
    runs = (("GPR_Matern tensor", lambda: lib.dmo_gp_predict(ctx, gpr._h, Xd.ptr, P, md.ptr, vd.ptr, L.GP_TENSOR), G * P * Npad * 4),
            ("MEGP_Matern tensor", lambda: lib.dmo_mtgp_predict(ctx, mt._h, Xd.ptr, P, md.ptr, vd.ptr, L.GP_TENSOR), P * Npad * 4),
            ("MEGP_Matern fp64", lambda: lib.dmo_mtgp_predict(ctx, mt._h, Xd.ptr, P, md.ptr, vd.ptr, L.GP_FP64), P * Npad * 8))
    for name, fn, kbytes in runs:
        L.profile_enable(True)
        ms = timed(lambda: L._check(fn(), name), reps=3)
        rep = L.profile_report()
        L.profile_enable(False)
        out[name] = (md.download(), vd.download())
        parts = ", ".join(f"{k} {v[0] / v[1]:.3f}" for k, v in rep.items())
        print(f"{name} P={P} N={N} M={M} d={d}: total {ms:.3f} ms [{parts}]; K_* written per predict {kbytes / 1e9:.3f} GB", flush=True)
    (mt_t, vt_t), (mt_f, vt_f) = out["MEGP_Matern tensor"], out["MEGP_Matern fp64"]
    prior = (np.diag(B) + 2e-3) * Ytr.std(0) ** 2
    print(f"MEGP tensor vs fp64: mean err / max|mean| {np.max(np.abs(mt_t - mt_f) / np.abs(mt_f).max(0)):.2e}, "
          f"var err / prior {np.max(np.abs(vt_t - vt_f) / prior):.2e}", flush=True)


def mtgp_fit_sweep():
    """MEGP_Matern training: one dmo_mtgp_lml_grad evaluation (median of warm calls, CUDA events per phase) for
    N in {1024, 2048, 4096}, M in {2, 3}, d = 30, with the counted float64 work (block Cholesky, triangular inverse and
    the sum of lambda_j A_j^-1: about M N^3 flop; gradient pass: about N^2 (2 d + M^2) flop), then one default megp_fit
    on ZDT1 data (d = 30, M = 2, N = 2048)."""
    from dmosopt_b200.model_gpytorch import megp_fit, megp_initial_raw, megp_natural, normalise_targets

    L.context()
    print(device_line(), flush=True)
    rng = np.random.default_rng(4)
    d = 30
    for N in (1024, 2048, 4096):
        for M in (2, 3):
            X = rng.random((N, d))
            Y = np.column_stack([np.sin(3 * X[:, :4].sum(axis=1) + k) + X[:, 4 + k] ** 2 for k in range(M)])
            yn, _, _ = normalise_targets(Y)
            ls, B, D, w, b = megp_natural(megp_initial_raw(d, M, seed=1))
            L.mtgp_lml_grad(X, yn, ls, B, D, w, b)  # warm-up
            L.profile_enable(True)
            walls = []
            for _ in range(5):
                L.timer_begin()
                L.mtgp_lml_grad(X, yn, ls, B, D, w, b)
                walls.append(L.timer_end())
            rep = L.profile_report()
            L.profile_enable(False)
            ph = {k: rep[k][0] / rep[k][1] for k in ("mtgp_lg_fit", "mtgp_lg_linv", "mtgp_lg_ainv", "mtgp_lg_grad") if k in rep}
            ms = float(np.median(walls))
            f3 = M * float(N) ** 3
            f2 = float(N) ** 2 * (2 * d + M * M)
            dense = ph["mtgp_lg_fit"] + ph["mtgp_lg_linv"] + ph["mtgp_lg_ainv"]
            parts = ", ".join(f"{k[8:]} {v:.2f} ms" for k, v in ph.items())
            print(f"mtgp_lml_grad N={N} M={M} d={d}: {ms:.2f} ms median of 5 [{parts}]; gradient pass {100 * ph['mtgp_lg_grad'] / ms:.1f} % "
                  f"of the call; M N^3 = {f3 / 1e9:.1f} GFLOP in {dense:.2f} ms = {f3 / dense / 1e9:.2f} TFLOP/s fp64 "
                  f"(Sigma lambda A^-1 alone: {f3 / 3 / ph['mtgp_lg_ainv'] / 1e9:.2f} TFLOP/s); N^2 (2d + M^2) = {f2 / 1e9:.2f} GFLOP "
                  f"in {ph['mtgp_lg_grad']:.2f} ms", flush=True)
    N, M = 2048, 2
    X = rng.random((N, d))
    g = 1.0 + 9.0 / (d - 1) * X[:, 1:].sum(axis=1)
    Y = np.column_stack((X[:, 0], g * (1.0 - np.sqrt(X[:, 0] / g))))
    yn, _, _ = normalise_targets(Y)
    t0 = time.perf_counter()
    hp, info = megp_fit(X, yn)
    wall = time.perf_counter() - t0
    print(f"megp_fit ZDT1 N={N} M={M} d={d} (defaults: lr 0.01, n_iter 5000): {info['iterations']} iterations, {wall:.1f} s "
          f"({1e3 * wall / info['iterations']:.1f} ms per iteration), loss {info['loss'][0]:.4f} -> {info['loss'][-1]:.4f}, "
          f"stop: {info['stop_reason']}", flush=True)


def egp_fit_sweep():
    """EGP_Matern training: one dmo_gp_lml_grad evaluation over M objectives (median of 5 warm calls, CUDA events per
    phase) for N in {1024, 2048, 4096}, M in {1, 2, 3}, d = 30, with the counted float64 work (Cholesky, triangular
    inverse and K^-1: about M N^3 flop), beside the same objectives as M one-task dmo_mtgp_lml_grad calls (the
    one-objective-at-a-time route), then one default egp_fit on ZDT1 data (d = 30, M = 2, N = 2048)."""
    from dmosopt_b200.model_gpytorch import egp_fit, egp_initial_raw, egp_natural

    L.context()
    print(device_line(), flush=True)
    rng = np.random.default_rng(5)
    d = 30
    phases = ("gp_lg_fit", "gp_lg_linv", "gp_lg_ainv", "gp_lg_grad")
    for N in (1024, 2048, 4096):
        X = rng.random((N, d))
        Y = np.column_stack([np.sin(3 * X[:, :4].sum(axis=1) + k) + X[:, 4 + k] ** 2 for k in range(3)])
        yn = (Y - Y.mean(0)) / Y.std(0)
        for M in (1, 2, 3):
            ls, s, nz, w, b = egp_natural(egp_initial_raw(d, M, seed=1))
            L.gp_lml_grad(X, yn[:, :M], ls, s, nz, w, b)  # warm-up
            L.profile_enable(True)
            walls = []
            for _ in range(5):
                L.timer_begin()
                L.gp_lml_grad(X, yn[:, :M], ls, s, nz, w, b)
                walls.append(L.timer_end())
            rep = L.profile_report()
            L.profile_enable(False)
            ph = {k: rep[k][0] / rep[k][1] for k in phases if k in rep}
            ms = float(np.median(walls))

            def one_task_calls():
                for m in range(M):
                    L.mtgp_lml_grad(X, yn[:, m], ls[m], np.array([[s[m]]]), nz[m : m + 1], w[m : m + 1], b[m : m + 1])

            one_task_calls()  # warm-up
            walls1 = []
            for _ in range(5):
                L.timer_begin()
                one_task_calls()
                walls1.append(L.timer_end())
            ms1 = float(np.median(walls1))
            f3 = M * float(N) ** 3
            dense = ph["gp_lg_fit"] + ph["gp_lg_linv"] + ph["gp_lg_ainv"]
            parts = ", ".join(f"{k[6:]} {v:.2f} ms" for k, v in ph.items())
            print(f"gp_lml_grad N={N} M={M} d={d}: {ms:.2f} ms median of 5 [{parts}]; M N^3 = {f3 / 1e9:.1f} GFLOP in {dense:.2f} ms = "
                  f"{f3 / dense / 1e9:.2f} TFLOP/s fp64 | {M} one-task mtgp_lml_grad calls: {ms1:.2f} ms median of 5 "
                  f"({ms1 / ms:.2f}x the batched call)", flush=True)
    N, M = 2048, 2
    X = rng.random((N, d))
    g = 1.0 + 9.0 / (d - 1) * X[:, 1:].sum(axis=1)
    Y = np.column_stack((X[:, 0], g * (1.0 - np.sqrt(X[:, 0] / g))))
    yn = (Y - Y.mean(0)) / Y.std(0)
    t0 = time.perf_counter()
    hp, info = egp_fit(X, yn)
    wall = time.perf_counter() - t0
    its = [i["iterations"] for i in info]
    print(f"egp_fit ZDT1 N={N} M={M} d={d} (defaults: lr 0.01, n_iter 5000): iterations per output {its}, {wall:.1f} s "
          f"({1e3 * wall / max(its):.1f} ms per lockstep iteration); stop: {[i['stop_reason'] for i in info]}", flush=True)


def svgp_fit_sweep(n_iter=None):
    """Variational training: per-call times (median of 5 warm calls, host clock around calls that end in a device
    synchronise) of dmo_svgp_fit_natgrad and dmo_svgp_fit_elbo_grad at d = 30, B = 50 for Z in {256, 512, 819, 1024, 2048}
    and L in {1, 3}, and of the VGP form at N in {1024, 2048, 4096}; then one fit of each class on ZDT1 data (N 2048, d 30,
    M 2) with the reference's defaults (n_iter: the reference's per class unless given)."""
    from dmosopt_b200 import model_gpflow as mg

    L.context()
    print(device_line(), flush=True)
    rng = np.random.default_rng(6)
    d, B = 30, 50

    def med(f):
        f()
        ts = []
        for _ in range(5):
            t0 = time.perf_counter()
            f()
            ts.append(time.perf_counter() - t0)
        return 1e3 * float(np.median(ts))

    for Zn in (256, 512, 819, 1024, 2048):
        N = max(4096, Zn)
        X = rng.random((N, d))
        for Lat in (1, 3):
            Y = np.column_stack([np.sin(3 * X[:, :4].sum(1) + k) for k in range(Lat)])
            st = L.SVGPFitState(X, Y, X[:Zn], Lat)
            s, ls, nz = np.ones(Lat), np.full((Lat, d), 1.0 + 0.1 * np.arange(Lat)[:, None]), np.full(Lat, 1e-2)
            b = rng.permutation(N)[:B]
            t_ng = med(lambda: st.natgrad(b, s, ls, nz, gamma=0.1))
            t_eg = med(lambda: st.elbo_grad(b, s, ls, nz))
            print(f"svgp_fit Z={Zn} L={Lat} d={d} B={B}: natgrad {t_ng:.2f} ms, elbo_grad {t_eg:.2f} ms", flush=True)
    for N in (1024, 2048, 4096):
        X = rng.random((N, d))
        Y = np.sin(3 * X[:, :4].sum(1))[:, None]
        st = L.SVGPFitState(X, Y, None, 1, inducing_is_data=True)
        s, ls, nz, b = np.ones(1), np.ones((1, d)), np.full(1, 1e-2), np.arange(N)
        t_ng = med(lambda: st.natgrad(b, s, ls, nz, gamma=1.0))
        t_eg = med(lambda: st.elbo_grad(b, s, ls, nz))
        print(f"vgp_fit N={N} d={d}: natgrad {t_ng:.2f} ms, elbo_grad {t_eg:.2f} ms", flush=True)
    N, M = 2048, 2
    X = rng.random((N, d))
    g = 1.0 + 9.0 / (d - 1) * X[:, 1:].sum(axis=1)
    Y = np.column_stack((X[:, 0], g * (1.0 - np.sqrt(X[:, 0] / g))))
    for cls in ("SVGP_Matern", "VGP_Matern", "SIV_Matern", "SPV_Matern", "CRV_Matern"):
        kw = {} if n_iter is None else {"n_iter": n_iter}
        t0 = time.perf_counter()
        m = getattr(mg, cls)(X, Y, d, M, np.zeros(d), np.ones(d), seed=1, fit="gpu", **kw)
        wall = time.perf_counter() - t0
        fi = m.fit_info
        print(f"{cls} fit ZDT1 N={N} d={d} M={M}{'' if n_iter is None else f' n_iter={n_iter}'}: iterations {fi['iterations']}, "
              f"stop {fi['stop_reason']}, {wall:.1f} s, ELBO {[round(float(e[-1]), 1) for e in fi['elbo']]}", flush=True)


def stream_sweep():
    """The HBM-bound kernels at the BASELINE shape: crowding / euclidean distance (n = 131072, M = 3), SBX + mutation
    (pop 65536, d 30), mean kernel's neighbours, hypervolume of a 65536-point 3-D front.  Prints time and the achieved
    fraction of the algorithmic bytes."""
    L.context()
    rng = np.random.default_rng(2)
    lib, ctx = L.load_library(), L.context()
    n, M = 131072, 3
    Y = L.DeviceArray((n, M)).upload(rng.random((n, M)))
    D = L.DeviceArray((n,))
    for name, fn in (("crowding", lib.dmo_crowding_distance), ("euclidean", lib.dmo_euclidean_distance)):
        ms = timed(lambda: L._check(fn(ctx, Y.ptr, n, M, D.ptr), name))
        print(f"{name} n={n} M={M}: {ms:.3f} ms; minimum bytes 8nM + 8n = {(8 * n * M + 8 * n) / 1e6:.1f} MB -> {(8 * n * M + 8 * n) / ms / 1e6:.1f} GB/s on the algorithmic bytes", flush=True)
    pop, d = 65536, 30
    X = L.DeviceArray((pop, d)).upload(rng.random((pop, d)))
    pool = L.DeviceArray((pop // 2,), np.int64).upload(rng.permutation(pop)[: pop // 2].astype(np.int64))
    Xg = L.DeviceArray((pop + 1, d))
    kind = L.DeviceArray((pop + 1,), np.int32)
    nch = np.zeros(1, dtype=np.int64)
    one, twenty = L.DeviceArray((d,)).upload(np.full(d, 1.0)), L.DeviceArray((d,)).upload(np.full(d, 20.0))
    lb, ub = L.DeviceArray((d,)).upload(np.zeros(d)), L.DeviceArray((d,)).upload(np.ones(d))
    ms = timed(lambda: L._check(lib.dmo_nsga2_generate(ctx, X.ptr, pop, d, pool.ptr, pop // 2, pop, 0.9, 0.1, 1.0 / d, one.ptr, twenty.ptr, lb.ptr, ub.ptr,
                                                      7, 1, Xg.ptr, kind.ptr, nch.ctypes.data, None), "generate"))
    by = 8 * d * 2 * int(nch[0])
    print(f"variation pop={pop} d={d}: {ms:.3f} ms for {int(nch[0])} children; 8d B read + 8d B written per child = {by / 1e6:.1f} MB -> {by / ms / 1e6:.1f} GB/s", flush=True)
    x = rng.random((pop, 3))
    F = L.DeviceArray((pop, 3)).upload(x / np.linalg.norm(x, axis=1, keepdims=True))
    import ctypes

    out = ctypes.c_double(0.0)
    ref = np.full(3, 1.1)
    ms = timed(lambda: L._check(lib.dmo_hypervolume(ctx, F.ptr, pop, 3, ref.ctypes.data, ctypes.byref(out)), "hv"), reps=2)
    print(f"hypervolume n={pop} M=3 (whole set non-dominated): {ms:.3f} ms, value {out.value:.6f}", flush=True)


def svgp_sweep():
    """The variational posterior (dmo_svgp_predict, fp64 and tensor) at P = 65536, d = 30, M = 3: SVGP with Z = 819 (its
    round(0.2 N) at N = 4096, its own Z per output: 3 K_* planes, 6 operator planes) and VGP with Z = N = 4096 (one K_*
    plane; one Lz^-1 shared by the outputs plus 3 q operators: 4 planes), both with q at its optimum; next to
    dmo_gp_predict with three distinct covariances (3 planes of N = 4096) in the same run.  Per plane: the variance
    contraction's time over the operator planes it walks.  Also the create time (Householder QR per latent) and
    dmo_svgp_optimal_q at N = 4096."""
    L.context()
    rng = np.random.default_rng(5)
    N, d, M, P = 4096, 30, 3, 65536
    Xtr = rng.random((N, d))
    Ytr = np.column_stack([np.sin(3 * Xtr[:, :4].sum(axis=1) + k) + Xtr[:, 4 + k] ** 2 for k in range(M)])
    yn = (Ytr - Ytr.mean(0)) / Ytr.std(0)
    ls, s = np.full((M, d), 0.5 * np.sqrt(d / 4)), np.ones(M)
    X = rng.random((P, d))
    Xd = L.DeviceArray((P, d)).upload(X)
    md, vd = L.DeviceArray((P, M)), L.DeviceArray((P, M))
    lib, ctx = L.load_library(), L.context()
    print(device_line(), flush=True)
    # GPR_Matern reference: three covariances (constants 1.0, 1.5, 2.0)
    cs = [1.0, 1.5, 2.0]
    Lf, alpha, _ = L.gp_fit(Xtr, yn.T, cs, [ls[0]] * M, [1e-3] * M, jitter=0.0)
    gpr = L.GPHandle(Xtr, alpha, Lf, cs, [ls[0]] * M, [1e-3] * M, Ytr.mean(0), Ytr.std(0), np.zeros(d), np.ones(d))
    models = [("GPR_Matern", None, gpr.covariance_groups()[0],
               lambda prec: lib.dmo_gp_predict(ctx, gpr._h, Xd.ptr, P, md.ptr, vd.ptr, prec), "gp_var")]
    for name, Zn in (("SVGP_Matern", 819), ("VGP_Matern", N)):
        vgp = Zn == N
        Z = np.stack([Xtr] * M) if vgp else np.stack([Xtr[rng.choice(N, Zn, replace=False)] for _ in range(M)])
        t0 = time.perf_counter()
        qm, qs = L.svgp_optimal_q(Xtr, yn.T, None if vgp else Z, s, ls, np.full(M, 1e-3), inducing_is_data=vgp)
        t_q = time.perf_counter() - t0
        t0 = time.perf_counter()
        h = L.SVGPHandle(Z, s, ls, qm, qs, Ytr.mean(0), Ytr.std(0), np.zeros(d), np.ones(d))
        t_c = time.perf_counter() - t0
        groups, planes = h.groups()
        print(f"{name} N={N} Z={Zn}: dmo_svgp_optimal_q {t_q * 1e3:.1f} ms, dmo_svgp_create {t_c * 1e3:.1f} ms; "
              f"{groups} K_* planes, {planes} operator planes", flush=True)
        models.append((name, h, planes, lambda prec, h=h: lib.dmo_svgp_predict(ctx, h._h, Xd.ptr, P, md.ptr, vd.ptr, prec), "svgp_var"))
    out = {}
    for name, _, planes, fn, var_key in models:
        for prec, pname in ((L.GP_FP64, "fp64"), (L.GP_TENSOR, "tensor")):
            L.profile_enable(True)
            ms = timed(lambda: L._check(fn(prec), name), reps=3)
            rep = L.profile_report()
            L.profile_enable(False)
            out[(name, pname)] = (md.download(), vd.download())
            vms = rep[var_key][0] / rep[var_key][1] if var_key in rep else float("nan")
            parts = ", ".join(f"{k} {v[0] / v[1]:.3f}" for k, v in rep.items())
            print(f"{name} {pname} P={P} d={d} M={M}: total {ms:.3f} ms [{parts}]; variance contraction per operator plane "
                  f"{vms / planes:.3f} ms ({planes} planes)", flush=True)
    for name in ("SVGP_Matern", "VGP_Matern"):
        (mf, vf), (mt, vt) = out[(name, "fp64")], out[(name, "tensor")]
        print(f"{name} tensor vs fp64: mean err / max|mean| {np.max(np.abs(mt - mf) / np.abs(mf).max(0)):.2e}, "
              f"var err / prior {np.max(np.abs(vt - vf) / Ytr.std(0) ** 2):.2e}", flush=True)


def deepgp_sweep():
    """The deep GP predict (dmo_dgp_predict) at P = 65536, d = 30, H = 3, T = 3, Z1 = Z2 = 128: MDSPP at J 3 and 8, MDGP at
    J 10, fp64 and tensor.  Per predict: the hidden layer (ProfileScope dgp_hidden: the dmo_svgp latent moments and the
    epilogue) and the layer-2 kernel (dgp_layer2) timed apart.  The layer-2 rate counts the useful work, 2 Z2^2 flop per
    (site, candidate, task): the two triangular mat-vecs; K_* and the mean are not counted."""
    L.context()
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from test_deepgp_cpu import problem

    rng = np.random.default_rng(7)
    P, d, H, T, Z = 65536, 30, 3, 3, 128
    lib, ctx = L.load_library(), L.context()
    print(device_line(), flush=True)
    X = rng.random((P, d))
    Xd = L.DeviceArray((P, d)).upload(X)
    md, vd = L.DeviceArray((P, T)), L.DeviceArray((P, T))
    for label, J, quad in (("MDSPP", 3, True), ("MDSPP", 8, True), ("MDGP", 10, False)):
        hp, ym, ys, _, _ = problem(rng, d, H, T, Z, Z, J=J, quadrature=quad)
        g = L.DGPHandle(hp["hidden_inducing_points"], hp["hidden_outputscale"], hp["hidden_lengthscale"], hp["hidden_variational_mean"],
                        np.tril(hp["hidden_chol_variational_covar"]), hp["mean_weights"], hp["mean_bias"], hp["last_inducing_points"],
                        hp["last_outputscale"], hp["last_lengthscale"], hp["last_variational_mean"],
                        np.tril(hp["last_chol_variational_covar"]), hp["mean_constant"], hp["task_noises"] + hp["noise"], ym, ys, np.zeros(d),
                        np.ones(d), quad_sites=hp["quad_sites"] if quad else None, n_sites=J)
        flop = 2.0 * Z * Z * J * P * T
        for pname, prec in (("fp64", L.GP_FP64), ("tensor", L.GP_TENSOR)):
            L.profile_enable(True)
            ms = timed(lambda: L._check(lib.dmo_dgp_predict(ctx, g._h, Xd.ptr, P, 1, 0, None, md.ptr, vd.ptr, prec), "dgp"), reps=5)
            rep = L.profile_report()
            L.profile_enable(False)
            hid = rep["dgp_hidden"][0] / rep["dgp_hidden"][1]
            l2 = rep["dgp_layer2"][0] / rep["dgp_layer2"][1]
            print(f"{label} J={J} {pname} P={P} d={d} H={H} T={T} Z1=Z2={Z}: predict {ms:.3f} ms; hidden layer {hid:.3f} ms, "
                  f"layer-2 kernel {l2:.3f} ms = {flop / l2 / 1e9:.2f} TFLOP/s useful ({flop:.3e} flop)", flush=True)
        g.close()


def deepgp_fit_sweep(n_epochs=200):
    """Deep GP training (dmo_dgp_fit) at N = 1000, d = 30, H = 3, T = 3, Z1 = Z2 = 128: MDSPP at B 10 (J 3 sites) and MDGP
    at B 50 (J = B = 50 draws per row).  Per configuration: the time of one epoch (dmo_dgp_fit_epoch: every loss_grad and
    Adam step, no host synchronisation inside) and of one step, the launches per step, the last layer's kernels timed
    apart (ProfileScope dgp_fit_last_fwd / dgp_fit_last_bwd / dgp_fit_gram) with their FP64 rate, and one capped
    deepgp_fit of n_epochs epochs.  The last-layer flop count from shapes, R = J B rows per task: the forward solve and
    Lq' a (2 R T Z^2), the backward Lq g and back solve (2 R T Z^2) and the lower halves of the two Gram products
    (2 R T Z^2)."""
    from dmosopt_b200 import model_gpytorch as mg

    L.context()
    print(device_line(), flush=True)
    rng = np.random.default_rng(3)
    N, d, H, T, Z = 1000, 30, 3, 3, 128
    X = rng.random((N, d))
    g = 1.0 + 9.0 / (d - 1) * X[:, 1:].sum(axis=1)
    Y = np.column_stack((X[:, 0], g * (1.0 - np.sqrt(X[:, 0] / g)), X[:, 0] * X[:, 1] + X[:, 2]))
    Y = (Y - Y.mean(0)) / Y.std(0)
    for label, quad, B in (("MDSPP", True, 10), ("MDGP", False, 50)):
        J = 3 if quad else B
        raw = mg.deepgp_initial_raw(X, T, quadrature=quad, num_hidden_dims=H, num_inducing_points=Z, rng=np.random.default_rng(1))
        st = L.DGPFitState(X, Y, H, Z, Z, J, quad, B)
        st.set_params(mg.deepgp_flatten(raw))
        perm = rng.permutation(N)
        nb = -(-N // B)
        st.epoch(perm, B, 0.01)  # warm-up
        n0 = L.launch_count()
        st.epoch(perm, B, 0.01)
        per_step = (L.launch_count() - n0) / nb
        L.synchronize()
        times = []
        for _ in range(3):
            t0 = time.perf_counter()
            st.epoch(perm, B, 0.01)  # ends in a device synchronise
            times.append((time.perf_counter() - t0) * 1e3)
        ms = min(times)
        L.profile_enable(True)
        st.epoch(perm, B, 0.01)
        rep = L.profile_report()
        L.profile_enable(False)
        R = J * B
        flop = 6.0 * R * T * Z * Z
        kms = {k: rep[k][0] / rep[k][1] for k in ("dgp_fit_last_fwd", "dgp_fit_last_bwd", "dgp_fit_gram")}
        last = sum(kms.values())
        parts = ", ".join(f"{k[8:]} {v:.3f} ms" for k, v in kms.items())
        print(f"{label} N={N} d={d} H={H} T={T} Z={Z} B={B} J={J}: epoch {ms:.2f} ms ({nb} steps), step {ms / nb:.3f} ms, "
              f"{per_step:.1f} launches per step; last layer per step {last:.3f} ms [{parts}] = "
              f"{flop / last / 1e9:.2f} TFLOP/s FP64 ({flop:.3e} flop)", flush=True)
        st.close()
        t0 = time.perf_counter()
        _, info = mg.deepgp_fit(X, Y, quadrature=quad, num_hidden_dims=H, num_inducing_points=Z, n_iter=n_epochs, batch_size=B, seed=0)
        s = time.perf_counter() - t0
        print(f"{label} deepgp_fit capped at {n_epochs} epochs: {s:.1f} s ({info['iterations']} epochs, {info['iterations'] * nb} steps), "
              f"loss {info['loss'][0]:.4f} -> {info['loss'][-1]:.4f}, final lr {info['lr'][-1]:g}", flush=True)


def many_sweep():
    """Many-objective runs.  (1) Rank (dmo_rank_nd) and truncation to half (dmo_remove_worst, no metric) at n = 131072,
    M 10 and 16, on bench.objective_sets' uniform and sphere sets, device-resident, CUDA events.  (2) dmo_hypervolume_mc
    per algorithm (epsilon 0.01, delta 0.25, 100000 monte_carlo points) on sphere fronts of 1000, 4000 and 16000 points,
    M 10 and 16, ref 1.1: host time of the whole call (it ends in a device synchronise), samples, dominance tests and
    tests/s, and the rate of the front-row bytes those tests read (M float64 each).  (3) The reference's
    compute_hypervolume_hybrid (oracle/_ref, on the host) at epsilon 0.05 on a 200-point front, with the GPU's hybrid on the
    same front and settings."""
    import bench

    L.context()
    print(device_line(), flush=True)
    lib, ctx = L.load_library(), L.context()
    n = 131072
    for M in (10, 16):
        for kind, Y in bench.objective_sets(n, M).items():
            d = L.DeviceArray((n, M)).upload(Y)
            x = L.DeviceArray((n, 1)).upload(np.zeros((n, 1)))
            r = L.DeviceArray((n,), np.int32)
            keep = n // 2
            perm = L.DeviceArray((keep,), np.int64)
            ms_rank = timed(lambda: L._check(lib.dmo_rank_nd(ctx, d.ptr, n, M, r.ptr), "rank"))
            ms_trunc = timed(lambda: L._check(lib.dmo_remove_worst(ctx, x.ptr, d.ptr, n, 1, M, L.METRIC_NONE, None, 0, keep, None, None, None,
                                                                   perm.ptr), "remove_worst"))
            rk = r.download()
            print(f"rank n={n} M={M} {kind}: {ms_rank:.3f} ms ({rk.max() + 1} fronts, {int((rk == 0).sum())} in front 0); "
                  f"truncation to {keep}: {ms_trunc:.3f} ms", flush=True)
    for M in (10, 16):
        for nf in (1000, 4000, 16000):
            F = bench.objective_sets(nf, M)["sphere"]
            ref = np.full(M, 1.1)
            for algo in ("hybrid", "fpras", "mcm2rv", "monte_carlo"):
                L.hypervolume_mc(F, ref, algo, 0.01, 0.25, seed=1, stream=0)  # warm-up
                t0 = time.perf_counter()
                v, info = L.hypervolume_mc(F, ref, algo, 0.01, 0.25, seed=1, stream=1)
                s = time.perf_counter() - t0
                rate = info["tests"] / s
                print(f"hv_mc n={nf} M={M} {algo}: {s * 1e3:.1f} ms, value {v:.6g}, ran {info['algorithm']}, samples {info['samples']}, "
                      f"tests {info['tests']:.3e}, {rate:.3e} tests/s, front-row reads {rate * M * 8 / 1e9:.1f} GB/s", flush=True)
    from oracle import reference_build

    path = reference_build.reference_path()
    if path is None:
        print("reference hybrid: not measured (oracle/_ref not built)", flush=True)
        return
    sys.path.insert(0, path)
    import contextlib
    import io

    from dmosopt import hv_adaptive

    for M in (10, 16):
        F = bench.objective_sets(200, M)["sphere"]
        ref = np.full(M, 1.1)
        t0 = time.perf_counter()
        v, info = L.hypervolume_mc(F, ref, "hybrid", 0.05, 0.25, seed=1, stream=2)
        s_gpu = time.perf_counter() - t0
        np.random.seed(0)
        t0 = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):  # the reference prints once per MCM2RV iteration
            res = hv_adaptive.compute_hypervolume_hybrid(F, ref, 0.05, 0.25)
        s_ref = time.perf_counter() - t0
        print(f"hybrid n=200 M={M} eps 0.05: GPU {s_gpu * 1e3:.1f} ms ({info['algorithm']}, {v:.6g}); reference on the host "
              f"{s_ref * 1e3:.1f} ms ({res.algorithm_used}, {res.hypervolume:.6g}, {res.num_comparisons} comparisons)", flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "many":
        many_sweep()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "deepgp_fit":
        deepgp_fit_sweep(int(sys.argv[2]) if len(sys.argv) > 2 else 200)
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "deepgp":
        deepgp_sweep()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "stream":
        stream_sweep()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "gp":
        gp_sweep()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "mtgp":
        mtgp_sweep()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "mtgp_fit":
        mtgp_fit_sweep()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "svgp":
        svgp_sweep()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "egp_fit":
        egp_fit_sweep()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "svgp_fit":
        svgp_fit_sweep(int(sys.argv[2]) if len(sys.argv) > 2 else None)
        sys.exit(0)
    main()
