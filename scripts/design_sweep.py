"""Good-lattice-point search on the GPU, phase by phase, against the reference's own ``sampling.glp``.

    python scripts/design_sweep.py [--dims 15 30 40 60 64 80] [--budget 90]

For each d (n = 10 d): the candidate count C, the time of each phase of ``dmosopt_b200.sampling.glp`` (host
enumeration, GPU screening of all C lattices, the exact pass over the shortlist, the ranked Gram-Schmidt decorrelation
of maxiter 5) and ``glp`` end to end, the pair-dims per second (C n^2 d over the screening time) and the screening
kernel's FP64 rate.  The reference (oracle/_ref, when built) is timed only where its estimated time, at the pair-dim
rate it reached on the smallest d, is within ``--budget`` seconds; the rest are printed as extrapolated.  Prints the
card name, power limit and clock first.

FP64 operations per pair-dim of the CD2 screening kernel (csrc/design.cu, l2_pairs_kernel): x_k - x_j (DADD), l_k + r_j
(DADD), (l_k + r_j) - 0.5 |x_k - x_j| (DFMA) and the running product (DMUL): 4 instructions, 5 flops (an FMA counts 2).
The kernel computes the upper triangle of 64 x 64 tiles only, so it performs C T (T + 1) / 2 64^2 d pair-dims, T =
ceil(n / 64).
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
from dmosopt_b200 import sampling  # noqa: E402

FLOPS_PER_PAIR_DIM = 5
H100_SXM_FP64_TFLOPS = 34.0  # data sheet, non-tensor FP64, at up to 700 W


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return f"device: {torch.cuda.get_device_properties(0).name}; nvidia-smi (name, power limit, sm clock, max sm clock): {q.stdout.strip() or q.stderr.strip()}"


def wall_s(fn, reps=3, warm=True):
    if warm:
        fn()
    best = math.inf
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        best = min(best, time.perf_counter() - t)
    return best


def kernel_ms(name, fn, reps=3):
    fn()
    best = math.inf
    for _ in range(reps):
        L.profile_enable(True)
        fn()
        L.synchronize()
        best = min(best, L.profile_report()[name][0])
        L.profile_enable(False)
    return best


def reference_glp():
    from oracle import reference_build

    ref = reference_build.reference_path()
    if ref is None:
        return None
    sys.path.insert(0, ref)
    try:
        from dmosopt import sampling as rs
    finally:
        sys.path.remove(ref)
    return rs.glp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", type=int, nargs="+", default=[15, 30, 40, 60, 64, 80])
    ap.add_argument("--budget", type=float, default=90.0, help="seconds the reference may take per d")
    a = ap.parse_args()
    L.context()
    print(card(), flush=True)
    ref = reference_glp()
    ref_rate = None  # pair-dims per second the reference reached
    for d in a.dims:
        n = 10 * d
        t_enum = wall_s(lambda: sampling.candidates(n, d), reps=1)
        N, rows, H = sampling.candidates(n, d)
        C = H.shape[0]
        if C == 0:
            print(f"d {d} n {n}: lattice {N}, no candidate (the design is the uniform draw)", flush=True)
            continue
        pd = C * rows * rows * d
        T = -(-rows // 64)
        pd_kernel = C * T * (T + 1) // 2 * 64 * 64 * d
        t_screen = wall_s(lambda: L.glp_cd2_terms(H, N, rows))
        k_ms = kernel_ms("l2_pairs_kernel", lambda: L.glp_cd2_terms(H, N, rows))
        best, short = sampling.select(H, N, rows)
        t_exact = wall_s(lambda: sampling._exact_cd2(H[short], N, rows, d))
        t_glp = wall_s(lambda: sampling.glp(n, d, np.random.default_rng(0)))
        X = sampling.glp(n, d, np.random.default_rng(0))

        def dec():
            x = X.copy()
            for _ in range(5):
                sampling.decorrelate(x, n, d)

        t_dec = wall_s(dec, reps=1)
        tflops = pd_kernel * FLOPS_PER_PAIR_DIM / (k_ms * 1e-3) / 1e12
        line = (f"d {d} n {n}: lattice {N} rows {rows} C {C} pair-dims {pd:.2e} | enumerate {t_enum * 1e3:.1f} ms, screen "
                f"{t_screen * 1e3:.2f} ms (kernel {k_ms:.2f} ms, {pd / t_screen:.2e} pair-dims/s, {tflops:.1f} TFLOP/s FP64 = "
                f"{100 * tflops / H100_SXM_FP64_TFLOPS:.0f} % of the data sheet's {H100_SXM_FP64_TFLOPS:.0f}), exact pass "
                f"{len(short)} lattices {t_exact * 1e3:.1f} ms, glp {t_glp * 1e3:.1f} ms | decorrelation maxiter 5 {t_dec * 1e3:.0f} ms")
        if ref is not None:
            est = pd / ref_rate if ref_rate else None
            if est is None and pd <= a.budget * 1e6 or est is not None and est <= a.budget:
                t0 = time.perf_counter()
                Xr = ref(n, d, np.random.default_rng(0))
                t_ref = time.perf_counter() - t0
                ref_rate = pd / t_ref
                same = np.array_equal(Xr, X)
                line += f" | reference glp {t_ref:.1f} s (measured, design {'identical' if same else 'DIFFERENT'})"
            else:
                rate = ref_rate or 1e6
                line += f" | reference glp ~{pd / rate:.0f} s (extrapolated at {rate:.2e} pair-dims/s, not run)"
        print(line, flush=True)


if __name__ == "__main__":
    main()
