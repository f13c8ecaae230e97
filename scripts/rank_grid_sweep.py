"""GPU timings of the two users of the cell grid in csrc/rank.cu, on device buffers, with the library's stream events.

  * dmo_nondominated_flags (the rank-0 filter in front of the hypervolume) at M = 2 and 3, n = 8192, 65 536, 131 072 and
    2^18 + 5, on a uniform cloud (few rank-0 rows) and a sphere shell (nearly one front);
  * dmo_remove_worst at the bench's size (131 072 merged rows, keep 65 536, M = 3, d = 30) on sets whose kept rows span few
    fronts, so that the truncation peels them: the bench's sphere set and a set of six thick shells.

Each case is warmed up, then timed `--reps` times (one call between two events each); the median and the minimum are
printed with a CRC of the call's output, so that two builds can be compared for equal results as well as for time.
One JSON line per case.

  python scripts/rank_grid_sweep.py [--reps 20]
"""

import argparse
import json
import os
import sys
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from dmosopt_b200 import _lib as L  # noqa: E402


def uniform(n, M, seed):
    return np.random.default_rng(seed).random((n, M))


def sphere(n, M, seed):
    rng = np.random.default_rng(seed)
    v = np.abs(rng.standard_normal((n, M)))
    return v / np.linalg.norm(v, axis=1, keepdims=True) * (1.0 + 0.01 * rng.random((n, 1)))


def shells(n, M, seed):
    rng = np.random.default_rng(seed)
    v = np.abs(rng.standard_normal((n, M))) + 1e-12
    return v / np.linalg.norm(v, axis=1, keepdims=True) * (1.0 + 0.05 * rng.integers(0, 6, size=(n, 1)) + 1e-4 * rng.random((n, 1)))


def timed(call, reps, warmup=3):
    for _ in range(warmup):
        call()
    L.synchronize()
    ts = []
    for _ in range(reps):
        L.timer_begin()
        call()
        ts.append(L.timer_end())
    return float(np.median(ts)), float(np.min(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    lib, ctx = L.load_library(), L.context()

    for M in (2, 3):
        for n in (8192, 65536, 131072, (1 << 18) + 5):
            for kind, make in (("uniform", uniform), ("sphere", sphere)):
                Y = make(n, M, 17 * n + M)
                dY = L.DeviceArray((n, M)).upload(Y)
                df = L.DeviceArray((n,), np.int32)

                def call():
                    L._check(lib.dmo_nondominated_flags(ctx, dY.ptr, n, M, df.ptr), "dmo_nondominated_flags")

                med, best = timed(call, args.reps)
                f = df.download()
                print(json.dumps({"case": "nondominated_flags", "M": M, "n": n, "data": kind, "median_ms": round(med, 4),
                                  "min_ms": round(best, 4), "rank0_rows": int((f == 0).sum()), "crc": zlib.crc32(f.tobytes())}), flush=True)
                dY.free()
                df.free()

    n, keep, M, d = 131072, 65536, 3, 30
    X = np.random.default_rng(5).random((n, d))
    dX = L.DeviceArray((n, d)).upload(X)
    Xo, Yo = L.DeviceArray((keep, d)), L.DeviceArray((keep, M))
    rk, perm = L.DeviceArray((keep,), np.int32), L.DeviceArray((keep,), np.int64)
    for kind, Y in (("bench sphere", bench.objective_sets(n, M)["sphere"]), ("shells", shells(n, M, 9))):
        dY = L.DeviceArray((n, M)).upload(Y)

        def call():
            L._check(lib.dmo_remove_worst(ctx, dX.ptr, dY.ptr, n, d, M, L.METRIC_NONE, None, 0, keep, Xo.ptr, Yo.ptr, rk.ptr, perm.ptr),
                     "dmo_remove_worst")

        med, best = timed(call, args.reps)
        L.profile_enable(True)
        call()
        rep = L.profile_report()
        L.profile_enable(False)
        r, p = rk.download(), perm.download()
        print(json.dumps({"case": "remove_worst", "M": M, "n": n, "keep": keep, "data": kind, "median_ms": round(med, 4),
                          "min_ms": round(best, 4), "peeled": "rank_peel" in rep and "rank_chain" not in rep, "fronts_kept": int(r.max()) + 1,
                          "crc": zlib.crc32(r.tobytes() + p.tobytes())}), flush=True)
        dY.free()


if __name__ == "__main__":
    main()
