"""Rank kernel timing on the merged objective set of a real bench generation (GP-predicted children + float32 parents)."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
import dmosopt_b200 as b2
from dmosopt_b200 import _lib as L

L.context()
pop, d, M, N = 65536, 30, 3, 4096
w = bench.workload(pop, d, M, N)
sm = b2.GPR_Matern(w["Xtr"], w["Ytr"], d, M, w["xlb"], w["xub"], optimizer=None, precision="tensor")
mdl = b2.Model(objective=sm)
y0 = sm.evaluate(w["X0"]).astype(np.float32)
opt = b2.NSGA2(popsize=pop, nInput=d, nOutput=M, model=mdl, distance_metric=None)
opt.initialize_strategy(w["X0"], y0, np.column_stack((w["xlb"], w["xub"])), np.random.default_rng(0))
for g in range(int(sys.argv[1]) if len(sys.argv) > 1 else 4):
    x_gen, st = opt.generate()
    y_gen = sm.evaluate(x_gen)
    Y = np.vstack((y_gen, opt.state.population_obj.astype(np.float64)))
    dY = L.DeviceArray(Y.shape).upload(Y)
    r = L.DeviceArray((Y.shape[0],), np.int32)
    lib, ctx = L.load_library(), L.context()
    for env in ("", "1"):
        if env:
            os.environ["DMO_RANK_NOSEG"] = "1"
        else:
            os.environ.pop("DMO_RANK_NOSEG", None)
        L.profile_enable(True)
        for _ in range(3):
            L._check(lib.dmo_rank_nd(ctx, dY.ptr, Y.shape[0], M, r.ptr), "rank")
        rep = L.profile_report()
        L.profile_enable(False)
        rk = r.download()
        print(f"gen {g} {'lex' if env else 'seg'}: chain {rep['rank_chain'][0] / rep['rank_chain'][1]:.3f} ms, fronts {rk.max() + 1}, front0 {int((rk == 0).sum())}, "
              f"distinct ids per objective {[len(np.unique(Y[:, j])) for j in range(M)]}", flush=True)
    os.environ.pop("DMO_RANK_NOSEG", None)
    opt.update(x_gen, y_gen, st)

