"""Where the resident NSGA-II generation step (dmo_nsga2_step, bench.py's `value`) spends its time, phase by phase.

Builds bench.py's workload (bench.workload, same seed, same GP model, pop 65 536, d 30, M 3, N_train 4096 by default)
and measures the fused step --rounds times in the same process.  Each round runs --warmup generations, then --steps
timed generations with the profile timers off (the whole step, by device events around the window and by the host
clock; host waits and kernel launches per generation), then --steps generations with the library's per-scope
CUDA-event timers on, and prints per generation:
  * device-timer ms of each phase (step_tournament, step_generate, step_gp, step_truncate, step_hv) and of the kernels
    inside them that have scopes of their own (gp_kstar, gp_var, rank_peel, ...);
  * beside the contraction: the lane's time (step_truncate + step_hv) against the contraction's window (gp_var), both from
    the point the mean is written, and the slack between them (positive: the lane finished inside the window);
  * the card's name, its power limit and the median SM clock sampled during the timed window.
--free-sms F1,F2,... sweeps the SMs the overlapped contraction leaves to the lane (GP_LANE_SMS, gp.cuh): it builds one
library per value into a temporary directory (gp_tensor.cu, the one source that reads the constant, compiled with
-DDMO_GP_LANE_SMS=F and linked with the tree's other objects) and measures each in a process of its own, the values
alternating within every round.
Usage: python scripts/step_phases.py [--steps 100] [--warmup 20] [--rounds 1] [--free-sms 4,11,14,18] [--json OUT.json]
"""

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PHASES = ("step_tournament", "step_generate", "step_gp", "step_truncate", "step_hv")


def card(device):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", str(device)],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return q[0].strip(), float(q[1])
    except Exception:
        return None, None


def measure(L, bench, rs, steps, warmup):
    clocks = bench.ClockSampler(0)
    clocks.start()
    for _ in range(warmup):
        rs.step()
    L.synchronize()
    clocks.mark_begin()
    w0, l0 = L.wait_count(), L.launch_count()
    t0 = time.perf_counter()
    L.timer_begin()
    for _ in range(steps):
        rs.step()
    ms_dev = L.timer_end()
    t_host = time.perf_counter() - t0
    waits, launches = L.wait_count() - w0 - 1, L.launch_count() - l0  # - 1: timer_end's own wait
    clocks.mark_end()
    L.profile_enable(True)
    for _ in range(steps):
        rs.step()
    prof = L.profile_report()
    L.profile_enable(False)
    clk = clocks.stop()
    K = steps
    out = {
        "sm_mhz_median": clk.get("sm_mhz"), "clock_reasons": clk.get("reasons"),
        "step_ms_device": ms_dev / K, "step_ms_host": t_host * 1e3 / K,
        "waits_per_step": waits / K, "launches_per_step": launches / K,
        "phases_ms": {k: prof[k][0] / K for k in PHASES if k in prof},
        "scopes_ms": {k: v[0] / K for k, v in sorted(prof.items()) if k not in PHASES},
        "scope_counts_per_step": {k: v[1] / K for k, v in sorted(prof.items())},
    }
    ph = out["phases_ms"]
    out["outside_gp_ms"] = out["step_ms_device"] - ph.get("step_gp", 0.0)
    if "gp_var" in out["scopes_ms"] and "step_truncate" in ph:
        out["lane_ms"] = ph["step_truncate"] + ph.get("step_hv", 0.0)
        out["lane_slack_ms"] = out["scopes_ms"]["gp_var"] - out["lane_ms"]
    return out


def build_free_sms(values, out_dir):
    """One library per GP_LANE_SMS value: gp_tensor.cu compiled with -DDMO_GP_LANE_SMS=F, the tree's other objects."""
    from dmosopt_b200 import build as b

    b.build(verbose=False)
    others = [os.path.join(b.OBJ, s.replace(".cu", ".o")) for s in b.SOURCES if s != "gp_tensor.cu"]
    libs = {}
    for f in values:
        obj = os.path.join(out_dir, f"gp_tensor_{f}.o")
        lib = os.path.join(out_dir, f"libdmosopt_b200_free{f}.so")
        subprocess.run([b._nvcc()] + [x for x in b.NVCC_FLAGS if x not in ("-Xptxas", "-v")] + [f"-DDMO_GP_LANE_SMS={f}", "-c",
                       os.path.join(b.CSRC, "gp_tensor.cu"), "-o", obj], check=True)
        subprocess.run([b._nvcc(), "-shared", "-o", lib, obj] + others + ["-gencode", "arch=compute_90a,code=sm_90a"], check=True)
        libs[f] = lib
    return libs


def sweep(args):
    values = [int(v) for v in args.free_sms.split(",")]
    rows = []
    with tempfile.TemporaryDirectory(prefix="dmo_free_sms_") as tmp:
        libs = build_free_sms(values, tmp)
        for rnd in range(args.rounds):
            for f in values:
                js = os.path.join(tmp, f"r{rnd}_f{f}.json")
                cmd = [sys.executable, os.path.abspath(__file__), "--lib", libs[f], "--json", js] + [
                    f"--{k}={getattr(args, k)}" for k in ("steps", "warmup", "pop", "dim", "obj", "ntrain", "seed")]
                subprocess.run(cmd, check=True, stdout=sys.stderr)
                with open(js) as fh:
                    res = json.load(fh)
                r = res["rounds"][0]
                rows.append({**r, "free_sms": f, "round": rnd, "card": res["card"], "power_limit_w": res["power_limit_w"]})
    print(f"\n{rows[0]['card']}, power limit {rows[0]['power_limit_w']} W, pop {args.pop}, dim {args.dim}, {args.obj} objectives, "
          f"N_train {args.ntrain}, {args.steps} generations")
    print(f"{'free SMs':>9}{'round':>6}{'step ms':>10}{'gp_var':>9}{'truncate':>9}{'hv':>8}{'slack':>9}{'SM MHz':>9}")
    for r in rows:
        ph, sc = r["phases_ms"], r["scopes_ms"]
        slack = r.get("lane_slack_ms")
        print(f"{r['free_sms']:>9}{r['round']:>6}{r['step_ms_device']:>10.3f}{sc.get('gp_var', float('nan')):>9.3f}"
              f"{ph.get('step_truncate', float('nan')):>9.3f}{ph.get('step_hv', float('nan')):>8.3f}"
              f"{(f'{slack:+.3f}' if slack is not None else '-'):>9}{(r['sm_mhz_median'] or float('nan')):>9.0f}")
    summary = {"steps": args.steps, "pop": args.pop, "dim": args.dim, "obj": args.obj, "ntrain": args.ntrain, "sweep": rows}
    print(json.dumps(summary), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=1, help="times the step is measured, one after the other")
    ap.add_argument("--pop", type=int, default=65536)
    ap.add_argument("--dim", type=int, default=30)
    ap.add_argument("--obj", type=int, default=3)
    ap.add_argument("--ntrain", type=int, default=4096)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--json", default=None, help="also write the result to this file")
    ap.add_argument("--free-sms", default=None, help="comma-separated GP_LANE_SMS values to sweep, one library each")
    ap.add_argument("--lib", default=None, help=argparse.SUPPRESS)  # the library a --free-sms child measures
    args = ap.parse_args()
    if args.free_sms:
        return sweep(args)

    import bench
    import dmosopt_b200 as b2
    from dmosopt_b200 import _lib as L

    if args.lib:
        L.load_library(args.lib)
    L.context(0)
    pop, d, M, N = args.pop, args.dim, args.obj, args.ntrain
    w = bench.workload(pop, d, M, N)
    sm = b2.GPR_Matern(w["Xtr"], w["Ytr"], d, M, w["xlb"], w["xub"], optimizer=None, precision="auto")
    y0 = sm.evaluate(w["X0"]).astype(np.float32)
    ref = y0.max(axis=0).astype(np.float64) + 0.1 * (y0.max(axis=0) - y0.min(axis=0))
    opt = b2.NSGA2(popsize=pop, nInput=d, nOutput=M, model=b2.Model(objective=sm), distance_metric=None)
    opt.initialize_strategy(w["X0"], y0, np.column_stack((w["xlb"], w["xub"])), np.random.default_rng(args.seed))
    rs = bench.ResidentStep(L, sm._gp, pop, d, M, w["xlb"], w["xub"], opt.state.population_parm,
                            opt.state.population_obj.astype(np.float64), opt.state.rank.copy(), ref, args.seed)
    rs.precision, rs.metric = L.GP_AUTO, L.METRIC_NONE
    name, plimit = card(0)

    results = []
    for rnd in range(args.rounds):
        out = measure(L, bench, rs, args.steps, args.warmup)
        out.update(round=rnd)
        results.append(out)
        ph, sc = out["phases_ms"], out["scopes_ms"]
        print(f"--- round {rnd}: {name}, power limit {plimit} W, median SM clock {out['sm_mhz_median']} MHz, "
              f"{args.steps} generations")
        print(f"{'phase':<18}{'ms / generation':>16}")
        for k in PHASES:
            if k in ph:
                print(f"{k:<18}{ph[k]:>16.3f}")
        for k, v in sc.items():
            print(f"  {k:<16}{v:>16.3f}")
        print(f"{'step (events)':<18}{out['step_ms_device']:>16.3f}")
        print(f"{'step (host)':<18}{out['step_ms_host']:>16.3f}")
        print(f"{'outside step_gp':<18}{out['outside_gp_ms']:>16.3f}")
        if "lane_slack_ms" in out:
            print(f"lane {out['lane_ms']:.3f} ms (truncation {ph['step_truncate']:.3f}, hypervolume {ph.get('step_hv', 0.0):.3f}) "
                  f"against the contraction's window {sc['gp_var']:.3f} ms: slack {out['lane_slack_ms']:+.3f} ms")
        print(f"host waits / generation {out['waits_per_step']:.2f}, launches / generation {out['launches_per_step']:.1f}", flush=True)

    print(f"\n{name}, power limit {plimit} W, pop {pop}, dim {d}, {M} objectives, N_train {N}")
    print(f"{'round':>6}{'step ms':>10}{'gp_var':>9}{'truncate':>9}{'hv':>8}{'slack':>9}{'SM MHz':>9}")
    for r in results:
        ph, sc = r["phases_ms"], r["scopes_ms"]
        slack = r.get("lane_slack_ms")
        print(f"{r['round']:>6}{r['step_ms_device']:>10.3f}{sc.get('gp_var', float('nan')):>9.3f}"
              f"{ph.get('step_truncate', float('nan')):>9.3f}{ph.get('step_hv', float('nan')):>8.3f}"
              f"{(f'{slack:+.3f}' if slack is not None else '-'):>9}{(r['sm_mhz_median'] or float('nan')):>9.0f}")
    summary = {"card": name, "power_limit_w": plimit, "steps": args.steps, "pop": pop, "dim": d, "obj": M, "ntrain": N,
               "rounds": results}
    print(json.dumps(summary), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
