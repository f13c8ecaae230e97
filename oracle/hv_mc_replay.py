"""Oracle: csrc/hv_mc.cu replayed draw for draw from its Philox stream.

Test infrastructure only (see oracle/__init__.py).

``oracle/hv_mc.py`` states the estimators' random variables with NumPy's generator; this module states what
``dmo_hypervolume_mc`` computes with its own generator, so that ``(value, samples, tests, algorithm)`` can be compared
for exact equality.  Every draw is ``Philox(seed)(ctr_lo, ctr_hi)`` with
  ctr_hi = draw << 32 | (stream_id & 0xFFFFFF) << 8 | purpose,  ctr_lo = the sample (or probe) index,
and the host arithmetic (W, the sampling CDF, U, M1, R, theta, the level-3 targets) is plain float64 in the code's
association order, so the result is reproduced bit for bit.

The replay applies each stopping rule one sample at a time in sample order, without the kernels' waves: it is the
statement the wave logic has to equal.  It evaluates samples in blocks, and FPRAS advances the trials of all live samples
of a block in lock step, but nothing it returns depends on the block sizes.  Each call returns ``(value, info)`` like
``_lib.hypervolume_mc`` plus a ``record`` of what happened (chosen boxes, per-sample xi, first dominators, eta, rounds,
discarded samples, the route), so tests can assert which edges a case reaches.
"""

import math

import numpy as np

from .hv_mc import filtered_front
from .philox import philox4x32_10, u01_53

P_FPRAS_SAMPLE, P_FPRAS_TRIAL, P_PROBE_SAMPLE, P_PROBE_TRIAL, P_MCM_SAMPLE, P_MCM_ETA, P_MC_SAMPLE = 1, 2, 3, 4, 5, 6, 7
N_PROBES = 50
MC_ROUNDS = 1000
RAN = {1: "FPRAS", 2: "MCM2RV", 3: "MonteCarlo", 4: "Hybrid-FPRAS", 5: "Hybrid-MCM2RV"}
_ELEMS = 1 << 22  # elements per vectorised dominance block


def ctr_hi(stream_id, purpose, draw):
    """``draw << 32 | (stream_id & 0xFFFFFF) << 8 | purpose`` (draw may be an array)."""
    return (np.asarray(draw, dtype=np.uint64) << np.uint64(32)) | np.uint64(((int(stream_id) & 0xFFFFFF) << 8) | int(purpose))


def philox(seed, s, stream_id, purpose, draw):
    return philox4x32_10(seed, np.asarray(s, dtype=np.uint64), ctr_hi(stream_id, purpose, draw))


def sample_uniforms(seed, s, stream_id, purpose, M):
    """u[:, 0 .. M] of samples s: call c gives u[2c] = u01_53(r.x, r.y) and, if 2c + 1 <= M, u[2c + 1] = u01_53(r.z, r.w)."""
    s = np.asarray(s, dtype=np.uint64)
    u = np.empty((s.size, M + 1))
    for c in range(M // 2 + 1):
        r = philox(seed, s, stream_id, purpose, c)
        u[:, 2 * c] = u01_53(r[0], r[1])
        if 2 * c + 1 <= M:
            u[:, 2 * c + 1] = u01_53(r[2], r[3])
    return u


def uniform_in(lo, hi, u):
    """lo + (hi - lo) * u, each operation rounded."""
    return lo + (hi - lo) * u


def randint(word, n):
    """(word * n) >> 32: the row a 32-bit word picks among n."""
    return ((np.asarray(word, dtype=np.uint64) * np.uint64(n)) >> np.uint64(32)).astype(np.int64)


def choose_box(cdf, u):
    """First i with cdf[i] > u, clamped to n - 1 (cdf is non-decreasing)."""
    return np.minimum(np.searchsorted(cdf, u, side="right"), len(cdf) - 1).astype(np.int64)


class Front:
    """The filtered front and the host quantities hv_mc.cu forms from it, in row order."""

    def __init__(self, F, ref):
        self.ref = np.asarray(ref, dtype=np.float64)
        self.F = filtered_front(F, self.ref)
        self.n, self.M = self.F.shape if len(self.F) else (0, self.ref.size)
        if self.n == 0:
            return
        D = self.ref - self.F
        v = np.ones(self.n)
        for j in range(self.M):
            v = v * D[:, j]
        self.v = v
        cum = np.add.accumulate(v)  # sequential, as the host loop
        self.W = float(cum[-1])
        self.cdf = cum / self.W
        self.ideal = self.F.min(axis=0)
        U = 1.0
        for j in range(self.M):
            U *= float(self.ref[j] - self.ideal[j])
        self.U = U


def budget_m1(eps, delta, nf):
    return 8.0 * (1.0 + eps) * float(nf) * math.log(2.0 / delta) / (eps * eps)


def mcm2rv_rv(eps, delta):
    """The real-valued R of run_mcm2rv and the hybrid's level 3, before the floor."""
    return (4.0 * (1.0 + eps * (1.0 - eps)) * math.log(2.0 / delta)) / (eps * eps * (1.0 - eps) * (1.0 - eps))


def theta(nf, U, W, V, Rv, M1):
    return ((float(nf) * float(nf) * (V * V + (U - V) * W) / (W * W)) * (Rv / M1))


def level3_targets(M1):
    cum, out = 0.0, []
    for f in (0.01, 0.02, 0.04, 0.08):
        cum += f
        out.append((cum, int(cum * M1)))
    return out


# ------------------------------------------------------------------------------------------------ FPRAS
def fpras_points(fr, seed, stream_id, purpose, s):
    """(boxes, x) of samples s: box by u[0] through the CDF, x uniform in [f_box, ref] by u[1 ..]."""
    u = sample_uniforms(seed, s, stream_id, purpose, fr.M)
    i = choose_box(fr.cdf, u[:, 0])
    return i, uniform_in(fr.F[i], fr.ref, u[:, 1:])


def fpras_xi(fr, seed, stream_id, s, cap):
    """(boxes, xi) of samples s: xi = index (from 1) of the first trial row k with x > f_k, 0 if none within cap trials.
    Trial t draws its row from word t & 3 of draw t >> 2.  All live samples advance together."""
    s = np.asarray(s, dtype=np.uint64)
    boxes, x = fpras_points(fr, seed, stream_id, P_FPRAS_SAMPLE, s)
    xi = np.zeros(s.size, dtype=np.int64)
    live = np.arange(s.size)
    ndraw = (cap + 3) // 4
    d0 = 0
    while live.size and d0 < ndraw:
        K = int(max(1, min(ndraw - d0, _ELEMS // (4 * fr.M * live.size))))
        d = np.arange(d0, d0 + K, dtype=np.uint64)
        r = philox4x32_10(seed, s[live][:, None], ctr_hi(stream_id, P_FPRAS_TRIAL, d)[None, :])
        k = np.stack([randint(w, fr.n) for w in r], axis=2).reshape(live.size, 4 * K)  # trial 4d + c
        dom = np.all(x[live][:, None, :] > fr.F[k], axis=2)
        t = np.arange(4 * d0, 4 * (d0 + K)) + 1
        dom &= t[None, :] <= cap
        hit = dom.any(axis=1)
        xi[live[hit]] = t[np.argmax(dom[hit], axis=1)]
        live = live[~hit]
        d0 += K
    return boxes, xi


class Fpras:
    """The FPRAS sample sequence: run(target) continues it until `target` tests are spent.  A sample whose xi exceeds the
    remaining budget is discarded, its tests are spent, and the next run resumes at the sample after it."""

    def __init__(self, fr, seed, stream_id):
        self.fr, self.seed, self.stream_id = fr, seed, stream_id
        self.tests = self.N = self.sum_xi = self.next = 0
        self.xi, self.boxes = [], []  # per consumed sample, in sample order (xi 0: not found within the run's budget)
        self.discards = []  # (sample index, remaining budget, run budget R0, xi or 0 if above R0)
        self.exact_hits = []  # samples whose xi met a run's target exactly (the next run resumes after them)
        self.runs = []  # (first sample, tests, N, sum of xi, target) at the start of each run

    def run(self, target):
        self.runs.append((self.next, self.tests, self.N, self.sum_xi, target))
        R0 = target - self.tests
        while self.tests < target:
            rem = target - self.tests
            mean = self.sum_xi / self.N if self.N else float(self.fr.n)
            B = int(min(1 << 16, max(64, 1.1 * rem / max(mean, 1.0) + 64)))
            s = np.arange(self.next, self.next + B, dtype=np.uint64)
            boxes, xi = fpras_xi(self.fr, self.seed, self.stream_id, s, R0)
            cum = np.cumsum(xi)
            bad = (xi == 0) | (cum > rem)
            stop = bad | (cum == rem)
            if not stop.any():
                self.xi.append(xi)
                self.boxes.append(boxes)
                self.N += B
                self.sum_xi += int(cum[-1])
                self.tests += int(cum[-1])
                self.next += B
                continue
            k = int(np.argmax(stop))
            self.xi.append(xi[: k + 1])
            self.boxes.append(boxes[: k + 1])
            if bad[k]:  # sample k straddles the target: discarded, its tests spent
                used = int(cum[k - 1]) if k else 0
                self.discards.append((self.next + k, rem - used, R0, int(xi[k])))
                self.N += k
            else:  # sample k meets the target exactly
                used = rem
                self.exact_hits.append(self.next + k)
                self.N += k + 1
            self.sum_xi += used
            self.tests = target
            self.next += k + 1

    def estimate(self):
        N = self.N if self.N > 0 else 1
        return (self.fr.W / float(self.fr.n)) * (float(self.sum_xi) / float(N)), N


# ------------------------------------------------------------------------------------------------ dominance scans
def scan(fr, lo, hi, seed, stream_id, purpose, s, want_eta):
    """x uniform in [lo, hi] by u[1 ..]; first[i] = index of the first row f_k <= x (-1: none); tests = rows scanned
    up to and including it (n if none), plus one for eta; eta[i] = [f_k <= x] for the row of r.x of draw 0 (purpose 6)."""
    s = np.asarray(s, dtype=np.uint64)
    x = uniform_in(lo, hi, sample_uniforms(seed, s, stream_id, purpose, fr.M)[:, 1:])
    first = np.empty(s.size, dtype=np.int64)
    C = max(1, _ELEMS // (fr.n * fr.M))
    for a in range(0, s.size, C):
        le = np.all(fr.F[None, :, :] <= x[a:a + C, None, :], axis=2)
        any_ = le.any(axis=1)
        first[a:a + C] = np.where(any_, np.argmax(le, axis=1), -1)
    dom = first >= 0
    tests = np.where(dom, first + 1, fr.n)
    eta = np.zeros(s.size, dtype=bool)
    if want_eta and dom.any():
        r = philox(seed, s[dom], stream_id, P_MCM_ETA, 0)
        k = randint(r[0], fr.n)
        eta[dom] = np.all(fr.F[k] <= x[dom], axis=1)
        tests = tests + dom
    return first, tests, eta


def run_mcm2rv(fr, eps, delta, seed, stream_id, rec):
    """Samples in order until the number of eta successes reaches R; the stopping sample's tests count."""
    R = int(math.floor(mcm2rv_rv(eps, delta)))
    N = Ssum = tests = nxt = 0
    firsts, etas = [], []
    while Ssum < R:
        B = 1 << 15
        s = np.arange(nxt, nxt + B, dtype=np.uint64)
        first, t, eta = scan(fr, fr.ideal, fr.ref, seed, stream_id, P_MCM_SAMPLE, s, True)
        c = np.cumsum(eta)
        if Ssum + int(c[-1]) < R:
            k = B
        else:
            k = int(np.argmax(Ssum + c >= R)) + 1
        firsts.append(first[:k])
        etas.append(eta[:k])
        N += int(np.count_nonzero(first[:k] >= 0))
        Ssum += int(c[k - 1])
        tests += int(t[:k].sum())
        nxt += k
    rec.update(R=R, mcm_attempts=nxt, mcm_first=np.concatenate(firsts), mcm_eta=np.concatenate(etas))
    return N, Ssum, tests


def probes(fr, seed, stream_id):
    """xi of the hybrid's 50 level-2 probes: c = rows strictly below x; xi = 1 + the first t with
    u01_53(r.x, r.y) * (n - t) < c, or n when c = 0."""
    p = np.arange(N_PROBES, dtype=np.uint64)
    boxes, x = fpras_points(fr, seed, stream_id, P_PROBE_SAMPLE, p)
    c = np.all(x[:, None, :] > fr.F[None, :, :], axis=2).sum(axis=1)
    xi = np.full(N_PROBES, fr.n, dtype=np.int64)
    t = np.arange(fr.n, dtype=np.uint64)
    for q in range(N_PROBES):
        if c[q] == 0:
            continue
        r = philox(seed, np.uint64(q), stream_id, P_PROBE_TRIAL, t)
        hit = u01_53(r[0], r[1]) * (fr.n - t.astype(np.int64)).astype(np.float64) < float(c[q])
        xi[q] = int(np.argmax(hit)) + 1
    return boxes, c, xi


# ------------------------------------------------------------------------------------------------ entry
def hypervolume_mc(F, ref, algorithm="hybrid", epsilon=0.01, delta=0.25, n_samples=100000, seed=0, stream=0):
    """(value, info) with info = {samples, tests, algorithm, record}, as dmo_hypervolume_mc computes them."""
    fr = Front(F, ref)
    rec = {"front": fr}
    info = {"samples": 0, "tests": 0, "algorithm": None, "record": rec}
    if fr.n == 0:
        return 0.0, info
    eps, delta, nf, W, U = float(epsilon), float(delta), fr.n, fr.W, fr.U
    M1 = budget_m1(eps, delta, nf) if algorithm != "monte_carlo" else None
    rec["M1"] = M1
    ran = {"hybrid": 0, "fpras": 1, "mcm2rv": 2, "monte_carlo": 3}[algorithm]

    def fpras_to(st, target):
        st.run(target)
        rec["fpras"] = st
        v, N = st.estimate()
        return v, N, st.tests

    def mcm2rv(extra):
        N, S, t = run_mcm2rv(fr, eps, delta, seed, stream, rec)
        return (W / float(nf)) * (float(N) / float(S)), N, t + extra

    if ran == 3:
        dom = tests = samples = nxt = rounds = 0
        while rounds < MC_ROUNDS and dom == 0:
            s = np.arange(nxt, nxt + n_samples, dtype=np.uint64)
            first, t, _ = scan(fr, fr.ideal, fr.ref, seed, stream, P_MC_SAMPLE, s, False)
            dom = int(np.count_nonzero(first >= 0))
            tests += int(t.sum())
            samples += n_samples
            nxt += n_samples
            rounds += 1
        rec.update(rounds=rounds, mc_first=first)
        value = U * (float(dom) / float(n_samples))
    elif ran == 1:
        value, samples, tests = fpras_to(Fpras(fr, seed, stream), int(M1))
    elif ran == 2:
        value, samples, tests = mcm2rv(0)
    else:
        ratio = W / U
        rec["ratio"] = ratio
        if ratio > 5.0:
            ran = 2
            value, samples, tests = mcm2rv(0)
        elif ratio < 1.2:
            ran = 1
            value, samples, tests = fpras_to(Fpras(fr, seed, stream), int(M1))
        else:
            boxes, c, pxi = probes(fr, seed, stream)
            mean_xi = 0.0
            for q in range(N_PROBES):
                mean_xi += float(pxi[q])
            mean_xi /= N_PROBES
            rec.update(probe_boxes=boxes, probe_count=c, probe_xi=pxi, mean_xi=mean_xi)
            if mean_xi > 20.0:
                ran = 2
                value, samples, tests = mcm2rv(0)
            elif mean_xi < 5.0:
                ran = 1
                value, samples, tests = fpras_to(Fpras(fr, seed, stream), int(M1))
            else:
                Rv = mcm2rv_rv(eps, delta)
                st = Fpras(fr, seed, stream)
                rec["level3"] = rounds = []
                decided = False
                for cum, target in level3_targets(M1):
                    st.run(target)
                    V, _ = st.estimate()
                    e1 = eps / math.sqrt(cum)
                    with np.errstate(divide="ignore", invalid="ignore"):  # e1 = 1: V / 0 is inf and theta NaN, as in C
                        th_upper = float(theta(nf, U, W, np.float64(V) / np.float64(1.0 - e1), Rv, M1))
                        th_lower = float(theta(nf, U, W, np.float64(V) / np.float64(1.0 + e1), Rv, M1))
                    threshold = 1.0 - cum
                    rounds.append((target, th_upper, th_lower, threshold))
                    if th_upper < threshold * 0.85:
                        ran = 5
                        value, samples, tests = mcm2rv(st.tests)
                        rec["fpras"] = st
                        decided = True
                        break
                    if th_lower > threshold * 1.15:
                        decided = True
                        break
                if ran != 5:
                    ran = 4
                    value, samples, tests = fpras_to(st, int(M1))
                rec["decided"] = decided
    rec["route"] = RAN[ran]
    info.update(samples=int(samples), tests=int(tests), algorithm=RAN[ran])
    return float(value), info
