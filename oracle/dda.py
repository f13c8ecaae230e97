"""Oracle: non-dominated ranking (rows A1/A2 of SURVEY.md section 8a).

Test infrastructure only (see oracle/__init__.py).

Restates ``dmosopt/dda.py``:
  * ``dominance_degree_matrix``  -> dda.py:13-47   (D[i,j] = #objectives with y_i <= y_j)
  * ``dda_ens`` / ``dda_insert`` -> dda.py:97-152  (ENS-SS insertion in argsort(Y[:,0]) order)
  * ``dda_non_dominated_sort``   -> dda.py:50-94   (front peeling on D)

and adds ``rank_canonical`` -- the canonical Pareto front index (length of the
longest domination chain ending at a point).  The CUDA kernel implements the
canonical rank; it equals ``dda_ens`` whenever objective 0 is tie-free
(SURVEY.md section 8a row A2), which tests assert.
"""

import numpy as np


def dominance_degree_matrix(Y):
    """D[i, j] = number of objectives k with Y[i,k] <= Y[j,k]  (dda.py:13-47).

    The reference builds this from per-objective comparison matrices filled in
    sorted order; the closed form is the same integer matrix.
    """
    Y = np.asarray(Y)
    return (Y[:, None, :] <= Y[None, :, :]).sum(axis=2).astype(np.intp)


def _zero_identical(D, d):
    """dda.py:108-115: identical vectors are made mutually non-dominating."""
    same = (D == d) & (D.T == d)
    D = D.copy()
    D[same] = 0
    return D


def dda_ens(Y):
    """Faithful restatement of dda.py:97-152 (the rank every sortMO uses).

    Points are inserted in ``np.argsort(Y[:, 0])`` order into the first front
    none of whose *current* members dominates them.
    """
    Y = np.asarray(Y)
    n, d = Y.shape
    D = _zero_identical(dominance_degree_matrix(Y), d)
    fronts = []
    rank = np.zeros(n, dtype=np.intp)
    for s in np.argsort(Y[:, 0]):
        placed = False
        for k, front in enumerate(fronts):
            if not np.any(D[front, s] == d):
                front.append(s)
                rank[s] = k
                placed = True
                break
        if not placed:
            fronts.append([s])
            rank[s] = len(fronts) - 1
    return rank


def dominates_matrix(Y):
    """dom[i, j] = True iff i dominates j (all <=, not identical)."""
    Y = np.asarray(Y)
    le = (Y[:, None, :] <= Y[None, :, :]).all(axis=2)
    eq = (Y[:, None, :] == Y[None, :, :]).all(axis=2)
    return le & ~eq


def rank_canonical(Y, block=2048):
    """Canonical non-dominated rank by front peeling; O(F * n^2 / block) memory-light.

    Equals dda.py:50-94 (``dda_non_dominated_sort``) for every input and
    ``dda_ens`` whenever objective 0 has no ties.
    """
    Y = np.asarray(Y, dtype=np.float64)
    n = Y.shape[0]
    rank = np.full(n, -1, dtype=np.int64)
    alive = np.arange(n)
    k = 0
    while alive.size:
        Ya = Y[alive]
        dominated = np.zeros(alive.size, dtype=bool)
        for s in range(0, alive.size, block):
            Yb = Ya[s : s + block]
            le = (Ya[:, None, :] <= Yb[None, :, :]).all(axis=2)
            eq = (Ya[:, None, :] == Yb[None, :, :]).all(axis=2)
            dominated[s : s + block] = (le & ~eq).any(axis=0)
        rank[alive[~dominated]] = k
        alive = alive[dominated]
        k += 1
    return rank


def rank_chain_dp(Y):
    """Canonical rank as longest-chain DP over the lexicographic order.

    This is the formulation the CUDA kernel uses (rank_i = 1 + max rank of the
    dominators of i, processed in lexicographic order); kept here so the DP
    itself is pinned against peeling on the CPU.
    """
    Y = np.asarray(Y, dtype=np.float64)
    n, d = Y.shape
    order = np.lexsort(tuple(Y[:, k] for k in range(d - 1, -1, -1)))
    Ys = Y[order]
    r = np.zeros(n, dtype=np.int64)
    for i in range(1, n):
        le = (Ys[:i] <= Ys[i]).all(axis=1)
        eq = (Ys[:i] == Ys[i]).all(axis=1)
        dom = le & ~eq
        if dom.any():
            r[i] = r[:i][dom].max() + 1
    out = np.empty(n, dtype=np.int64)
    out[order] = r
    return out


# ------------------------------------------------------------------------------------------ brute-force checks (torch)
# j dominates i  <=>  Y[j] <= Y[i] in every objective and the rows are not identical (for float64 without NaN: some
# objective is strictly smaller; -0.0 == +0.0).  Every target row is tested against every row, in chunks of targets, on
# any torch device; nothing here uses the library.  NaN is outside the contract these checks state.


def _as_tensor(a, dtype, device):
    import torch

    if isinstance(a, torch.Tensor):
        return a.to(device=device, dtype=dtype)
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device=device)


def _dominator_chunks(Y, device, chunk):
    """Yields (s, e, dom) with dom[t, j] = row j dominates row s + t, for consecutive target chunks [s, e)."""
    import torch

    Yt = _as_tensor(Y, torch.float64, device)
    if Yt.ndim != 2:
        raise ValueError(f"Y must be (n, M), got shape {tuple(Yt.shape)}")
    n, M = Yt.shape
    if chunk is None:
        chunk = max(1, min(n, (1 << 25) // max(n, 1)))
    cols = [Yt[:, k].contiguous() for k in range(M)]
    for s in range(0, n, chunk):
        e = min(n, s + chunk)
        le = torch.ones((e - s, n), dtype=torch.bool, device=Yt.device)
        lt = torch.zeros((e - s, n), dtype=torch.bool, device=Yt.device)
        for k in range(M):
            src = cols[k][None, :]
            tgt = cols[k][s:e, None]
            le &= src <= tgt
            lt |= src < tgt
        yield s, e, le & lt


def _fail(what, bad, lines):
    shown = "\n  ".join(lines)
    raise AssertionError(f"{what}: {bad} row(s) wrong; first offenders:\n  {shown}")


def check_ranks(Y, r, device="cpu", chunk=None, show=8):
    """Asserts the chain identity on every row: r[i] == 0 if nothing dominates i, else 1 + max r[j] over the j dominating i.

    By induction over the dominance order this identity holds for exactly one rank vector, the canonical rank
    (``rank_canonical``), so checking it everywhere is an exact comparison -- at O(n^2 M) compares, without peeling.
    Memory: chunk x n booleans (default chunk: 2^25 / n targets).  Raises AssertionError naming the first wrong rows,
    the expected rank and a dominator that sets it."""
    import torch

    n = len(r)
    rt = _as_tensor(np.asarray(r, dtype=np.int64) if not isinstance(r, torch.Tensor) else r, torch.int64, device)
    if rt.shape != (n,):
        raise ValueError("r must be one rank per row")
    if n and (int(rt.min()) < 0 or int(rt.max()) >= (1 << 31) - 1):
        raise AssertionError(f"check_ranks: ranks out of range [{int(rt.min())}, {int(rt.max())}]")
    r32 = rt.to(torch.int32)
    bad_total, lines = 0, []
    for s, e, dom in _dominator_chunks(Y, device, chunk):
        if dom.shape[1] != n:
            raise ValueError(f"{dom.shape[1]} rows but {n} ranks")
        vals = torch.where(dom, r32[None, :], torch.full((), -1, dtype=torch.int32, device=rt.device))
        mx, arg = vals.max(dim=1)
        expect = mx.to(torch.int64) + 1  # no dominator: -1 + 1 = 0
        wrong = torch.nonzero(expect != rt[s:e]).flatten()
        bad_total += int(wrong.numel())
        for t in wrong[: max(0, show - len(lines))].tolist():
            i = s + t
            who = f"dominator {int(arg[t])} with rank {int(rt[int(arg[t])])}" if int(mx[t]) >= 0 else "no dominator"
            lines.append(f"row {i}: rank {int(rt[i])}, expected {int(expect[t])} ({who})")
        del vals, dom
    if bad_total:
        _fail("check_ranks", bad_total, lines)


def check_flags(Y, f, device="cpu", chunk=None, show=8):
    """Asserts f[i] == (some row dominates i) on every row (f: 0 = rank 0, nonzero = dominated)."""
    import torch

    n = len(f)
    ft = _as_tensor(np.asarray(f) if not isinstance(f, torch.Tensor) else f, torch.int64, device) != 0
    bad_total, lines = 0, []
    for s, e, dom in _dominator_chunks(Y, device, chunk):
        if dom.shape[1] != n:
            raise ValueError(f"{dom.shape[1]} rows but {n} flags")
        has, arg = dom.to(torch.uint8).max(dim=1)
        has = has != 0
        wrong = torch.nonzero(has != ft[s:e]).flatten()
        bad_total += int(wrong.numel())
        for t in wrong[: max(0, show - len(lines))].tolist():
            i = s + t
            who = f"dominated by row {int(arg[t])}" if bool(has[t]) else "nothing dominates it"
            lines.append(f"row {i}: flag {int(ft[i])}, expected {int(has[t])} ({who})")
        del dom
    if bad_total:
        _fail("check_flags", bad_total, lines)
