"""Epsilon-nondominated archive (Woodruff & Herman's epsilon-box sort, dmosopt/MOEA.py:470-595), restated twice.

``sequential`` inserts the rows one at a time, as the archive's ``sortinto`` does:
  * a row's box is floor(y / eps) per objective, after nan_to_num; an eps of 0 or NaN counts as 1e-8;
  * a row whose box is dominated by an archived box is rejected;
  * archived rows whose boxes the row's box dominates leave;
  * in the same box the newcomer replaces the archived row unless the archived row is strictly closer to the box's
    corner (box * eps) in squared distance; otherwise the newcomer is rejected;
  * a row that survives is appended.

``batch`` computes the same archive in one pass: group the rows by box, take in each box the row of least distance
(the last one on a tie; every distance is NaN when an eps is infinite, and then the last row), keep the boxes no other
occupied box dominates and list their rows in ascending order.

Both square with ``d * d`` (correctly rounded, like the GPU); the reference squares with libm ``pow``, which is not
always correctly rounded, so the two can disagree only when two rows of one box have distances a few ulp apart.
"""

import math

import numpy as np


def clean_eps(eps):
    """The archive's epsilons: 0 and NaN become 1e-8."""
    return np.array([1e-8 if (e == 0 or np.isnan(e)) else float(e) for e in np.ravel(eps)], dtype=np.float64)


def boxes_and_dist(Y, eps):
    """(nan_to_num'ed rows, float64 boxes, squared corner distances) of the first len(eps) columns of Y.
    Raises OverflowError where some y / eps is infinite (the reference's math.floor)."""
    e = clean_eps(eps)
    Y = np.nan_to_num(np.asarray(Y, dtype=np.float64))
    if Y.ndim == 1:
        Y = Y[None, :]
    y = Y[:, : e.shape[0]]
    with np.errstate(over="ignore", invalid="ignore"):
        q = y / e
        if np.isinf(q).any():
            raise OverflowError("cannot convert float infinity to integer")
        box = np.floor(q) + 0.0  # -0.0 -> +0.0: the same box as +0.0
        d = y - box * e
        sq = d * d
    dist = sq[:, 0].copy() if y.shape[0] else np.zeros(0)
    for j in range(1, y.shape[1]):
        dist = dist + sq[:, j]
    return Y, box, dist


def sequential(Y, eps):
    """Kept row indices, inserting row 0, 1, ... in order (the archive's order: ascending)."""
    _, box, dist = boxes_and_dist(Y, eps)
    B = [[math.floor(v) for v in row] for row in box]  # Python ints, compared exactly
    arch = []  # row indices, in archive order
    for i in range(len(B)):
        b = B[i]
        rejected = False
        survivors = []
        for a in arch:
            ab = B[a]
            le = all(x <= y for x, y in zip(ab, b))
            ge = all(x >= y for x, y in zip(ab, b))
            if le and not ge:  # archived box dominates
                rejected = True
            elif ge and not le:  # the new box dominates the archived one
                continue
            elif le and ge and dist[a] < dist[i]:  # same box, archived row strictly closer
                rejected = True
            elif le and ge:
                continue  # same box: the newcomer replaces it
            if rejected:
                break
            survivors.append(a)
        if not rejected:
            arch = survivors + [i]
    return np.array(arch, dtype=np.int64)


def groups_and_winners(Y, eps):
    """(distinct boxes (k, M), winner row of each) of the rows of Y, the boxes in lexicographic order."""
    _, box, dist = boxes_and_dist(Y, eps)
    n = box.shape[0]
    if n == 0:
        return box, np.zeros(0, dtype=np.int64)
    key = np.zeros(n) if np.isinf(clean_eps(eps)).any() else dist
    uniq, inv = np.unique(box, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    order = np.lexsort((-np.arange(n), key, inv))  # by box, then least distance, then last row
    first = np.ones(n, dtype=bool)
    first[1:] = inv[order[1:]] != inv[order[:-1]]
    return uniq, order[first].astype(np.int64)


def dominated(B, chunk=2048):
    """dominated[i] = some row of B dominates row i (<= everywhere, < somewhere)."""
    B = np.asarray(B, dtype=np.float64)
    out = np.zeros(B.shape[0], dtype=bool)
    for s in range(0, B.shape[0], chunk):
        t = B[s : s + chunk, None, :]
        out[s : s + chunk] = (np.all(B[None] <= t, axis=2) & np.any(B[None] < t, axis=2)).any(axis=1)
    return out


def batch(Y, eps):
    """Kept row indices, ascending: the winners of the boxes no other occupied box dominates."""
    uniq, win = groups_and_winners(Y, eps)
    return np.sort(win[~dominated(uniq)])
