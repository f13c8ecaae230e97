"""The brute-force dominance checks of oracle/dda.py (check_ranks, check_flags) on the CPU: they accept the canonical
ranks and rank-0 flags of random, tied and duplicated sets, and reject every single-entry corruption (a rank moved by
+-1, a flag flipped).  The GPU rank tests rely on these checks being exact in both directions."""

import numpy as np
import pytest

from oracle import dda


def _sets():
    rng = np.random.default_rng(7)
    out = {
        "uniform3": rng.random((300, 3)),
        "uniform2": rng.random((257, 2)),
        "uniform6": rng.random((200, 6)),
        "one_objective": rng.integers(0, 20, size=(150, 1)).astype(np.float64),
        "ties": rng.integers(0, 4, size=(240, 3)).astype(np.float64),
        "signed_zero": np.where(rng.random((120, 2)) < 0.5, -0.0, 0.0) + rng.integers(0, 2, size=(120, 2)),
        "chain": np.column_stack((np.arange(60.0), np.arange(60.0) * 2.0))[rng.permutation(60)],
        "single": np.array([[1.0, 2.0, 3.0]]),
    }
    base = rng.random((90, 4))
    out["duplicates"] = np.vstack((base, base[rng.integers(0, 90, size=70)]))[rng.permutation(160)]
    x = rng.random((200, 3))
    out["extremes"] = np.where(rng.random((200, 3)) < 0.2, np.inf, x)
    out["extremes"][rng.random((200, 3)) < 0.1] = -np.inf
    out["extremes"][:10, 0] = 5e-324
    out["extremes"][10:20, 1] = 1e300
    return out


SETS = _sets()


@pytest.mark.parametrize("name", sorted(SETS))
def test_checks_accept_the_canonical_rank(name):
    Y = SETS[name]
    r = dda.rank_canonical(Y)
    assert np.array_equal(r, dda.rank_chain_dp(Y))
    dda.check_ranks(Y, r)
    dda.check_ranks(Y, r, chunk=7)  # chunk boundaries do not matter
    dda.check_flags(Y, (r > 0).astype(np.int32))
    dda.check_flags(Y, (r > 0).astype(np.int32), chunk=13)


@pytest.mark.parametrize("name", sorted(SETS))
def test_check_ranks_rejects_every_single_entry_off_by_one(name):
    Y = SETS[name]
    r = dda.rank_canonical(Y)
    rows = range(len(r)) if len(r) <= 60 else np.random.default_rng(len(r)).choice(len(r), size=60, replace=False)
    for i in rows:
        for d in (-1, 1):
            bad = r.copy()
            bad[i] += d
            with pytest.raises(AssertionError, match="check_ranks"):
                dda.check_ranks(Y, bad, chunk=64)


@pytest.mark.parametrize("name", sorted(SETS))
def test_check_flags_rejects_every_single_flip(name):
    Y = SETS[name]
    f = (dda.rank_canonical(Y) > 0).astype(np.int32)
    rows = range(len(f)) if len(f) <= 60 else np.random.default_rng(len(f) + 1).choice(len(f), size=60, replace=False)
    for i in rows:
        bad = f.copy()
        bad[i] ^= 1
        with pytest.raises(AssertionError, match="check_flags"):
            dda.check_flags(Y, bad, chunk=64)


def test_failure_report_names_the_row_and_the_expected_dominator():
    Y = np.array([[0.0, 0.0], [1.0, 1.0], [2.0, 2.0], [2.0, 2.0]])
    with pytest.raises(AssertionError) as ei:
        dda.check_ranks(Y, np.array([0, 1, 1, 2]))
    msg = str(ei.value)
    assert "row 2: rank 1, expected 2 (dominator 1 with rank 1)" in msg and "1 row(s) wrong" in msg
    with pytest.raises(AssertionError) as ei:
        dda.check_flags(Y, np.array([0, 1, 0, 1]))
    assert "row 2: flag 0, expected 1 (dominated by row 0)" in str(ei.value)


def test_identical_rows_do_not_dominate_each_other():
    Y = np.array([[1.0, 1.0], [1.0, 1.0], [-0.0, 2.0], [0.0, 2.0]])
    dda.check_ranks(Y, np.array([0, 0, 0, 0]))
    dda.check_flags(Y, np.array([0, 0, 0, 0]))
