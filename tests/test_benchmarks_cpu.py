"""WFG1, MaF1/2/4 and generate_problem_space without a GPU: the vectorised oracle (oracle/benchmarks_many.py) and the
package's problem spaces against the reference's own outputs (tests/golden/benchmarks.npz), and the refusals that
happen before any launch."""

import numpy as np
import pytest

from conftest import load_golden
from dmosopt_b200 import benchmarks as bm
from oracle import benchmarks_many as obm


@pytest.fixture(scope="module")
def g():
    return load_golden("benchmarks")


def test_fixture_covers_every_new_problem_and_nan_rows(g):
    keys = [str(k) for k in g["keys"]]
    assert {k.split("_")[0] for k in keys} == {"wfg1", "maf1", "maf2", "maf4"}
    assert {int(k.split("_")[1]) for k in keys if k.startswith("maf")} == {3, 5, 10, 16}
    for k in keys:
        if k.startswith("wfg1"):
            assert np.isnan(g[k + "_Y"]).any(axis=1).sum() >= 3, k  # the nan and negative rows
            assert np.isfinite(g[k + "_Y"][:20]).all(), k


def test_oracle_against_reference_rows(g):
    for key in g["keys"]:
        key = str(key)
        nm, M, _ = key.split("_")
        Y = getattr(obm, nm)(g[key + "_X"], int(M))
        np.testing.assert_allclose(Y, g[key + "_Y"], rtol=1e-12, atol=0, equal_nan=True, err_msg=key)


def test_generate_problem_space_matches_reference(g):
    for i in range(int(g["n_spaces"])):
        nm, M, d = (str(a) for a in g[f"space{i}_args"])
        sp = bm.generate_problem_space(nm, int(M), int(d) if d else None)
        assert list(sp.keys()) == [str(s) for s in g[f"space{i}_names"]], (nm, M, d)
        assert all(type(v) is list and len(v) == 2 and all(type(b) is float for b in v) for v in sp.values())
        assert np.array_equal(np.array(list(sp.values()), dtype=np.float64), g[f"space{i}_bounds"]), (nm, M, d)


def test_generate_problem_space_defaults():
    assert len(bm.generate_problem_space("maf1", 5)) == 14 and len(bm.generate_problem_space("wfg1", 3)) == 12
    assert len(bm.generate_problem_space("dtlz3", 3)) == 7 and len(bm.generate_problem_space("dtlz7", 3)) == 22
    assert len(bm.generate_problem_space("unknown", 4)) == 14
    assert bm.generate_problem_space("wfg4", 2, 3) == {"x1": [0.0, 2.0], "x2": [0.0, 4.0], "x3": [0.0, 6.0]}


@pytest.fixture
def no_launch(monkeypatch):
    from dmosopt_b200 import _lib

    def refuse(*a, **k):
        raise AssertionError("the refusal must come before any library call")

    monkeypatch.setattr(_lib, "benchmark_eval", refuse)


def test_wfg1_empty_windows_refused_where_the_reference_raises(g, no_launch):
    rng = np.random.default_rng(3)
    for (M, d), err in zip(g["wfg1_raising_shapes"], g["wfg1_raising_errors"]):
        M, d = int(M), int(d)
        X = rng.random((4, d)) * 2 * np.arange(1, d + 1)
        if str(err) == "ValueError":
            for x in (X, X[0]):
                with pytest.raises(ValueError, match="empty"):
                    bm.wfg1(x, M)
            with pytest.raises(ValueError):
                obm.wfg1(X, M)
        else:
            assert str(err) == "", err
            assert (M - 2) * (d - M + 1) < d
            with pytest.raises(AssertionError, match="before any library call"):  # accepted: goes on to the launch
                bm.wfg1(X, M)
            assert obm.wfg1(X, M).shape == (4, M)
    # at n_obj >= 4 the reference's default n_var = n_obj + 9 always has an empty window
    for M in range(4, 17):
        with pytest.raises(ValueError):
            bm.wfg1(np.ones(M + 9), M)


def test_wfg_position_parameter_other_than_default_refused(no_launch):
    x = np.ones(12)
    for fn in (bm.wfg1, bm.wfg4):
        with pytest.raises(NotImplementedError):
            fn(x, 3, k=4)
    with pytest.raises(AssertionError, match="before any library call"):  # k = n_obj - 1 spelled out is the default
        bm.wfg1(x, 3, k=2)
