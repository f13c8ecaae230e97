"""The Monte-Carlo hypervolume estimators (csrc/hv_mc.cu) checked for EXACT equality with their draw-for-draw replay
(oracle/hv_mc_replay.py).

Every draw is a pure function of (seed, stream_id, purpose, sample index, draw index), the stopping rules are applied in
sample order to integer sums, and the host arithmetic is plain float64, so (value, samples, tests, algorithm) must equal
the replay bit for bit, whatever the wave and grid sizes.  The replay stops one sample at a time without waves, so a wave
that resumes at the wrong sample, a tile scan that miscounts its rows or a draw taken from the wrong Philox word changes
`samples` or `tests` even where it moves the estimate by far less than the statistical tests in
test_gpu_many_objectives.py can see.

Each case (oracle/hv_mc_cases.py) also asserts the edge it claims from the replay's record: the route taken, a discarded
straddling sample, first dominators at tile edges, redraw rounds, zero-volume boxes never chosen.
tests/test_hv_mc_replay_cpu.py checks the same claims without a GPU.
"""

import numpy as np
import pytest

from oracle import hv_mc_cases as cases
from oracle import hv_mc_replay as replay

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from dmosopt_b200 import _lib

    _lib.context()
    return _lib


def outcome(value, info):
    return (np.float64(value).tobytes(), info["samples"], info["tests"], info["algorithm"])


def run(L, F, ref, case):
    return L.hypervolume_mc(F, ref, case.algo, case.eps, case.delta, n_samples=case.n_samples, seed=case.seed, stream=case.stream)


@pytest.mark.parametrize("case", cases.CASES, ids=[c.id for c in cases.CASES])
def test_matches_the_replay(L, case):
    F, ref = cases.case_input(case)
    want = replay.hypervolume_mc(F, ref, **case.args())
    if case.claim:
        case.claim(F, ref, want[1])
    got = run(L, F, ref, case)
    assert outcome(*got) == outcome(*want), (got, want[0], {k: v for k, v in want[1].items() if k != "record"})


@pytest.mark.parametrize("algo", ["fpras", "mcm2rv", "hybrid", "monte_carlo"])
def test_dropped_rows_change_nothing(L, algo):
    """Rows on ref, NaN rows and dominated rows are dropped before the estimators run: the unfiltered input gives the
    filtered input's exact result, duplicated, zero-volume and subnormal-volume rows included."""
    F, junk, ref = cases.underflow_front()
    case = cases.Case("junk", None, algo, 0.15, 0.25, n_samples=20000, seed=9, stream=4)
    want = replay.hypervolume_mc(F, ref, **case.args())
    a = run(L, F, ref, case)
    b = run(L, np.vstack((junk[:3], F[:7], junk[3:], F[7:])), ref, case)
    assert outcome(*a) == outcome(*b) == outcome(*want)


def test_plugin_defaults_match_the_replay(L):
    """What dmosopt_b200.hv.AdaptiveHyperVolume runs for ten objectives: the hybrid at epsilon 0.01, delta 0.25, call i
    on stream i with HV_MC_DEFAULT_SEED."""
    from dmosopt_b200 import hv as bhv

    F, ref = cases.plugin_front()
    h = bhv.AdaptiveHyperVolume(ref)
    assert (h.mc_epsilon, h.mc_delta) == (0.01, 0.25)
    for stream in (0, 1):
        want, info = replay.hypervolume_mc(F, ref, "hybrid", 0.01, 0.25, seed=bhv.HV_MC_DEFAULT_SEED, stream=stream)
        assert info["algorithm"] == "MCM2RV" and info["record"]["ratio"] > 5.0, info["algorithm"]
        assert np.float64(h.compute_hypervolume(F)).tobytes() == np.float64(want).tobytes(), (stream, info["algorithm"])
