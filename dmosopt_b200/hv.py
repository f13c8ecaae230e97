"""Mirror of the hypervolume entry points on the GPU.

  * AdaptiveHyperVolume.compute_hypervolume   dmosopt/hv.py:123-241: 'box' exact (1 <= M <= 8); 'monte_carlo', 'fpras',
                                              'mcm2rv' and 'hybrid' (dmosopt/hv_adaptive.py) as Monte-Carlo estimates
                                              (2 <= M <= 16, csrc/hv_mc.cu)
  * HyperVolumeBoxDecomposition               dmosopt/hv_box_decomposition.py:62-351
  * compute_hypervolume_box_decomposition     dmosopt/hv_box_decomposition.py:445-464
"""

import numpy as np

from . import _lib


class HyperVolumeBoxDecomposition:
    def __init__(self, ref_point):
        self.ref_point = np.asarray(ref_point, dtype=np.float64)
        self.d = len(self.ref_point)

    def compute_hypervolume(self, points):
        points = np.asarray(points, dtype=np.float64)
        if len(points) == 0:
            return 0.0
        if points.shape[1] != self.d:
            raise ValueError(f"Points dimension {points.shape[1]} doesn't match ref point {self.d}")
        return _lib.hypervolume(points, self.ref_point)

    def select_candidates(self, pareto_front, candidate_means, candidate_variances, n_select=1, batch_size=100):
        sel, score = _lib.ehvi_select(pareto_front, candidate_means, candidate_variances, self.ref_point, n_select, nds=False, return_scores=True)
        return sel, score[sel]


def compute_hypervolume_box_decomposition(points, ref_point):
    return HyperVolumeBoxDecomposition(ref_point).compute_hypervolume(points)


HV_MC_DEFAULT_SEED = 0x5EED_4F7  # the Philox key of the Monte-Carlo estimators when seed is None


class AdaptiveHyperVolume:
    """dmosopt.hv.AdaptiveHyperVolume with the same constructor, plus ``seed`` for the Monte-Carlo estimators.

    Call i of ``compute_hypervolume`` draws with (seed, stream i mod 2^24): every call estimates afresh, and a sequence of
    calls is reproducible from the seed (None: HV_MC_DEFAULT_SEED)."""

    def __init__(self, ref_point, dimension_threshold_exact=10, monte_carlo_samples=100000, use_adaptive_mc=True, mc_epsilon=0.01,
                 mc_delta=0.25, seed=None):
        self.ref_point = np.asarray(ref_point, dtype=np.float64)
        self.n_objectives = len(self.ref_point)
        self.dimension_threshold_exact = dimension_threshold_exact
        self.monte_carlo_samples = monte_carlo_samples
        self.use_adaptive_mc = use_adaptive_mc
        self.mc_epsilon = mc_epsilon
        self.mc_delta = mc_delta
        self.seed = HV_MC_DEFAULT_SEED if seed is None else int(seed)
        self.calls = 0

    def compute_hypervolume(self, pareto_front, algorithm=None, verbose=False):
        pareto_front = np.asarray(pareto_front, dtype=np.float64)
        if len(pareto_front) == 0:
            return 0.0
        if algorithm in (None, "auto"):
            if self.n_objectives < self.dimension_threshold_exact:
                algorithm = "box"
            else:
                algorithm = "hybrid" if self.use_adaptive_mc else "monte_carlo"
        if algorithm == "box":
            return _lib.hypervolume(pareto_front, self.ref_point)
        if algorithm not in _lib.HVMC_ALGORITHMS:
            raise ValueError(f"Unknown algorithm: {algorithm}")
        value, info = _lib.hypervolume_mc(pareto_front, self.ref_point, algorithm, self.mc_epsilon, self.mc_delta, self.monte_carlo_samples,
                                          seed=self.seed, stream=self.calls % (1 << 24))
        self.calls += 1
        if verbose:
            print(f"Computing hypervolume using '{algorithm}' ({info['algorithm']}) for {self.n_objectives} objectives: "
                  f"{info['samples']} samples, {info['tests']} dominance tests")
        return value
