#!/usr/bin/env python
"""Generate tests/golden/early_stopping.npz from the *reference itself*: the early-stopping rule of its exact-GP training.

Run with the reference package importable (a checkout of dmosopt on PYTHONPATH; gpytorch is not needed, the module
imports with ``_has_gpytorch = False``):

    PYTHONPATH=<dmosopt checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_early_stopping.py

Nothing outside ``tests/golden/`` is written.
"""

import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def save(name, **arrays):
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **arrays)
    print(f"wrote {name}.npz  ({os.path.getsize(path)} bytes)")


def early_stopping_sequences(rng, n=3000):
    """Seeded loss sequences for the exact-GP early-stopping rule: (names, (6, n) array)."""
    it = np.arange(n, dtype=np.float64)
    seqs = {
        "exponential_decay": 1.0 + 5.0 * np.exp(-it / 300.0),
        "plateau": 2.0 + 3.0 * np.exp(-it / 50.0),
        "noisy_plateau": 2.0 + 3.0 * np.exp(-it / 100.0) + 0.01 * rng.standard_normal(n),
        "slow_drift": 5.0 - 2e-4 * it + 1e-5 * rng.standard_normal(n),
        "oscillation": 2.0 + 0.5 * np.sin(it / 20.0) * np.exp(-it / 2000.0),
        "never_converging": 10.0 + np.cumsum(0.5 * rng.standard_normal(n)),
    }
    return list(seqs), np.stack(list(seqs.values()))


def gen_early_stopping():
    """AdaptiveEarlyStopping with EarlyStoppingConfig.for_model_type(EXACT_GP) and threshold_pct = 0.1 (the default
    min_loss_pct_change), driven as MEGP_Matern's training loop drives it (dmosopt/model_gpytorch.py:1769-1816): the loss
    of iteration it is appended, and from it = warmup_iterations on should_stop(it, losses) is asked.  Records the
    iteration it at which the loop breaks (-1: never) and the reason."""
    from dmosopt.model_gpytorch import AdaptiveEarlyStopping, EarlyStoppingConfig, ModelType

    rng = np.random.default_rng(31)
    names, losses = early_stopping_sequences(rng)
    stop_it, reasons = [], []
    for seq in losses:
        config = EarlyStoppingConfig.for_model_type(ModelType.EXACT_GP)
        config.threshold_pct = 0.1
        es = AdaptiveEarlyStopping(config)
        log, at, why = [], -1, ""
        for it, v in enumerate(seq):
            log.append(float(v))
            if it >= config.warmup_iterations:
                stop, reason = es.should_stop(it, np.array(log), compute_validation=None)
                if stop:
                    at, why = it, reason
                    break
        stop_it.append(at)
        reasons.append(why)
    save("early_stopping", names=np.array(names), losses=losses, stop_it=np.array(stop_it), reasons=np.array(reasons))


if __name__ == "__main__":
    gen_early_stopping()
