"""Host logic of the resident MO-CMA-ES surrogate epoch (dmosopt_b200.MOASMO.optimize on dmo_cmaes_step_record /
dmo_cmaes_step_apply) without a GPU: which CMAES epochs are eligible, the shared host arithmetic of update_strategy
against the plugin's former inline code, and the positional front cut of the step against CMAES._select."""

import numpy as np
import pytest

import fake_backend


class _FakeGP:
    pass


def _gp(mean_variance=False, handle=True):
    import dmosopt_b200 as b2

    sm = b2.GPR_Matern.__new__(b2.GPR_Matern)
    sm._gp, sm.return_mean_variance = (_FakeGP() if handle else None), mean_variance
    return sm


def _cmaes(model, cls=None, **kw):
    import dmosopt_b200 as b2

    return (cls or b2.CMAES)(popsize=10, nInput=3, nOutput=2, model=model, **kw)


class _Feasibility:
    def rank(self, x):
        return np.zeros(len(x))


def test_eligibility():
    import dmosopt_b200 as b2
    from dmosopt_b200.MOASMO import resident_eligible

    class _Sub(b2.CMAES):
        pass

    m = b2.Model(objective=_gp())
    assert resident_eligible(_cmaes(m), m)
    # CMAES's sortMO never reads the y-metric
    for metric in ("crowding", "euclidean", lambda y: y[:, 0]):
        assert resident_eligible(_cmaes(m, distance_metric=metric), m)

    assert not resident_eligible(_cmaes(m, cls=_Sub), m)
    assert not resident_eligible(_cmaes(m, adaptive_population_size=True), m)
    assert not resident_eligible(_cmaes(m, optimize_mean_variance=True), m)
    assert not resident_eligible(_cmaes(m), m, optimize_mean_variance=True)
    for sm in (_gp(mean_variance=True), _gp(handle=False), None):
        mm = b2.Model(objective=sm)
        assert not resident_eligible(_cmaes(mm), mm)
    mf = b2.Model(objective=_gp())
    mf.feasibility = _Feasibility()
    opt = _cmaes(mf)
    assert opt.x_distance_metrics is not None and not resident_eligible(opt, mf)


def _inline_update(p, psucc, pidx, C, chosen, not_chosen):
    """update_strategy's host arithmetic as the plugin computed it inline before it moved into _strategy_scalars."""
    from dmosopt_b200.CMAES import _stable_order

    cp, d, ptarg = p.cp, p.d, p.ptarg
    fac = lambda ps: np.exp((ps - ptarg) / (d * (1.0 - ptarg)))  # noqa: E731
    ch_off = np.flatnonzero(chosen[:C])
    par = pidx[ch_off]
    off_psucc = (1.0 - cp) * psucc[par] + cp
    off_fac = fac(off_psucc)
    new_psucc = psucc.copy()
    nc_off = np.flatnonzero(not_chosen[:C])
    ev_parent = np.concatenate((par, pidx[nc_off]))
    ev_success = np.concatenate((np.ones(len(par), dtype=bool), np.zeros(len(nc_off), dtype=bool)))
    seg = None
    if len(ev_parent) > 0:
        order = _stable_order(ev_parent)
        ep, es = ev_parent[order], ev_success[order]
        first = np.r_[True, ep[1:] != ep[:-1]]
        seg_start = np.flatnonzero(first)
        k_in_parent = np.arange(len(ep)) - np.repeat(seg_start, np.diff(np.r_[seg_start, len(ep)]))
        f_ev = np.empty(len(ep))
        for k in range(int(k_in_parent.max()) + 1):
            sel = np.flatnonzero(k_in_parent == k)
            q = ep[sel]
            new_psucc[q] = (1.0 - cp) * new_psucc[q] + np.where(es[sel], cp, 0.0)
            f_ev[sel] = fac(new_psucc[q])
        seg = (f_ev, ep[seg_start], np.r_[seg_start, len(ep)])
    ch = np.flatnonzero(chosen)
    ch_is_off = ch < C
    slot = np.full(len(chosen), -1, dtype=np.int64)
    slot[ch_off] = np.arange(len(ch_off))
    src_par = pidx[ch]
    psucc_n = new_psucc[src_par]
    src_idx = src_par.astype(np.int64)
    if len(ch_off) > 0:
        o = slot[ch[ch_is_off]]
        psucc_n[ch_is_off] = off_psucc[o]
        src_idx[ch_is_off] = o
    return ch_off, par, off_psucc, off_fac, seg, ch, src_idx, psucc_n


@pytest.mark.parametrize("P,lambda_,share", [(10, 1, 0.5), (11, 2, 0.3), (64, 1, 0.0), (64, 2, 1.0), (257, 2, 0.6)])
def test_strategy_scalars_are_the_former_inline_arithmetic(P, lambda_, share):
    import dmosopt_b200 as b2
    from dmosopt_b200.CMAES import _strategy_scalars

    opt = b2.CMAES(popsize=P, nInput=4, nOutput=2, model=b2.Model(), lambda_=lambda_)
    p = opt.opt_params
    rng = np.random.default_rng(P * 7 + lambda_)
    mu = p.mu
    C = lambda_ * mu
    psucc = rng.random(P)
    pidx = np.concatenate((rng.integers(0, mu, C), np.arange(P))).astype(np.int64)
    # P of the C + P candidates are chosen; share: the fraction of them that are offspring
    n_off = min(C, int(round(share * P)))
    chosen = np.zeros(C + P, dtype=bool)
    chosen[rng.choice(C, n_off, replace=False)] = True
    chosen[C + rng.choice(P, P - n_off, replace=False)] = True
    h = _strategy_scalars(p, psucc, pidx, C, chosen, ~chosen)
    ch_off, par, off_psucc, off_fac, seg, ch, src_idx, psucc_n = _inline_update(p, psucc, pidx, C, chosen, ~chosen)
    for got, want in ((h.ch_off, ch_off), (h.par, par), (h.off_psucc, off_psucc), (h.off_fac, off_fac), (h.ch, ch), (h.src_idx, src_idx),
                      (h.psucc, psucc_n)):
        assert got.dtype == want.dtype and np.array_equal(got, want)
    if seg is None:
        assert len(h.seg_row) == 0 and len(h.ev_fac) == 0
    else:
        assert np.array_equal(h.ev_fac, seg[0]) and np.array_equal(h.seg_row, seg[1]) and np.array_equal(h.seg_start, seg[2])
    assert len(h.ch) == P


def _positional_cut(rank, pop):
    """The step's front cut: cumulative front sizes b, the mid front [b_R, b_R+1) with b_R <= pop < b_R+1."""
    b = np.r_[0, np.cumsum(np.bincount(rank, minlength=len(rank)))]
    R = int(np.flatnonzero((b[:-1] <= pop) & (b[1:] > pop))[0])
    return int(b[R]), int(b[R + 1])


class _Picks:
    """A stand-in for the hypervolume-improvement selection: records its inputs, picks the last k candidates."""

    calls = []

    def __init__(self, ref_point, nds):
        self.ref = ref_point

    def do(self, F, means, variances, k):
        _Picks.calls.append((F, means, k))
        return np.arange(len(means) - k, len(means))


@pytest.mark.parametrize("seed,n,pop,fronts", [(1, 30, 20, 4), (2, 30, 20, 1), (3, 40, 20, 40), (4, 25, 12, 5), (5, 64, 32, 8)])
def test_positional_front_cut_matches_select(monkeypatch, seed, n, pop, fronts):
    import dmosopt_b200 as b2
    from dmosopt_b200 import _lib

    fake_backend.install(monkeypatch)
    rng = np.random.default_rng(seed)
    rank = np.sort(rng.integers(0, fronts, n))
    rank = np.unique(rank, return_inverse=True)[1]  # contiguous ranks 0..max
    rank = rank[rng.permutation(n)]
    monkeypatch.setattr(_lib, "rank_nd", lambda Y: rank.astype(np.intp))
    Y = rng.random((n, 2))
    opt = b2.CMAES(popsize=pop, nInput=3, nOutput=2, model=b2.Model())
    opt.indicator = _Picks
    _Picks.calls.clear()
    chosen, not_chosen, r = opt._select(None, Y, None, None)
    lo, hi = _positional_cut(rank, pop)
    k = pop - lo
    want = np.zeros(n, dtype=bool)
    want[:lo] = True
    if k > 0:
        picks = np.arange(k) if lo == 0 else np.arange(hi - lo - k, hi - lo)
        want[lo + picks] = True
        if lo > 0:
            (F, means, kk), = _Picks.calls
            assert kk == k and np.array_equal(F, Y[:lo]) and np.array_equal(means, Y[lo:hi])
        else:
            assert not _Picks.calls
    assert np.array_equal(chosen, want) and np.array_equal(not_chosen, ~want) and np.count_nonzero(chosen) == pop
