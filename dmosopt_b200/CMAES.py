"""MO-CMA-ES optimizer plugin on the GPU path.

Drop-in for ``dmosopt.CMAES.CMAES`` (dmosopt/CMAES.py:26-537), selected by ``optimizer_name="dmosopt_b200.CMAES"``.

  generate_strategy : non-dominated rank of the parents (dmo_rank_nd), parent draw, then
                      x = x_p + sigma_p * (A_p @ z) for lambda*mu offspring (dmo_cmaes_sample; CMAES.py:231-271)
  _select           : rank of offspring + parents, whole fronts first, the overflowing front split by the
                      hypervolume-improvement score (dmo_ehvi_select; CMAES.py:167-229)
  update_strategy   : success-rate / step-size recurrences (vectorised on the host, O(n) scalars) and the rank-one
                      Cholesky updates of all chosen offspring in one batch (dmo_cmaes_update_cholesky;
                      CMAES.py:273-414, 489-537)
"""

from concurrent.futures import ThreadPoolExecutor
from typing import Any, Dict, Optional

import numpy as np

from . import _lib
from .MOEA import MOEA, Struct, remove_duplicates, remove_worst
from .NSGA2 import population_diversity
from .indicators import HypervolumeImprovement


def sortMO(x, y, x_distance_metrics=None):
    """CMAES.sortMO (CMAES.py:455-486): (perm, rank) with rank in the original order."""
    rank = _lib.rank_nd(y)
    keys = []
    if x_distance_metrics:
        rmax = int(rank.max())
        for fn in x_distance_metrics:
            dist = np.zeros_like(rank)
            for front in range(rmax + 1):
                idx = rank == front
                dist[idx] = fn(x[idx, :])
            keys.append(-dist)
    if not keys:  # np.lexsort((rank,)) is a stable sort by rank
        return _stable_order(rank), rank
    return np.lexsort(keys + [rank]), rank


# one worker thread: generate_strategy ranks the parents on the GPU while the calling thread draws the normal variates
# (both release the GIL; the library is not re-entrant, so the caller makes no library call until it has joined)
_worker = ThreadPoolExecutor(max_workers=1, thread_name_prefix="dmosopt_b200_cmaes")


def _stable_order(rank):
    """np.argsort(rank, kind="stable") for non-negative integers: NumPy sorts 16-bit keys with a radix sort, so one or two
    16-bit passes (least significant half first) beat its merge sort on 64-bit keys by 3x at the sizes of this plugin."""
    rank = np.asarray(rank)
    if rank.size == 0 or int(rank.min()) < 0:
        return np.argsort(rank, kind="stable")
    top = int(rank.max())
    if top < 65536:
        return np.argsort(rank.astype(np.uint16), kind="stable")
    if top < (1 << 32):
        low = np.argsort((rank & 0xFFFF).astype(np.uint16), kind="stable")
        return low[np.argsort((rank[low] >> 16).astype(np.uint16), kind="stable")]
    return np.argsort(rank, kind="stable")


def _strategy_scalars(p, psucc, pidx, C, chosen, not_chosen):
    """The host arithmetic of update_strategy (CMAES.py:273-411), shared by the plugin and MOASMO's resident generation:
    the success rates and step-size factors are NumPy's (its float64 ``exp`` is not CUDA's), everything they scale stays
    on the device.  ``p`` the optimizer parameters, ``psucc`` the parents' success rates, ``pidx`` the parent of each of
    the C + P candidates (offspring first), ``chosen`` / ``not_chosen`` the selection masks.  Returns a Struct of
      ch_off, par, off_psucc, off_fac   the chosen offspring (candidate rows), their parents, success rates and step-size
                                        factors;
      seg_row, seg_start, ev_fac        the parents' success / failure events: one segment per parent, its factors in
                                        order (dmo_scale_rows);
      ch, src_idx, psucc                the next parent set: candidate rows, the strategy rows each takes (an index into
                                        the chosen offspring when ch < C, else into the parents) and its success rates."""
    cp, d, ptarg = p.cp, p.d, p.ptarg
    fac = lambda ps: np.exp((ps - ptarg) / (d * (1.0 - ptarg)))  # noqa: E731

    # chosen offspring: their success rate advances from the parent's
    ch_off = np.flatnonzero(chosen[:C])  # offspring are the first C candidates
    par = pidx[ch_off]
    off_psucc = (1.0 - cp) * psucc[par] + cp
    off_fac = fac(off_psucc)

    # parents: one success event per chosen offspring (ascending candidate index), then one failure event per not-chosen
    # offspring; the recurrences are sequential per parent: the scalar success rates are advanced event rank by event rank
    # here, the step-size rows take their factors in the same order on the device
    new_psucc = psucc.copy()
    nc_off = np.flatnonzero(not_chosen[:C])
    ev_parent = np.concatenate((par, pidx[nc_off]))
    ev_success = np.concatenate((np.ones(len(par), dtype=bool), np.zeros(len(nc_off), dtype=bool)))
    seg_row, seg_start, f_ev = np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64), np.zeros(0)
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
        seg_row, seg_start = ep[seg_start], np.r_[seg_start, len(ep)]

    # the next parent set (CMAES.py:385-411)
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
        src_idx[ch_is_off] = o  # these rows come from the updated offspring arrays
    return Struct(ch_off=ch_off, par=par, off_psucc=off_psucc, off_fac=off_fac, seg_row=seg_row, seg_start=seg_start, ev_fac=f_ev, ch=ch,
                  src_idx=src_idx, psucc=psucc_n)


class CMAES(MOEA):
    def __init__(
        self,
        popsize: int,
        nInput: int,
        nOutput: int,
        model: Optional[Any] = None,
        distance_metric: Optional[Any] = None,
        optimize_mean_variance: bool = False,
        **kwargs,
    ):
        super().__init__(name="CMAES", popsize=popsize, nInput=nInput, nOutput=nOutput, optimize_mean_variance=optimize_mean_variance, **kwargs)
        self.model = model
        self.x_distance_metrics = None
        if getattr(self.model, "feasibility", None) is not None:
            self.x_distance_metrics = [self.model.feasibility.rank]
        if np.isscalar(self.opt_params.di_mutation):
            self.opt_params.di_mutation = np.asarray([self.opt_params.di_mutation] * nInput)
        self.state = None
        self.indicator = HypervolumeImprovement
        self.optimize_mean_variance = optimize_mean_variance

    @property
    def default_parameters(self) -> Dict[str, Any]:
        """CMAES.py:82-120."""
        nInput, nOutput, popsize = self.nInput, self.nOutput, self.popsize
        ptarg = 1.0 / (5.0 + 0.5)
        return {
            "sigma": 0.001,
            "mu": popsize // 2,
            "lambda_": 1,
            "d": 1.0 + nOutput / 2.0,
            "ptarg": ptarg,
            "cp": ptarg / (1.0 + ptarg),
            "cc": 2.0 / (nInput + 2.0),
            "ccov": 2.0 / (nInput**2 + 6.0),
            "pthresh": 0.44,
            "di_mutation": 30.0,
            "max_population_size": 600,
            "min_population_size": 100,
            "adaptive_population_size": False,
        }

    def initialize_state(self, x, y, bounds, local_random=None, **params):
        """CMAES.py:122-165."""
        dim, n = self.nInput, self.opt_params.popsize
        p = self.opt_params
        sigmas = np.asarray([p.sigma * (1.0 / (p.di_mutation + 1.0))] * n)
        # the per-parent Cholesky factors, their inverses and the evolution paths live in HBM (_lib.ResidentRows): at pop
        # 131 072, d = 24 they are 1.2 GB that the reference re-indexes on the host every generation; NumPy still sees
        # them as arrays (np.asarray(state.A), state.A[i]) through a device -> host copy on demand
        A = _lib.identity_rows(n, dim)
        Ainv = _lib.identity_rows(n, dim)
        pc = _lib.resident_rows(np.zeros((n, dim)))
        psucc = np.asarray([p.ptarg] * n)
        order, rank = sortMO(x, y, self.x_distance_metrics)
        idx = order[:n]
        # parents_x and sigmas are (n, dim) per-parent rows as well: resident, read by NumPy on demand
        return Struct(bounds=bounds, parents_x=_lib.resident_rows(x[idx]), parents_y=y[idx].copy(), sigmas=_lib.resident_rows(sigmas), A=A, Ainv=Ainv,
                      pc=pc, psucc=psucc, rank=rank[idx].copy())

    def _select(self, candidates_x, candidates_y, candidates_ps, candidates_inds):
        """CMAES.py:167-229."""
        popsize = self.opt_params.popsize
        n = candidates_y.shape[0]  # candidates_x is only materialised on the host when x distance metrics need it
        if n <= popsize:
            return np.ones(n, dtype=bool), np.zeros(n, dtype=bool), _lib.rank_nd(candidates_y)
        order, rank = sortMO(candidates_x, candidates_y, self.x_distance_metrics)
        order_inv = np.empty(n, dtype=np.intp)  # np.argsort(order): the inverse permutation
        order_inv[order] = np.arange(n)
        chosen = np.zeros(n, dtype=bool)
        not_chosen = np.zeros(n, dtype=bool)
        mid_front = None
        full = False
        chosen_count = 0
        # indices grouped by rank, ascending inside a front (= np.argwhere(rank == r) front by front); without extra sort keys
        # that is the order sortMO has just computed
        by_rank = order if not self.x_distance_metrics else np.argsort(rank, kind="stable")
        bounds_r = np.searchsorted(rank[by_rank], np.arange(int(np.max(rank)) + 2))
        for r in range(int(np.max(rank)) + 1):
            front_r = order_inv[by_rank[bounds_r[r] : bounds_r[r + 1]]]  # (sic) the reference maps fronts through order_inv (:190)
            if chosen_count + len(front_r) <= popsize and not full:
                chosen[front_r] = True
                chosen_count += len(front_r)
            elif mid_front is None and chosen_count < popsize:
                mid_front = front_r.copy()
                full = True
            else:
                not_chosen[front_r] = True
        k = popsize - chosen_count
        if k > 0:
            ref = np.max(candidates_y, axis=0) + 1
            indicator = self.indicator(ref_point=ref, nds=True)
            assert len(mid_front) > 0
            if chosen_count > 0:
                selected = indicator.do(candidates_y[chosen], candidates_y[mid_front, :], np.ones_like(candidates_y[mid_front, :]), k)
            else:
                selected = np.arange(k)
            assert len(selected) == k
            chosen[mid_front[selected]] = True
            mask = np.ones(len(mid_front), dtype=bool)
            mask[selected] = False
            not_chosen[mid_front[mask]] = True
        return chosen, not_chosen, rank

    def generate_strategy(self, **params):
        """CMAES.py:231-271."""
        rng = self.local_random
        st = self.state
        dim, mu, lambda_ = self.nInput, self.opt_params.mu, self.opt_params.lambda_
        if self.x_distance_metrics:  # host callables: keep everything on the calling thread
            arz = rng.normal(size=(lambda_ * mu, dim))
            order, rank = sortMO(np.asarray(st.parents_x), st.parents_y, self.x_distance_metrics)
        else:  # same draws in the same order (sortMO consumes no random numbers), the device rank overlaps them
            pending = _worker.submit(sortMO, None, st.parents_y, None)
            arz = rng.normal(size=(lambda_ * mu, dim))
            order, rank = pending.result()
        # fronts in rank order until at least mu parents are collected (CMAES.py:249-258) == the first mu indices of a
        # stable sort by rank
        parent_selection = (order if not self.x_distance_metrics else _stable_order(rank))[:mu]
        js = rng.choice(len(parent_selection), size=lambda_ * mu)
        p_idx = parent_selection[js]
        # sample, the reference's global rescale (sic, CMAES.py:269-270) and MOEA.generate's clip on the device; the
        # offspring matrix comes back read-only with its device copy kept for the surrogate and the update
        x_new = _lib.cmaes_generate(st.parents_x, st.sigmas, st.A, p_idx, arz, self.bounds[:, 0], self.bounds[:, 1])
        return x_new, {"p_idx": p_idx}

    def update_strategy(self, x_gen, y_gen, state, **params):
        """CMAES.py:273-414.  Scalars per individual (success rates, step-size factors, selection masks) are computed on
        the host; every (n, dim) / (n, dim, dim) array (positions, step sizes, factors, paths) stays in HBM and is
        re-assembled there."""
        st, p = self.state, self.opt_params
        p_idxs = np.asarray(state["p_idx"])
        xlb, xub = self.bounds[:, 0], self.bounds[:, 1]
        P, C = st.parents_x.shape[0], x_gen.shape[0]
        xg_d, px_d, sig_d = _lib.rows_of(x_gen), _lib.rows_of(st.parents_x), _lib.rows_of(st.sigmas)
        A_d, Ainv_d, pc_d = _lib.resident_rows(st.A), _lib.resident_rows(st.Ainv), _lib.resident_rows(st.pc)
        candidates_y = np.vstack((y_gen, st.parents_y))
        candidates_x = np.vstack((np.asarray(x_gen), np.asarray(px_d))) if self.x_distance_metrics else None
        is_off = np.concatenate((np.ones(C, dtype=bool), np.zeros(P, dtype=bool)))
        pidx = np.concatenate((p_idxs, np.arange(P, dtype=np.int_)))
        chosen, not_chosen, rank = self._select(candidates_x, candidates_y, is_off, pidx)
        h = _strategy_scalars(p, st.psucc, pidx, C, chosen, not_chosen)

        # ---- chosen offspring: their own strategy parameters start from the parent's (copied before any update)
        last_steps = _lib.gather_rows(sig_d, h.par)
        off_sigmas = _lib.scale_rows(_lib.gather_rows(sig_d, h.par), h.off_fac)
        off_A, off_Ainv, off_pc = _lib.gather_rows(A_d, h.par), _lib.gather_rows(Ainv_d, h.par), _lib.gather_rows(pc_d, h.par)
        if len(h.ch_off) > 0:
            z = _lib.cmaes_step_z(xg_d, h.ch_off, px_d, h.par, xlb, xub, last_steps)
            off_A, off_Ainv, off_pc = _lib.cmaes_update_cholesky(off_A, off_Ainv, off_pc, z, h.off_psucc, p.cc, p.ccov, p.pthresh)
        # ---- parents: the step-size rows take their event factors in order, in place (the old rows were copied above)
        if len(h.seg_row) > 0:
            _lib.scale_rows(sig_d, h.ev_fac, seg_row=h.seg_row, seg_start=h.seg_start)

        # ---- assemble the next parent set (CMAES.py:385-411): one device-side gather per state array, a surviving
        # parent keeps its rows, a chosen offspring brings its own
        ch, src_idx = h.ch, h.src_idx
        ch_is_off = ch < C
        sel = ch_is_off if len(h.ch_off) > 0 else None
        alt = (lambda a: a) if sel is not None else (lambda a: None)
        sigmas_n = _lib.gather_rows(sig_d, src_idx, alt=alt(off_sigmas), sel=sel)
        A_n = _lib.gather_rows(A_d, src_idx, alt=alt(off_A), sel=sel)
        Ainv_n = _lib.gather_rows(Ainv_d, src_idx, alt=alt(off_Ainv), sel=sel)
        pc_n = _lib.gather_rows(pc_d, src_idx, alt=alt(off_pc), sel=sel)
        x_idx = np.where(ch_is_off, ch, ch - C)  # candidate row -> row of x_gen / of the old parents
        st.parents_x = _lib.gather_rows(px_d, x_idx, alt=alt(xg_d), sel=sel)
        st.parents_y = candidates_y[ch]
        st.rank = rank[ch]
        st.sigmas, st.A, st.Ainv, st.pc, st.psucc = sigmas_n, A_n, Ainv_n, pc_n, h.psucc
        _lib.mirror_drop(x_gen)  # the offspring matrix has been consumed: callers that keep it hold host memory only
        if p.adaptive_population_size:
            self.update_population_size()

    def get_population_strategy(self):
        """CMAES.py:416-430."""
        x, y = remove_duplicates(np.asarray(self.state.parents_x), self.state.parents_y.copy())
        if len(x) > 0:
            x, y, _ = remove_worst(x, y, self.popsize)
        return x, y

    def update_population_size(self):
        """CMAES.py:432-452."""
        p = self.opt_params
        diversity, cd_spread = population_diversity(self.state.rank, self.state.parents_y)
        if diversity < 0.1 or cd_spread < 2.0:
            new_size = min(p.max_population_size, int(p.popsize * 1.1))
        elif diversity > 0.4 and cd_spread > 1.0:
            new_size = max(p.min_population_size, int(p.popsize * 0.9))
        else:
            new_size = p.popsize
        p.popsize = new_size
        p.mu = p.popsize // 2
