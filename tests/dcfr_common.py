"""Oracles of Discounted CFR for the parity tests: the pinned Linear / Vanilla CFR oracles (oracle/cfr_numpy.py in float32,
oracle/cfr2_numpy.py in float64) with DCFR's regret update and average weight, and nothing else changed.

DCFR at iteration counter i, t = i + 1, factors {a_t, b_t, w_t} = pokerrl_b200.dcfr.factors (float32):
    x = d + R_old,  R_new = x * (x > 0 ? a_t : b_t),  sigma = regret matching of R_new,  S += sigma * reach_p * w_t"""
import numpy as np

import cfr2_numpy as o2
from cfr_numpy import OracleCFR, OracleTree
from pokerrl_b200 import dcfr


def step_factors(params, i):
    """float32 (a_t, b_t, w_t) of iteration counter i"""
    a, b, w = dcfr.factors(*params, i + 1)[i]
    return a, b, w


class FastOracleTree(OracleTree):
    """OracleTree with the showdown rows of ValueFiller.py:127-158 computed for all of a seat's hands at once: per hand the
    same float32 additions and subtractions in the same (ascending opponent) order, so the same bits - 24-hand BigLeduc
    affordable for 50 iterations"""

    def _call_eq_final(self, reach, c):
        if not hasattr(self, "_masks"):
            self._masks = {}
        if c not in self._masks:  # per opponent hand: my hands it loses to / beats (both live, no shared card)
            hr, h = self.hand_ranks[c], np.arange(self.R)
            live = [(h != c) & (h != ho) & (ho != c) for ho in range(self.R)]
            self._masks[c] = [(live[ho] & (hr > hr[ho]), live[ho] & (hr < hr[ho])) for ho in range(self.R)]
        eq = np.zeros((2, self.R), np.float32)
        opp = reach[::-1]  # row p: the opponent's reach
        for ho, (gt, lt) in enumerate(self._masks[c]):
            r = opp[:, ho:ho + 1]
            eq = np.where(gt, eq + r, np.where(lt, eq - r, eq))
        return eq * self.eq_const


class OracleDCFR(OracleCFR):
    """float32, one-card games: the operation order of the kernels (csrc/cfr_levels.cu), bit for bit.  The schedule, values,
    regret matching and normalised average are Vanilla CFR's (OracleCFR), on a FastOracleTree."""

    def __init__(self, ft, params=dcfr.DEFAULT):
        self.params = tuple(params)
        self.ft, self.algo, self.delay = ft, "DCFR", 0
        self.tree = FastOracleTree(ft)
        self.R = self.tree.R
        self.ev_normalizer = ft.game_cls.EV_NORMALIZER
        self.curr_series, self.avg_series = [], []
        self.reset()

    def evaluate_avg(self):
        et = FastOracleTree(self.ft)
        et.fill_uniform()
        for n in et.decision_nodes():
            et.strategy[n] = np.copy(self.avg_strat[n])
        et.update_reach()
        return self._mbb(et.compute_ev())

    def _compute_regrets(self, p):
        ft, t = self.ft, self.tree
        a, b, _ = step_factors(self.params, self.iter_counter)
        for n in self._nodes_of(p):
            fc, A = ft.first_child[n], int(ft.n_children[n])
            ev_all = np.zeros((self.R, A), np.float32)
            for i in range(A):
                ev_all[:, i] = t.ev[fc + i, p]
            strat_ev = np.expand_dims(t.ev[n, p], axis=-1).repeat(A, axis=-1)
            last = self.regret[n] if self.iter_counter > 0 else np.zeros((self.R, A), np.float32)
            x = ev_all - strat_ev + last
            self.regret[n] = x * np.where(x > 0, a, b)

    def _add_strategy_to_average(self, p):
        ft, t = self.ft, self.tree
        _, _, w = step_factors(self.params, self.iter_counter)
        for n in self._nodes_of(p):
            A = int(ft.n_children[n])
            contrib = t.strategy[n] * np.expand_dims(t.reach[n, p], axis=1)
            contrib = contrib * w
            if self.iter_counter > 0:
                self.avg_strat_sum[n] += contrib
            else:
                self.avg_strat_sum[n] = contrib
            s = np.expand_dims(np.sum(self.avg_strat_sum[n], axis=1), axis=1)
            with np.errstate(divide="ignore", invalid="ignore"):
                self.avg_strat[n] = np.where(s == 0, np.full(shape=A, fill_value=1.0 / A), self.avg_strat_sum[n] / s)


class Oracle2DCFR:
    """float64, any flat tree, on an oracle/cfr2_numpy.Oracle2Tree, with the tables of the C oracle's interface:
    regret / avg = float64 [n_slots, R] (avg = the reach-weighted sums), half_iteration(p) without advancing the counter."""

    def __init__(self, tree, params=dcfr.DEFAULT, ev_normalizer=1.0):
        self.t, self.params, self.ev_normalizer = tree, tuple(params), ev_normalizer
        self.ft, self.R = tree.ft, tree.R
        ft = self.ft
        self.dec = np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]
        self.regret = np.zeros((ft.n_slots, self.R))
        self.avg = np.zeros((ft.n_slots, self.R))
        self.iter_counter = 0
        tree.fill_uniform()

    def _rows(self, n):
        fs, A = int(self.ft.first_slot[n]), int(self.ft.n_children[n])
        return slice(fs, fs + A), A

    @staticmethod
    def _matching(reg, A):  # reg [A, R] -> strategy [R, A]
        rp = np.maximum(reg, 0).T
        s = rp.sum(axis=1, keepdims=True)
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(s > 0, rp / s, 1.0 / A)

    def set_strategies_from_regrets(self):
        for n in self.dec:
            rows, A = self._rows(n)
            self.t.strategy[n] = self._matching(self.regret[rows], A)
        self.t.update_reach()

    def half_iteration(self, p):
        t, ft = self.t, self.ft
        a, b, w = (float(x) for x in step_factors(self.params, self.iter_counter))
        t.compute_ev()
        mine = self.dec[ft.kind[self.dec] == p]
        for n in mine:
            rows, A = self._rows(n)
            fc = ft.first_child[n]
            d = t.ev[fc:fc + A, p] - t.ev[n, p][None, :]
            x = d + self.regret[rows]
            self.regret[rows] = x * np.where(x > 0, a, b)
            t.strategy[n] = self._matching(self.regret[rows], A)
        t.update_reach()
        for n in mine:
            rows, _ = self._rows(n)
            self.avg[rows] += (t.strategy[n] * t.reach[n, p][:, None]).T * w

    def iteration(self, n=1):
        for _ in range(n):
            for p in (0, 1):
                self.half_iteration(p)
            self.iter_counter += 1

    def _metric(self, expl):
        return float(sum(expl[p] * self.ev_normalizer for p in range(2)) / 2)

    def exploitability_current(self):
        return self._metric(self.t.compute_ev())

    def exploitability_average(self):
        keep = self.t.strategy
        strat = list(keep)
        for n in self.dec:
            rows, A = self._rows(n)
            s = self.avg[rows].sum(axis=0)[:, None]
            with np.errstate(divide="ignore", invalid="ignore"):
                strat[n] = np.where(s == 0, 1.0 / A, self.avg[rows].T / s)
        self.t.strategy = strat
        self.t.update_reach()
        e = self._metric(self.t.compute_ev())
        self.t.strategy = keep
        self.t.update_reach()
        return e


class OneSeat(o2.Oracle2CFR):
    """the pinned float64 oracle (any of its algorithms) restricted to one seat's update: half_iteration(p) leaves the other
    seat's tables alone and does not advance the counter (the values and reach rows it recomputes are those of the
    unchanged profile); iteration() is a plain iteration of both seats"""

    seat = None  # None: both seats

    def _nodes_of(self, p):
        return super()._nodes_of(p) if self.seat is None or p == self.seat else np.zeros(0, np.int64)

    def half_iteration(self, p):
        self.seat = p
        k = self.iter_counter
        self.iteration()
        self.iter_counter, self.seat = k, None
