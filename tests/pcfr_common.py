"""Oracles of Predictive CFR+ for the parity tests, built like tests/dcfr_common.py builds DCFR's: the pinned float32 oracle
(oracle/cfr_numpy.py) and a float64 restatement on oracle/cfr2_numpy.Oracle2Tree, with PCFR+'s rules and nothing else changed.

PCFR+ at iteration counter i, t = i + 1, w_t = pokerrl_b200.dcfr.factors(*pcfr_params(gamma))[i, 2] (float32), d = v(child) - v(node):
    R_new = max(d + R_old, 0),  Q = max(R_new + d, 0),  sigma = regret matching of Q,  S += sigma * reach_p * w_t"""
import numpy as np

from cfr_numpy import OracleCFR
from dcfr_common import FastOracleTree
from pokerrl_b200 import dcfr


def step_weight(gamma, i):
    """float32 w_t of iteration counter i"""
    return dcfr.factors(*dcfr.pcfr_params(gamma), i + 1)[i, 2]


class OraclePCFR(OracleCFR):
    """float32, one-card games: the operation order of the kernels (csrc/cfr_levels.cu, PRED), bit for bit.  Schedule, values
    and the normalised average are Vanilla CFR's (OracleCFR) on a FastOracleTree; `pred` holds the predictions Q per node."""

    def __init__(self, ft, gamma=2.0):
        self.gamma = float(gamma)
        self.ft, self.algo, self.delay = ft, "PCFRPlus", 0
        self.tree = FastOracleTree(ft)
        self.R = self.tree.R
        self.ev_normalizer = ft.game_cls.EV_NORMALIZER
        self.curr_series, self.avg_series = [], []
        self.reset()

    def reset(self):
        self.pred = [None] * self.ft.n_nodes
        super().reset()

    def evaluate_avg(self):
        et = FastOracleTree(self.ft)
        et.fill_uniform()
        for n in et.decision_nodes():
            et.strategy[n] = np.copy(self.avg_strat[n])
        et.update_reach()
        return self._mbb(et.compute_ev())

    def _compute_regrets(self, p):
        ft, t = self.ft, self.tree
        for n in self._nodes_of(p):
            fc, A = ft.first_child[n], int(ft.n_children[n])
            ev_all = np.zeros((self.R, A), np.float32)
            for i in range(A):
                ev_all[:, i] = t.ev[fc + i, p]
            d = ev_all - np.expand_dims(t.ev[n, p], axis=-1).repeat(A, axis=-1)
            last = self.regret[n] if self.regret[n] is not None else np.zeros((self.R, A), np.float32)
            self.regret[n] = np.maximum(d + last, np.float32(0))
            self.pred[n] = np.maximum(self.regret[n] + d, np.float32(0))

    def _compute_new_strategy(self, p):
        for n in self._nodes_of(p):
            A = int(self.ft.n_children[n])
            q = self.pred[n]
            q_sum = np.expand_dims(np.sum(q, axis=1), axis=1).repeat(A, axis=1)
            with np.errstate(divide="ignore", invalid="ignore"):
                self.tree.strategy[n] = np.where(q_sum > 0.0, q / q_sum,
                                                 np.full(shape=(self.R, A), fill_value=1.0 / A, dtype=np.float32))

    def _add_strategy_to_average(self, p):
        ft, t = self.ft, self.tree
        w = step_weight(self.gamma, self.iter_counter)
        for n in self._nodes_of(p):
            A = int(ft.n_children[n])
            contrib = (t.strategy[n] * np.expand_dims(t.reach[n, p], axis=1)) * w
            if self.iter_counter > 0:
                self.avg_strat_sum[n] += contrib
            else:
                self.avg_strat_sum[n] = contrib
            s = np.expand_dims(np.sum(self.avg_strat_sum[n], axis=1), axis=1)
            with np.errstate(divide="ignore", invalid="ignore"):
                self.avg_strat[n] = np.where(s == 0, np.full(shape=A, fill_value=1.0 / A), self.avg_strat_sum[n] / s)


class Oracle2PCFR:
    """float64, any flat tree, on an oracle/cfr2_numpy.Oracle2Tree: regret / pred / avg = float64 [n_slots, R] (avg = the
    reach-weighted sums), half_iteration(p) without advancing the counter."""

    def __init__(self, tree, gamma=2.0, ev_normalizer=1.0):
        self.t, self.gamma, self.ev_normalizer = tree, float(gamma), ev_normalizer
        self.ft, self.R = tree.ft, tree.R
        ft = self.ft
        self.dec = np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]
        self.regret = np.zeros((ft.n_slots, self.R))
        self.pred = np.zeros((ft.n_slots, self.R))
        self.avg = np.zeros((ft.n_slots, self.R))
        self.iter_counter = 0
        tree.fill_uniform()

    def _rows(self, n):
        fs, A = int(self.ft.first_slot[n]), int(self.ft.n_children[n])
        return slice(fs, fs + A), A

    @staticmethod
    def matching(q, A):  # q [A, R] -> strategy [R, A]
        rp = np.maximum(q, 0).T
        s = rp.sum(axis=1, keepdims=True)
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(s > 0, rp / s, 1.0 / A)

    def set_strategies_from_predictions(self):
        for n in self.dec:
            rows, A = self._rows(n)
            self.t.strategy[n] = self.matching(self.pred[rows], A)
        self.t.update_reach()

    def half_iteration(self, p):
        t, ft = self.t, self.ft
        w = float(step_weight(self.gamma, self.iter_counter))
        t.compute_ev()
        mine = self.dec[ft.kind[self.dec] == p]
        for n in mine:
            rows, A = self._rows(n)
            fc = ft.first_child[n]
            d = t.ev[fc:fc + A, p] - t.ev[n, p][None, :]
            self.regret[rows] = np.maximum(d + self.regret[rows], 0.0)
            self.pred[rows] = np.maximum(self.regret[rows] + d, 0.0)
            t.strategy[n] = self.matching(self.pred[rows], A)
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
