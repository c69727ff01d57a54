"""ctypes driver of the two-card C oracle (oracle/cfr2_oracle.c, float64, OpenMP).  TEST INFRASTRUCTURE ONLY
(tests/, smoke(), bench.py's cpu_baseline / --impl reference legs).  Same interface as cfr2_numpy.Oracle2CFR."""
import ctypes as C
import os
import subprocess
from math import comb

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcfr2_oracle.so")
_lib = None
ALGOS = {"VanillaCFR": 0, "CFRPlus": 1, "LinearCFR": 2, "DCFR": 3, "PCFRPlus": 4}  # include/pokerrl_b200.h PRL_ALGO_*


class Orc2(C.Structure):
    _fields_ = [("n_nodes", C.c_int32), ("n_levels", C.c_int32), ("n_slots", C.c_int32), ("R", C.c_int32),
                ("n_deck", C.c_int32), ("n_boards", C.c_int32), ("n_sym", C.c_int32), ("pad", C.c_int32)] + \
               [(k, C.c_void_p) for k in ("level_start", "parent", "first_child", "n_children", "slot", "board", "kind",
                                          "acted_last", "pot", "hand_cards", "board_ranks", "board_blocked", "board_prob",
                                          "board_mult", "sym_perm", "board_order", "board_nlive")] + \
               [("K", C.c_double)] + [(k, C.c_void_p) for k in ("reach", "ev", "ev_br", "regret", "strat", "avg", "pred")] + \
               [(k, C.c_double) for k in ("fa", "fb", "fw")]


def build():
    subprocess.check_call(["make", "-s", "-C", _HERE])
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        tp = C.POINTER(Orc2)
        L.orc2_set_threads.argtypes = [C.c_int]
        L.orc2_prepare.argtypes = [tp]
        L.orc2_fill_uniform.argtypes = [tp]
        L.orc2_reach.argtypes = [tp, C.c_void_p]
        L.orc2_values.argtypes = [tp, C.c_void_p, C.c_int, C.c_int]
        L.orc2_values_levels.argtypes = [tp, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
        L.orc2_match.argtypes = [tp, C.c_void_p]
        L.orc2_regret_match.argtypes = [tp]
        L.orc2_exploitability.argtypes = [tp, C.c_void_p]
        L.orc2_regret_update.argtypes = [tp, C.c_int, C.c_int, C.c_int]
        L.orc2_avg_update.argtypes = [tp, C.c_int, C.c_int, C.c_int, C.c_int]
        L.orc2_average_strategy.argtypes = [tp, C.c_int, C.c_void_p]
        L.orc2_fold_row.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
        L.orc2_showdown_row.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                        C.c_double, C.c_void_p]
        for f in ("orc2_prepare", "orc2_fill_uniform", "orc2_reach", "orc2_values", "orc2_values_levels", "orc2_match",
                  "orc2_regret_match",
                  "orc2_exploitability",
                  "orc2_regret_update", "orc2_avg_update", "orc2_average_strategy", "orc2_fold_row", "orc2_showdown_row"):
            getattr(L, f).restype = None
        _lib = L
    return _lib


def set_factors(t, algo, it, dcfr_params=None, pcfr_gamma=2.0):
    """the factors of iteration counter `it` into the Orc2 struct t before a DCFR / PCFR+ update: the float32 row
    {a_t, b_t, w_t} of pokerrl_b200.dcfr.factors (PCFR+: of pcfr_params(gamma)), the numbers the kernels read"""
    if algo not in ("DCFR", "PCFRPlus"):
        return
    from pokerrl_b200 import dcfr
    params = (dcfr.DEFAULT if dcfr_params is None else dcfr_params) if algo == "DCFR" else dcfr.pcfr_params(pcfr_gamma)
    t.fa, t.fb, t.fw = (float(x) for x in dcfr.factors(*params, it + 1)[it])


def terminal_rows(hand_cards, ranks, reach, K, n_deck=52):
    """(showdown, fold) float64 rows of ONE board for an opponent reach row (unit pot, no folder sign)"""
    L = lib()
    R = len(ranks)
    hc = np.ascontiguousarray(hand_cards, np.int8)
    rk = np.ascontiguousarray(ranks, np.int32)
    ro = np.ascontiguousarray(reach, np.float64)
    live = np.nonzero(rk >= 0)[0]
    order = np.ascontiguousarray(live[np.lexsort((live, rk[live]))], np.int32)
    blocked = np.ascontiguousarray(rk < 0, np.uint8)
    sd, fo = np.zeros(R), np.zeros(R)
    L.orc2_showdown_row(R, n_deck, hc.ctypes.data, rk.ctypes.data, order.ctypes.data, len(order), ro.ctypes.data, K,
                        sd.ctypes.data)
    L.orc2_fold_row(R, n_deck, hc.ctypes.data, blocked.ctypes.data, ro.ctypes.data, K, fo.ctypes.data)
    return sd, fo


class Oracle2CSolver:
    """ft: FlatTree of a two-card game; board_ranks int32 [n_boards_total, R] in global board id order (-1 = blocked)."""

    def __init__(self, ft, board_ranks, algo="CFRPlus", delay=0, ev_normalizer=None, n_threads=None, lean=False,
                 dcfr_params=None, pcfr_gamma=2.0):
        self.ft, self.algo_name, self.algo = ft, algo, ALGOS[algo]
        self.delay = delay if algo == "CFRPlus" else 0
        self.dcfr_params, self.pcfr_gamma = dcfr_params, pcfr_gamma
        self.lean = bool(lean)  # True: value passes compute only what the half-iteration needs (the GPU's schedule)
        self.ev_normalizer = ft.game_cls.EV_NORMALIZER if ev_normalizer is None else ev_normalizer
        L = self.L = lib()
        self.n_threads = L.orc2_set_threads(int(n_threads or 0))
        rules = ft.rules
        R, N, S = ft.R, ft.n_nodes, ft.n_slots
        self.R = R
        lut = rules.get_lut_holder()
        hc = np.ascontiguousarray(lut.LUT_IDX_2_HOLE_CARDS, np.int8)
        bc = ft.board_cards()
        nb = bc.shape[0]
        blocked = np.zeros((nb, R), np.uint8)
        for k in range(bc.shape[1]):
            col = bc[:, k]
            blocked |= ((hc[None, :, 0] == col[:, None]) | (hc[None, :, 1] == col[:, None])) & (col[:, None] >= 0)
        sp = ft.board_spec.sym_perm
        self._a = dict(
            level_start=np.ascontiguousarray(ft.level_start, np.int64), parent=ft.parent.astype(np.int32),
            first_child=ft.first_child.astype(np.int32), n_children=ft.n_children.astype(np.int32),
            slot=ft.slot.astype(np.int32), board=ft.board.astype(np.int32), kind=ft.kind.astype(np.int8),
            acted_last=ft.acted_last.astype(np.int8), pot=ft.pot.astype(np.float64), hand_cards=hc,
            board_ranks=np.ascontiguousarray(board_ranks, np.int32), board_blocked=blocked,
            board_prob=ft.board_prob.astype(np.float64), board_mult=ft.board_mult.astype(np.float64),
            sym_perm=None if sp is None else np.ascontiguousarray(sp, np.int16),
            board_order=np.zeros((nb, R), np.int32), board_nlive=np.zeros(nb, np.int32))
        self.reach, self.ev, self.ev_br = (np.zeros((N, 2, R)) for _ in range(3))
        self.regret, self.strat, self.avg = (np.zeros((S, R)) for _ in range(3))
        self._avg_norm = np.zeros((S, R))
        # PCFR+: the predictions; the strategy is regret matching of these rows
        self.pred = np.zeros((S, R)) if algo == "PCFRPlus" else None
        t = Orc2()
        t.n_nodes, t.n_levels, t.n_slots, t.R = N, ft.n_levels, S, R
        t.n_deck, t.n_boards, t.n_sym = rules.N_CARDS_IN_DECK, nb, 0 if sp is None else sp.shape[0]
        for k, a in self._a.items():
            setattr(t, k, None if a is None else a.ctypes.data)
        n_hole = rules.N_HOLE_CARDS
        t.K = comb(t.n_deck, n_hole) / comb(t.n_deck - n_hole, n_hole)
        for k in ("reach", "ev", "ev_br", "regret", "strat", "avg"):
            setattr(t, k, getattr(self, k).ctypes.data)
        t.pred = None if self.pred is None else self.pred.ctypes.data
        self.t = t
        L.orc2_prepare(C.byref(t))
        self.reset()

    def reset(self):
        self.iter_counter = 0
        for a in (self.regret, self.strat, self.avg) + (() if self.pred is None else (self.pred,)):
            a[:] = 0
        self.L.orc2_fill_uniform(C.byref(self.t))
        self.L.orc2_reach(C.byref(self.t), self.strat.ctypes.data)

    def match(self):
        """strategy = regret matching of the regret rows (PCFR+: of the predictions), reach refreshed: after the caller
        set the tables"""
        self.L.orc2_regret_match(C.byref(self.t))
        self.L.orc2_reach(C.byref(self.t), self.strat.ctypes.data)

    def compute_ev(self, mask=3, with_br=True):
        self.L.orc2_values(C.byref(self.t), self.strat.ctypes.data, mask, int(with_br))
        out = np.zeros(2)
        self.L.orc2_exploitability(C.byref(self.t), out.ctypes.data)
        return out

    def half_iteration(self, p):
        """seat p's part of an iteration (_CFRBase.py:123-128); the caller advances iter_counter after seat 1"""
        t = C.byref(self.t)
        if self.lean:
            self.L.orc2_values(t, self.strat.ctypes.data, 1 << p, 0)
        else:
            self.L.orc2_values(t, self.strat.ctypes.data, 3, 1)
        set_factors(self.t, self.algo_name, self.iter_counter, self.dcfr_params, self.pcfr_gamma)
        self.L.orc2_regret_update(t, p, self.algo, self.iter_counter)
        self.L.orc2_reach(t, self.strat.ctypes.data)
        self.L.orc2_avg_update(t, p, self.algo, self.iter_counter, self.delay)

    def iteration(self, n=1):
        for _ in range(n):
            for p in (0, 1):  # _CFRBase.py:122-134
                self.half_iteration(p)
            self.iter_counter += 1

    def _metric(self, expl):
        return float(sum(expl[p] * self.ev_normalizer for p in range(2)) / 2)

    def exploitability_current(self):
        """of the current strategy: regret matching of the regrets (PCFR+: of the predictions), as the updates leave it"""
        return self._metric(self.compute_ev())

    def exploitability_average(self):
        t = C.byref(self.t)
        self.L.orc2_average_strategy(t, self.algo, self._avg_norm.ctypes.data)
        self.L.orc2_reach(t, self._avg_norm.ctypes.data)
        self.L.orc2_values(t, self._avg_norm.ctypes.data, 3, 1)
        out = np.zeros(2)
        self.L.orc2_exploitability(t, out.ctypes.data)
        self.L.orc2_reach(t, self.strat.ctypes.data)
        return self._metric(out)
