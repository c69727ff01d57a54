"""ctypes driver of the C oracle (oracle/cfr_oracle.c).  TEST INFRASTRUCTURE ONLY (tests/, smoke(), bench.py's
cpu_baseline / --impl reference legs).  Mirrors pokerrl_b200.solver.CFRSolver with numpy host buffers."""
import ctypes as C
import os
import subprocess

import numpy as np

from pokerrl_b200 import _native as nat  # struct layouts + enums of include/pokerrl_b200.h only

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libcfr_oracle.so")
_lib = None


def build():
    subprocess.check_call(["make", "-s", "-C", _HERE])
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        L = C.CDLL(_LIB_PATH)
        tp, bp, ip = C.POINTER(nat.PrlTree), C.POINTER(nat.PrlBuffers), C.POINTER(C.c_int)
        L.orc_reach_pass.argtypes = [tp, bp, C.c_int, ip]
        L.orc_value_pass.argtypes = [tp, bp, C.c_int, C.c_int, ip]
        L.orc_root_exploitability.argtypes = [tp, bp, C.c_void_p]
        L.orc_cfr_half_iteration.argtypes = [tp, bp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, ip]
        L.orc_pairwise_sum.argtypes = [C.c_void_p, C.c_int]
        L.orc_pairwise_sum.restype = C.c_float
        _lib = L
    return _lib


ALGOS = {"VanillaCFR": nat.ALGO_VANILLA, "CFRPlus": nat.ALGO_CFR_PLUS, "LinearCFR": nat.ALGO_LINEAR}


class OracleCSolver:
    def __init__(self, ft, algo="CFRPlus", delay=0, avg_f64=True, n_threads=None):
        self.ft, self.algo, self.delay = ft, ALGOS[algo], (delay if algo == "CFRPlus" else 0)
        self.avg_f64 = bool(avg_f64) and algo == "CFRPlus"
        self.L = lib()
        self.n_threads = self.L.orc_set_threads(int(n_threads or 0))
        R = ft.R
        self.R = self.ld = R
        rules = ft.rules
        assert rules.N_HOLE_CARDS == 1
        bc = ft.node_board_cards()[:, 0].astype(np.int32)
        self._arrs = dict(
            level_start=np.ascontiguousarray(ft.level_start, np.int64),
            parent=ft.parent.astype(np.int32), first_child=ft.first_child.astype(np.int32),
            n_children=ft.n_children.astype(np.int32), slot=ft.slot.astype(np.int32),
            kind=ft.kind.astype(np.int8), acted_last=ft.acted_last.astype(np.int8),
            pot=ft.pot.astype(np.float32), board=np.where(bc >= 0, bc, -1).astype(np.int32))
        t = nat.PrlTree()
        t.n_nodes, t.n_levels, t.n_slots, t.n_range, t.ld = ft.n_nodes, ft.n_levels, ft.n_slots, R, R
        t.n_hole, t.n_deck, t.n_suits = 1, rules.N_CARDS_IN_DECK, rules.N_SUITS
        t.pair_bonus, t.max_actions = rules.PAIR_BONUS or 0, ft.max_actions
        for k, a in self._arrs.items():
            setattr(t, k, a.ctypes.data)
        self.tree = t
        N, S = ft.n_nodes, ft.n_slots
        self.reach, self.ev, self.ev_br = (np.zeros((2, N, R), np.float32) for _ in range(3))
        self.reach_eval = np.zeros((2, N, R), np.float32)
        self.regret, self.strat = np.zeros((S, R), np.float32), np.zeros((S, R), np.float32)
        self.avg = np.zeros((S, R), np.float64 if self.avg_f64 else np.float32)
        self.bufs = self._bufs(self.reach)
        self.bufs_eval = self._bufs(self.reach_eval)
        self.ev_normalizer = ft.game_cls.EV_NORMALIZER
        self.reset()

    def _bufs(self, reach):
        b = nat.PrlBuffers()
        b.reach, b.ev, b.ev_br = reach.ctypes.data, self.ev.ctypes.data, self.ev_br.ctypes.data
        b.regret, b.strat, b.avg = self.regret.ctypes.data, self.strat.ctypes.data, self.avg.ctypes.data
        return b

    def reset(self):
        self.iter_counter = 0
        self.regret[:] = 0
        self.strat[:] = 0
        self.avg[:] = 0
        self.modes = [nat.STRAT_UNIFORM64, nat.STRAT_UNIFORM64]
        self.L.orc_reach_pass(C.byref(self.tree), C.byref(self.bufs), 3, nat.modes(*self.modes))

    def iteration(self, n=1):
        for _ in range(n):
            for p in (0, 1):
                self.L.orc_cfr_half_iteration(C.byref(self.tree), C.byref(self.bufs), self.algo, p,
                                              self.iter_counter, self.delay, int(self.avg_f64),
                                              nat.modes(*self.modes))
                self.modes[p] = nat.STRAT_F32
            self.iter_counter += 1

    def _metric(self, bufs):
        out = np.zeros(2, np.float32)
        self.L.orc_root_exploitability(C.byref(self.tree), C.byref(bufs), out.ctypes.data)
        return sum(float(out[p]) * self.ev_normalizer for p in range(2)) / 2

    def exploitability_current(self):
        self.L.orc_value_pass(C.byref(self.tree), C.byref(self.bufs), 3, 1, nat.modes(*self.modes))
        return self._metric(self.bufs)

    def average_modes(self):
        if self.algo != nat.ALGO_CFR_PLUS:
            return [nat.STRAT_AVG_SUM] * 2
        if self.iter_counter == self.delay + 1:
            return [nat.STRAT_F32] * 2
        return [nat.STRAT_AVG_F64 if self.avg_f64 else nat.STRAT_AVG_F32] * 2

    def exploitability_average(self):
        m = nat.modes(*self.average_modes())
        self.L.orc_reach_pass(C.byref(self.tree), C.byref(self.bufs_eval), 3, m)
        self.L.orc_value_pass(C.byref(self.tree), C.byref(self.bufs_eval), 3, 1, m)
        return self._metric(self.bufs_eval)
