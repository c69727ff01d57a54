"""The restricted Nash response restated in float64 on oracle/cfr2_numpy.Oracle2Tree, for the parity tests.

Exploiter seat s, opponent seat o = 1 - s: a fixed model (probability p) or a free strategy (1 - p).  Both learn by CFR+
(the rules of oracle/cfr2_numpy.Oracle2CFR).  Seat s's counterfactual values are linear in the opponent's reach, so they are
p * (values against the model) + (1 - p) * (values against the free copy), each from one Oracle2Tree pass; the free copy's
update is plain CFR+ against the exploiter (its true values are 1 - p times those, which leaves regret matching as it is)."""
import numpy as np


class Oracle2RNR:
    """regret / avg = float64 [n_slots, R]: seat s's rows are the exploiter's, seat o's the free copy's; the strategies are
    regret matching of `regret`.  model = float64 [n_slots, R], read at seat o's nodes."""

    def __init__(self, tree, seat, p, model, delay=0):
        self.t, self.seat, self.p, self.delay = tree, int(seat), float(p), int(delay)
        ft = self.ft = tree.ft
        self.R = tree.R
        self.model = np.asarray(model, np.float64)
        self.dec = np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]
        self.regret = np.zeros((ft.n_slots, self.R))
        self.avg = np.zeros((ft.n_slots, self.R))
        self.iter_counter = 0

    def _rows(self, n):
        fs, A = int(self.ft.first_slot[n]), int(self.ft.n_children[n])
        return slice(fs, fs + A), A

    @staticmethod
    def matching(reg, A):  # [A, R] -> [R, A]
        rp = np.maximum(reg, 0).T
        s = rp.sum(axis=1, keepdims=True)
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(s > 0, rp / s, 1.0 / A)

    def _play(self, own, opp):
        """values / reach of the tree with seat s playing `own` and seat o playing `opp` ("current", "avg", "model")"""
        t, ft = self.t, self.ft
        for n in self.dec:
            rows, A = self._rows(n)
            which = own if ft.kind[n] == self.seat else opp
            if which == "model":
                t.strategy[n] = self.model[rows].T.copy()
            elif which == "avg":
                t.strategy[n] = self.avg[rows].T.copy()
            else:
                t.strategy[n] = self.matching(self.regret[rows], A)
        t.update_reach()
        t.compute_ev()
        return t.ev.copy(), t.ev_br.copy(), t.reach.copy()

    def values(self, q):
        """float64 [n_nodes, R]: the counterfactual values of seat q's update"""
        ev_free = self._play("current", "current")[0][:, q]
        if q != self.seat:
            return ev_free
        ev_model = self._play("current", "model")[0][:, q]
        return self.p * ev_model + (1.0 - self.p) * ev_free

    def half_iteration(self, q):
        """seat q's CFR+ update at this iteration counter (the counter does not advance)"""
        ft, i, d0 = self.ft, self.iter_counter, self.delay
        v = self.values(q)
        for n in self.dec[ft.kind[self.dec] == q]:
            rows, A = self._rows(n)
            fc = ft.first_child[n]
            self.regret[rows] = np.maximum(v[fc:fc + A] - v[n][None, :] + self.regret[rows], 0.0)
            self._avg_step(rows, self.matching(self.regret[rows], A).T, i)

    def _avg_step(self, rows, s, i):
        """CFR+'s averaging step of iteration counter i (CFRPlus.py:65-87)"""
        d0 = self.delay
        if i > d0:
            cw = sum(range(d0 + 1, i + 1))
            nw = i - d0 + 1
            self.avg[rows] = cw / (cw + nw) * self.avg[rows] + nw / (cw + nw) * s
        elif i == d0:
            self.avg[rows] = s

    def pending_step(self, q, due):
        """seat q's averaging step of iteration `due` from the regrets as they are, at its post-deal nodes: the step the board
        engine's paired form applies before its own (the trunk averages in its own launch, nothing is pending there)"""
        for n in self.dec[(self.ft.kind[self.dec] == q) & (self.ft.cdepth[self.dec] > 0)]:
            rows, A = self._rows(n)
            self._avg_step(rows, self.matching(self.regret[rows], A).T, due)

    def iteration(self):
        for q in (0, 1):
            if q != self.seat and self.p == 1.0:
                continue
            self.half_iteration(q)
        self.iter_counter += 1

    def exploitation_exploitability(self, source="avg"):
        """chips: the value of seat s's strategy `source` against the model, and of a best response of seat o to it"""
        ev, _, reach = self._play(source, "model")
        s, o = self.seat, 1 - self.seat
        exploitation = float((ev[0, s] * reach[0, s]).sum())
        _, ev_br, reach = self._play(source, "current")
        return exploitation, float((ev_br[0, o] * reach[0, o]).sum())


class TableAgent:
    """an agent that answers from a natural-order table [n_slots, R] of the flat tree `ft` (queried on trees over the same
    boards, whose slot order is that of `ft`)"""

    def __init__(self, ft, table, n_actions):
        self.ft, self.table, self.n_actions = ft, np.asarray(table, np.float32), n_actions

    def get_a_probs_for_public_tree(self, tree):
        import torch
        ft = tree.flat
        assert ft.n_slots == self.ft.n_slots and np.array_equal(ft.board_spec.boards, self.ft.board_spec.boards)
        dec = np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]
        out = np.zeros((dec.size, ft.R, self.n_actions), np.float32)
        for d, n in enumerate(dec):
            fs, fc, A = int(ft.first_slot[n]), int(ft.first_child[n]), int(ft.n_children[n])
            out[d][:, ft.action[fc:fc + A]] = self.table[fs:fs + A].T
        return torch.from_numpy(out).to(tree.dtree.device)


def random_model(ft, seed, skew=3.0):
    """a random strategy of every decision node of `ft`, float32 rows summing to one (float64 of those values returned)"""
    rng = np.random.default_rng(seed)
    m = np.zeros((ft.n_slots, ft.R))
    for n in np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]:
        fs, A = int(ft.first_slot[n]), int(ft.n_children[n])
        x = rng.uniform(0.0, 1.0, (A, ft.R)) ** skew + 1e-3
        m[fs:fs + A] = x / x.sum(axis=0, keepdims=True)
    return m.astype(np.float32).astype(np.float64)
