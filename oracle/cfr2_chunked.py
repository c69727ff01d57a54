"""Float64 results of a two-card game with ONE chance layer, computed a chunk of boards at a time (oracle/cfr2_oracle.c).
TEST INFRASTRUCTURE ONLY (tests/test_oracle_cfr2_chunked.py, tests/test_gpu_board_full_game.py,
tests/test_gpu_board_full_game_dcfr_pcfr.py).

The full Flop5Holdem game (134 459 board classes) does not fit the monolithic oracle: each of its float64 node vectors would
take ~45 GB.  But everything below the chance node is per board, and the chance node's row is linear in its children
(sum of mult_b * child_b, then the sum over the suit permutations; the deal probability sits in the reach).  So:
  1. every chunk is a `BoardSpec` slice that keeps the game's board_prob, board_mult and sym_perm (NOT renormalised): the
     sum of the chunks' chance-node rows is the game's chance-node row;
  2. the summed rows are set into a one-board tree of the same game, and only the levels above the chance node are swept
     (`orc2_values_levels`, keep_chance): values, best response and exploitability of the trunk; for an update, the regrets,
     matching, average and reach of the updating seat's trunk nodes;
  3. for an update, every chunk is swept again with the updated trunk rows in place: its post-update board rows go to a
     callback, so nothing full-size is ever held.

`SyntheticProfile` is the deterministic input both sides load: regrets and average rows (PCFR+: and predictions) from an
integer hash of (board class, local node, hand), in float32 values that are exact in float64."""
import ctypes as C

import numpy as np

import cfr2_c
from pokerrl_b200.game.holdem_boards import BoardSpec

_M32 = 0xFFFFFFFF
_TRUNK_KEY = 0x7FFFFFFF
_PRED_SALT = 0x5BD1E995


def _mix(x):
    """32-bit integer finaliser on non-negative int64 tensors (every product stays below 2^63: same bits on any device)"""
    x = (((x >> 16) ^ x) * 0x45D9F3B) & _M32
    x = (((x >> 16) ^ x) * 0x45D9F3B) & _M32
    return (x >> 16) ^ x


def decision_rows(st):
    """local child nodes that own a table row (children of decision nodes), ascending: the board engine's `local_rows` order"""
    return [c for d in range(st["n_local"]) if st["kind"][d] <= 1
            for c in range(st["first_child"][d], st["first_child"][d] + st["n_children"][d])]


def board_slots(ft, rows):
    """int64 [n_boards, len(rows)]: table slot of local node rows[k] on board j of the flat tree ft"""
    st = ft.board_subtree()
    nb = ft.board_spec.boards.shape[0]
    j = np.arange(nb, dtype=np.int64)[:, None]
    s0 = np.array([int(ft.slot[st["node_base"][c] + st["node_k"][c]]) for c in rows], np.int64)
    m = np.array([st["node_m"][c] for c in rows], np.int64)
    return s0[None, :] + j * m[None, :]


def n_trunk_slots(ft):
    st = ft.board_subtree()
    return int((ft.slot[:st["chance_node"] + 1] >= 0).sum())


class SyntheticProfile:
    """Regret and average rows of a late run, without running one.  Per entry a hash picks an exact zero (1/8), a negative
    (1/4) or a positive regret of 1 .. 2^20 units; per (decision node, hand) a second hash makes 1/8 of the hands all <= 0
    (regret matching falls back to uniform) and 1/8 pure (one positive action).  The average rows are integer weights
    0 .. 255 (1/8 zero) normalised per hand (uniform where all are 0).  Units: regret 2^(regret_exp - 20), average
    2^avg_exp (CFR+: 0, a strategy; Vanilla / Linear CFR, DCFR, PCFR+: reach-weighted sums of the size of one iteration's
    contribution), each as (trunk, board) exponents, so that one update's increment is not lost in the inputs.
    pcfr=True (PCFR+): the regrets are clipped at 0, and prediction rows come from a third hash of the same keys by the
    regrets' construction, clipped at 0 (exact zeros, all-zero hands whose matching is uniform, pure hands), in the regrets'
    units; the row methods then return (regret, avg, pred)."""

    def __init__(self, ft, seed=1, regret_exp=(0, 0), avg_exp=(0, 0), pcfr=False):
        st = ft.board_subtree()
        self.R = ft.R
        self.seed = int(seed) & _M32
        self.regret_exp, self.avg_exp, self.pcfr = regret_exp, avg_exp, bool(pcfr)
        self.rows = decision_rows(st)
        par = [st["parent"][c] for c in self.rows]
        self._board = self._meta(self.rows, par, [c - st["first_child"][p] for c, p in zip(self.rows, par)],
                                 [st["n_children"][p] for p in par])
        nts = n_trunk_slots(ft)
        node_of = {int(ft.slot[n]): n for n in range(st["chance_node"] + 1) if ft.slot[n] >= 0}
        tn = [node_of[s] for s in range(nts)]
        tp = [int(ft.parent[n]) for n in tn]
        self._trunk = self._meta(list(range(nts)), tp, [n - int(ft.first_child[p]) for n, p in zip(tn, tp)],
                                 [int(ft.n_children[p]) for p in tp])
        self.n_trunk_slots = nts

    @staticmethod
    def _meta(node, parent, action, n_act):
        groups = {p: i for i, p in enumerate(dict.fromkeys(parent))}
        return dict(node=np.array(node, np.int64), parent=np.array(parent, np.int64), action=np.array(action, np.int64),
                    n_act=np.array(n_act, np.int64), group=np.array([groups[p] for p in parent], np.int64),
                    n_groups=len(groups))

    @staticmethod
    def _signed(e, g, meta, t):
        """integer regrets (units) from the entry hashes e and the (decision node, hand) hashes g"""
        import torch
        mag = (e & 0xFFFFF) + 1
        sel = (e >> 20) & 15
        val = torch.where(sel < 2, torch.zeros_like(mag), torch.where(sel < 6, -mag, mag))
        mode = g & 7
        chosen = ((g >> 3) % t(meta["n_act"])[None, :, None]) == t(meta["action"])[None, :, None]
        val = torch.where(mode == 0, -val.abs(), val)
        return torch.where(mode == 1, torch.where(chosen, mag, -val.abs()), val)

    def _rows(self, keys, meta, part, device):
        import torch
        t = lambda a: torch.as_tensor(a, dtype=torch.int64, device=device)  # noqa: E731
        kc = _mix(t(keys) ^ self.seed)[:, None]                                          # [n, 1]
        ke = _mix(kc ^ ((t(meta["node"]) * 0x9E3779B1) & _M32)[None, :])[..., None]      # [n, rows, 1]
        kg = _mix(kc ^ (((t(meta["parent"]) + 32) * 0x9E3779B1) & _M32)[None, :])[..., None]
        h = torch.arange(self.R, dtype=torch.int64, device=device)[None, None, :]
        e, g = _mix(ke ^ h), _mix(kg ^ h)
        val = self._signed(e, g, meta, t)
        if self.pcfr:
            val = val.clamp(min=0)
        unit = 2.0 ** (self.regret_exp[part] - 20)
        regret = (val.to(torch.float64) * unit).to(torch.float32)
        z = (e >> 24) & 0xFF
        w = torch.where(z < 32, torch.zeros_like(z), z).to(torch.float64)
        gid = t(meta["group"])
        tot = torch.zeros(w.shape[0], meta["n_groups"], w.shape[2], dtype=torch.float64, device=device).index_add_(1, gid, w)
        tot = tot[:, gid]
        avg = torch.where(tot > 0, w / torch.where(tot > 0, tot, torch.ones_like(tot)), 1.0 / t(meta["n_act"])[None, :, None])
        avg = (avg.to(torch.float32).to(torch.float64) * 2.0 ** self.avg_exp[part]).to(torch.float32)
        if not self.pcfr:
            return regret, avg
        e3, g3 = _mix(_mix(ke ^ _PRED_SALT) ^ h), _mix(_mix(kg ^ _PRED_SALT) ^ h)
        pred = (self._signed(e3, g3, meta, t).clamp(min=0).to(torch.float64) * unit).to(torch.float32)
        return regret, avg, pred

    def board_rows(self, classes, device="cpu"):
        """(regret, avg[, pred]) float32 [len(classes), len(self.rows), R] of the given global board classes"""
        return self._rows(np.asarray(classes, np.int64), self._board, 1, device)

    def trunk_rows(self, device="cpu"):
        """(regret, avg[, pred]) float32 [n_trunk_slots, R]"""
        return tuple(x[0] for x in self._rows(np.array([_TRUNK_KEY], np.int64), self._trunk, 0, device))

    def tables(self, ft, first_class, device="cpu"):
        """(regret, avg[, pred]) float64 [ft.n_slots, R] over a flat tree whose boards are the classes first_class,
        first_class + 1, ... (device: where the hash runs; integer arithmetic, so any device gives the same bits)"""
        nb = ft.board_spec.boards.shape[0]
        out = []
        tr, br = self.trunk_rows(device), self.board_rows(np.arange(first_class, first_class + nb), device)
        slots = board_slots(ft, self.rows)
        for k in range(len(tr)):
            tab = np.zeros((ft.n_slots, self.R))
            tab[:self.n_trunk_slots] = tr[k].cpu().numpy()
            tab[slots.ravel()] = br[k].cpu().numpy().reshape(-1, self.R)
            out.append(tab)
        return out


def spec_slice(spec, lo, hi):
    """boards lo .. hi-1 of `spec` with the game's own deal probabilities, multiplicities and suit permutations"""
    return BoardSpec(spec.boards[lo:hi], spec.board_prob[lo:hi], spec.board_mult[lo:hi], spec.sym_perm,
                     "%s [%d:%d]" % (spec.note, lo, hi))


class ChunkedOracle:
    """tree_fn(BoardSpec) -> FlatTree of the game; ranks: int32 [n_boards, R] of spec.boards (-1: the hand holds a board
    card); tables(ft, first_class, key) -> (regret, avg) float64 [ft.n_slots, R] for the chunk tree ft of the classes
    first_class, ..., and (regret, avg, pred) for a PCFR+ key (`key` names one set of tables; runs that share one
    computation of values must share the strategy: the regrets, or PCFR+'s predictions).  dcfr_params / pcfr_gamma: the
    factors of DCFR / PCFR+ runs (pokerrl_b200.dcfr)."""

    def __init__(self, tree_fn, spec, ranks, tables, chunk=2048, n_threads=None, dcfr_params=None, pcfr_gamma=2.0):
        self.tree_fn, self.spec, self.ranks, self.tables, self.chunk = tree_fn, spec, ranks, tables, int(chunk)
        self.n_threads = n_threads
        self.dcfr_params, self.pcfr_gamma = dcfr_params, pcfr_gamma
        self.n_boards = spec.boards.shape[0]
        self.L = cfr2_c.lib()
        self.trunk_ft = tree_fn(spec_slice(spec, 0, 1))
        st = self.trunk_ft.board_subtree()
        self.chance_node, self.chance_level = st["chance_node"], st["chance_level"]
        self.nts = n_trunk_slots(self.trunk_ft)
        self.n_trunk_nodes = self.chance_node + 1
        sp = spec.sym_perm
        self.perms = np.arange(self.trunk_ft.R)[None] if sp is None else np.asarray(sp, np.int64)

    def _solver(self, ft, lo, algo="CFRPlus", delay=0):
        nb = ft.board_spec.boards.shape[0]
        rk = np.full((nb + 1, ft.R), -1, np.int32)  # global board 0 is the empty pre-deal board
        rk[1:] = self.ranks[lo:lo + nb]
        return cfr2_c.Oracle2CSolver(ft, rk, algo, delay=delay, n_threads=self.n_threads, lean=True,
                                     dcfr_params=self.dcfr_params, pcfr_gamma=self.pcfr_gamma)

    def chunks(self):
        for lo in range(0, self.n_boards, self.chunk):
            hi = min(lo + self.chunk, self.n_boards)
            yield lo, hi, self.tree_fn(spec_slice(self.spec, lo, hi))

    def _set(self, o, ft, lo, key):
        """the tables of `key` into solver o; strategy = regret matching of the regrets (PCFR+ solver: of the predictions)"""
        tabs = self.tables(ft, lo, key)
        o.regret[:], o.avg[:] = tabs[:2]
        if o.pred is not None:
            o.pred[:] = tabs[2]
        self.L.orc2_regret_match(C.byref(o.t))

    def _factors(self, o, algo, it):
        cfr2_c.set_factors(o.t, algo, it, self.dcfr_params, self.pcfr_gamma)

    # ------------------------------------------------------------------------------------------------ evaluation
    def evaluate(self, key, algo="CFRPlus", forms=("current", "average")):
        """Both seats' ev / ev_br at the chance node, and the exploitability, of the current strategy (regret matching of
        the regrets; PCFR+: of the predictions) and of the average strategy (CFR+: the average rows; the others: the
        normalised sums).
        Also abs_ev / abs_br: sum over the suit permutations s and boards b of |mult_b v_b[perm_s(h)]| (error bounds)."""
        R = self.trunk_ft.R
        acc = {f: {k: np.zeros((2, R)) for k in ("ev", "ev_br", "abs_ev", "abs_br")} for f in forms}
        ch = self.chance_node
        for lo, hi, ft in self.chunks():
            o = self._solver(ft, lo, algo)
            self._set(o, ft, lo, key)
            kids = np.arange(ft.first_child[ch], ft.first_child[ch] + ft.n_children[ch])
            mult = np.asarray(ft.board_mult, np.float64)[ft.board[kids]][:, None, None]
            for form in forms:
                s = o.strat
                if form == "average":
                    self.L.orc2_average_strategy(C.byref(o.t), o.algo, o._avg_norm.ctypes.data)
                    s = o._avg_norm
                self.L.orc2_reach(C.byref(o.t), s.ctypes.data)
                self.L.orc2_values(C.byref(o.t), s.ctypes.data, 3, 1)
                a = acc[form]
                a["ev"] += o.ev[ch]
                a["ev_br"] += o.ev_br[ch]
                a["abs_ev"] += (mult * np.abs(o.ev[kids])).sum(axis=0)
                a["abs_br"] += (mult * np.abs(o.ev_br[kids])).sum(axis=0)
            del o
        t = self._trunk_solver(key, algo)
        out = {}
        for form in forms:
            a = acc[form]
            for k in ("abs_ev", "abs_br"):
                a[k] = a[k][:, self.perms].sum(axis=1)
            s = t.strat
            if form == "average":
                self.L.orc2_average_strategy(C.byref(t.t), t.algo, t._avg_norm.ctypes.data)
                s = t._avg_norm
            self.L.orc2_reach(C.byref(t.t), s.ctypes.data)
            t.ev[ch], t.ev_br[ch] = a["ev"], a["ev_br"]
            self.L.orc2_values_levels(C.byref(t.t), s.ctypes.data, 3, 1, self.chance_level, 1)
            e = np.zeros(2)
            self.L.orc2_exploitability(C.byref(t.t), e.ctypes.data)
            nt = self.n_trunk_nodes
            out[form] = dict(a, expl=t._metric(e), expl_seat=e, reach=t.reach[:nt].copy(), trunk_ev=t.ev[:nt].copy(),
                             trunk_br=t.ev_br[:nt].copy())
        return out

    def _trunk_solver(self, key, algo, delay=0):
        t = self._solver(self.trunk_ft, 0, algo, delay)
        self._set(t, self.trunk_ft, 0, key)
        return t

    # ------------------------------------------------------------------------------------------------ half-iteration
    def half_iterations(self, p, runs, on_chunk, chance_ev=None, pending=False):
        """Seat p's half-iteration (_CFRBase.py:123-128) from the given tables, for every run (key, algo, iteration, delay).
        The runs share one value sweep per chunk, so they must share the strategy: the regrets (CFR+, Vanilla / Linear CFR
        and DCFR runs together), or the predictions (PCFR+ runs only).  on_chunk(lo, hi, ft, run index, regret, avg[,
        pred]) receives each chunk's post-update tables (float64 [ft.n_slots, R]; the trunk rows are the game's; pred for
        PCFR+).  chance_ev: seat p's chance-node row under the given strategy if known (evaluate()['current']['ev'][p]),
        else one more pass.  pending (p = 1, averages kept as sums): seat 0's average contribution of the same iteration
        is added to the post-deal rows first, under the given profile (the deferred form of the board engine, whose trunk
        rows already hold it: the trunk's are left alone).
        Returns per run the updated trunk rows: dict(regret, strat, avg[, pred] [n_trunk_slots, R], reach [n_trunk_nodes,
        2, R])."""
        ch, nts = self.chance_node, self.nts
        key0, algo0 = runs[0][0], runs[0][1]
        pcfr = algo0 == "PCFRPlus"
        if any((algo == "PCFRPlus") != pcfr for _, algo, _, _ in runs):
            raise ValueError("PCFR+ runs (strategies from the predictions) need a pass of their own")
        if pending and (p != 1 or any(algo == "CFRPlus" for _, algo, _, _ in runs)):
            raise ValueError("pending: seat 0's contribution to sums, before seat 1's update")
        if chance_ev is None:
            chance_ev = np.zeros(self.trunk_ft.R)
            for lo, hi, ft in self.chunks():
                o = self._solver(ft, lo, algo0)
                self._set(o, ft, lo, key0)
                self.L.orc2_reach(C.byref(o.t), o.strat.ctypes.data)
                self.L.orc2_values(C.byref(o.t), o.strat.ctypes.data, 1 << p, 0)
                chance_ev += o.ev[ch, p]
                del o
        trunk = []
        for key, algo, it, delay in runs:
            t = self._trunk_solver(key, algo, delay)
            tt = C.byref(t.t)
            self.L.orc2_reach(tt, t.strat.ctypes.data)
            t.ev[ch, p] = chance_ev
            self.L.orc2_values_levels(tt, t.strat.ctypes.data, 1 << p, 0, self.chance_level, 1)
            self._factors(t, algo, it)
            self.L.orc2_regret_update(tt, p, cfr2_c.ALGOS[algo], it)
            self.L.orc2_reach(tt, t.strat.ctypes.data)
            self.L.orc2_avg_update(tt, p, cfr2_c.ALGOS[algo], it, t.delay)
            trunk.append(dict(regret=t.regret[:nts].copy(), strat=t.strat[:nts].copy(), avg=t.avg[:nts].copy(),
                              reach=t.reach[:self.n_trunk_nodes].copy(), **({"pred": t.pred[:nts].copy()} if pcfr else {})))
            del t
        for lo, hi, ft in self.chunks():
            o = self._solver(ft, lo, algo0)
            tt = C.byref(o.t)
            for k, (key, algo, it, delay) in enumerate(runs):
                self._set(o, ft, lo, key)
                self._factors(o, algo, it)
                if k == 0:
                    self.L.orc2_reach(tt, o.strat.ctypes.data)
                    self.L.orc2_values(tt, o.strat.ctypes.data, 1 << p, 0)
                if pending:  # seat 0's contribution under the given profile; its trunk rows are replaced below
                    self.L.orc2_reach(tt, o.strat.ctypes.data)
                    self.L.orc2_avg_update(tt, 0, cfr2_c.ALGOS[algo], it, 0)
                self.L.orc2_regret_update(tt, p, cfr2_c.ALGOS[algo], it)
                # the chunk's trunk rows above came from its own share of the chance node: the game's go in their place
                o.regret[:nts], o.strat[:nts] = trunk[k]["regret"], trunk[k]["strat"]
                if pcfr:
                    o.pred[:nts] = trunk[k]["pred"]
                self.L.orc2_reach(tt, o.strat.ctypes.data)
                self.L.orc2_avg_update(tt, p, cfr2_c.ALGOS[algo], it, delay if algo == "CFRPlus" else 0)
                o.avg[:nts] = trunk[k]["avg"]
                on_chunk(lo, hi, ft, k, o.regret, o.avg, *((o.pred,) if pcfr else ()))
            del o
        return trunk
