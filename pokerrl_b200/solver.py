"""Device-resident public tree + tabular CFR engine (host side: PyTorch tensors as buffers, ctypes into CUDA).

This is the engine behind the reference-shaped façades in `pokerrl_b200.cfr` / `pokerrl_b200.game.PublicTree` /
`pokerrl_b200.eval.br`.  All arithmetic happens in libpokerrl_b200.so; this file only owns buffers and the
iteration schedule of `PokerRL/cfr/_CFRBase.py:110-134`.
"""
import ctypes as C
import os

import numpy as np
import torch

from pokerrl_b200 import _native as nat
from pokerrl_b200 import algorithm
from pokerrl_b200 import dcfr as _dcfr


def _require_cuda(device):
    """torch.device of the GPU to use: the given one, else the process's CURRENT device (under torchrun each rank sets
    its own with torch.cuda.set_device; never silently cuda:0)."""
    if not torch.cuda.is_available():
        raise RuntimeError("pokerrl_b200 needs a CUDA device (sm_90a); there is no CPU fallback.")
    d = torch.device(device if device is not None else "cuda:%d" % torch.cuda.current_device())
    if d.type != "cuda":
        raise RuntimeError("pokerrl_b200 runs on CUDA devices only, got %r" % (device,))
    return torch.device("cuda:%d" % (d.index if d.index is not None else torch.cuda.current_device()))


def _stream(device=None):
    """the torch stream of `device` (default: current device) - launches go where the buffers live"""
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _on(device):
    """context: make `device` current for the ctypes launches inside (kernels run on the CURRENT device)"""
    return torch.cuda.device(device)


def structure_records(ft, order):
    """16-byte structure records of the two-card sweeps (prl_tree_t.node_rec2 / work_rec2), host side.
    node record  n: {parent, slot, first slot of the parent's children, kind(parent) | n_children(parent) << 8}
    work record  t: {node = order[t], its first child, first slot of its children, kind | n_children << 8};
                    terminal entries: {node, board id, pot as float bits, kind | (acted_last & 0xff) << 8}"""
    par = ft.parent.astype(np.int64)
    has_par = par >= 0
    sp_ = np.where(has_par, par, 0)
    fc_par = ft.first_child[sp_].astype(np.int64)
    nrec = np.zeros((ft.n_nodes, 4), np.int32)
    nrec[:, 0] = par
    nrec[:, 1] = ft.slot
    nrec[:, 2] = np.where(has_par, ft.slot[np.maximum(fc_par, 0)], 0)
    nrec[:, 3] = np.where(has_par, ft.kind[sp_].astype(np.int64) | (ft.n_children[sp_].astype(np.int64) << 8), 0)
    order = np.asarray(order).astype(np.int64)
    fc = ft.first_child[order].astype(np.int64)
    nonterm = (ft.n_children[order] > 0) & (fc >= 0)
    wrec = np.zeros((ft.n_nodes, 4), np.int32)
    wrec[:, 0] = order
    wrec[:, 1] = np.where(nonterm, fc, 0)
    wrec[:, 2] = np.where(nonterm, ft.slot[np.maximum(fc, 0)], 0)
    wrec[:, 3] = ft.kind[order].astype(np.int64) | (ft.n_children[order].astype(np.int64) << 8)
    term = ~nonterm  # terminal entries: {node, board id, pot (float bits), kind | (acted_last & 0xff) << 8}
    wrec[term, 1] = ft.board[order[term]]
    wrec[term, 2] = ft.pot[order[term]].astype(np.float32).view(np.int32)
    wrec[term, 3] = ft.kind[order[term]].astype(np.int64) | ((ft.acted_last[order[term]].astype(np.int64) & 0xff) << 8)
    return nrec, wrec


class DeviceTree:
    """FlatTree uploaded to HBM + the prl_tree_t descriptor handed to the C ABI."""

    def __init__(self, ft, device=None):
        self.ft = ft
        self.device = _require_cuda(device)
        rules = ft.rules
        self.R = ft.R
        # row stride: R for the one-card games (padding Leduc rows 6 -> 8 floats only adds bytes to a latency-bound sweep);
        # two-card rows (R = 1326) are padded to a multiple of 4 floats so that every row starts 16-byte aligned
        self.ld = ft.R if rules.N_HOLE_CARDS == 1 else -(-ft.R // 4) * 4
        dev = self.device

        def up(a, dt):
            return torch.from_numpy(np.ascontiguousarray(a).astype(dt)).to(dev)

        board = ft.board.copy().astype(np.int32)
        if rules.N_HOLE_CARDS == 1:
            # one-card games: kernels take the board card itself (-1 = none)
            bc = ft.node_board_cards()[:, 0].astype(np.int32)
            board = np.where(bc >= 0, bc, -1).astype(np.int32)
        self.t_parent = up(ft.parent, np.int32)
        self.t_first_child = up(ft.first_child, np.int32)
        self.t_n_children = up(ft.n_children, np.int32)
        self.t_slot = up(ft.slot, np.int32)
        self.t_kind = up(ft.kind, np.int8)
        self.t_acted_last = up(ft.acted_last, np.int8)
        self.t_pot = up(ft.pot, np.float32)
        self.t_board = up(board, np.int32)
        self._level_start = np.ascontiguousarray(ft.level_start, dtype=np.int64)
        d = nat.PrlTree()
        d.n_nodes, d.n_levels, d.n_slots = ft.n_nodes, ft.n_levels, ft.n_slots
        d.n_range, d.ld, d.n_hole = self.R, self.ld, rules.N_HOLE_CARDS
        d.n_deck, d.n_suits = rules.N_CARDS_IN_DECK, rules.N_SUITS
        d.pair_bonus = rules.PAIR_BONUS or 0
        d.max_actions = ft.max_actions
        d.level_start = self._level_start.ctypes.data
        d.parent, d.first_child = self.t_parent.data_ptr(), self.t_first_child.data_ptr()
        d.n_children, d.slot = self.t_n_children.data_ptr(), self.t_slot.data_ptr()
        d.kind, d.acted_last = self.t_kind.data_ptr(), self.t_acted_last.data_ptr()
        d.pot, d.board = self.t_pot.data_ptr(), self.t_board.data_ptr()
        order, level_nonterm = ft.work_order()
        self.t_order = up(order, np.int32)
        self._level_nonterm = np.ascontiguousarray(level_nonterm, dtype=np.int64)
        d.order, d.level_nonterm = self.t_order.data_ptr(), self._level_nonterm.ctypes.data
        d.meta = None
        self.desc = d
        if rules.N_HOLE_CARDS == 1:
            # the one-card kernels assume chance child k deals card k (boards ascending, PublicTree.py:193-203)
            ch = np.nonzero(ft.kind == nat.KIND_CHANCE)[0]
            assert np.all(ft.n_children[ch] == rules.N_CARDS_IN_DECK)
            fc0 = ft.first_child[ch[0]] if ch.size else 0
            assert ch.size == 0 or np.array_equal(board[fc0:fc0 + rules.N_CARDS_IN_DECK],
                                                  np.arange(rules.N_CARDS_IN_DECK))
        with _on(dev):
            if rules.N_HOLE_CARDS == 1:
                self.t_meta = torch.zeros(ft.n_nodes, 4, dtype=torch.int32, device=dev)
                nat.call("prl_pack_node_meta", C.byref(d), C.c_void_p(self.t_meta.data_ptr()), _stream(dev))
                d.meta = self.t_meta.data_ptr()
            else:
                self._init_two_card(ft, d, up)

    def _init_two_card(self, ft, d, up):
        """Board tables of the Hold'em family: card masks, deal probabilities, parent weights, strength-order tables
        (hand ranks by the GPU evaluator, then prl_board_order_tables), suit-permutation tables."""
        from math import comb
        from pokerrl_b200.hand_eval import hand_rank_all_hands_on_given_boards
        rules, dev = ft.rules, self.device
        lut = rules.get_lut_holder()
        self.t_hand_cards = up(lut.LUT_IDX_2_HOLE_CARDS, np.int8)
        bc = ft.board_cards()  # [n_boards_total, n_board_cards], global board id order
        nb = bc.shape[0]
        mask = np.zeros(nb, np.uint64)
        for k in range(bc.shape[1]):
            live = bc[:, k] >= 0
            mask[live] |= (np.uint64(1) << bc[live, k].astype(np.uint64))
        self.t_board_mask = torch.from_numpy(mask.view(np.int64)).to(dev)
        self.t_board_prob = up(ft.board_prob, np.float32)
        self.t_board_mult = up(ft.board_mult, np.float32)
        is_complete = (bc >= 0).sum(axis=1) == rules.N_TOTAL_BOARD_CARDS
        self.t_board_complete = up(is_complete, np.uint8)
        complete = np.nonzero(is_complete)[0]
        gs = torch.full((nb, self.R), -1, dtype=torch.int16, device=dev)
        ge, pos = torch.full_like(gs, -1), torch.full_like(gs, -1)
        n_deck = rules.N_CARDS_IN_DECK
        row_order = torch.full((nb, n_deck, n_deck - 1), -1, dtype=torch.int16, device=dev)
        row_pos = torch.zeros((nb, self.R, 4), dtype=torch.uint8, device=dev)
        self.t_board_ranks = torch.full((nb, self.R), -1, dtype=torch.int32, device=dev)
        CH = 16384
        for i in range(0, complete.size, CH):
            ids = torch.from_numpy(complete[i:i + CH]).to(dev)
            ranks = hand_rank_all_hands_on_given_boards(bc[complete[i:i + CH]], device=dev)
            self.t_board_ranks[ids] = ranks
            g1, g2, g3 = (torch.empty((ids.numel(), self.R), dtype=torch.int16, device=dev) for _ in range(3))
            ro = torch.empty((ids.numel(), n_deck, n_deck - 1), dtype=torch.int16, device=dev)
            rp = torch.zeros((ids.numel(), self.R, 4), dtype=torch.uint8, device=dev)
            nat.call("prl_board_order_tables", C.c_void_p(ranks.data_ptr()), int(ids.numel()), self.R, n_deck,
                     C.c_void_p(g1.data_ptr()), C.c_void_p(g2.data_ptr()), C.c_void_p(g3.data_ptr()),
                     C.c_void_p(ro.data_ptr()), C.c_void_p(rp.data_ptr()), _stream(dev))
            gs[ids], ge[ids], pos[ids], row_order[ids], row_pos[ids] = g1, g2, g3, ro, rp
        self.t_board_gs, self.t_board_ge, self.t_board_pos = gs, ge, pos
        self.t_board_row_order, self.t_board_row_pos = row_order, row_pos
        # packed per-hand showdown record (one 16-byte load in terminal2_kernel): see prl_tree_t.board_hand_rec
        self.t_board_hand_rec = None
        if os.environ.get("PRL_NO_HAND_REC", "0") != "1":
            rec = torch.zeros((nb, self.R, 8), dtype=torch.int16, device=dev)
            row_base = self.t_hand_cards.to(torch.int16) * 53  # [R, 2]
            for i in range(0, nb, CH):
                sl = slice(i, min(nb, i + CH))
                rec[sl, :, 0], rec[sl, :, 1] = gs[sl], ge[sl]
                q = row_pos[sl].to(torch.int16)
                rec[sl, :, 2], rec[sl, :, 3] = row_base[:, 0] + q[:, :, 0], row_base[:, 0] + q[:, :, 2]
                rec[sl, :, 4], rec[sl, :, 5] = row_base[:, 1] + q[:, :, 1], row_base[:, 1] + q[:, :, 3]
            self.t_board_hand_rec = rec
        sp = ft.board_spec.sym_perm
        self.t_sym_perm = up(sp, np.int16) if sp is not None else None
        dec_per_level = [int(((ft.kind[int(ft.level_start[k]):int(ft.level_start[k + 1])] <= nat.KIND_P1)).sum())
                         for k in range(ft.n_levels)]
        self._level_ndec = np.ascontiguousarray(dec_per_level, dtype=np.int64)
        ch = ft.kind == nat.KIND_CHANCE
        d.level_ndec = self._level_ndec.ctypes.data
        d.hand_cards = self.t_hand_cards.data_ptr()
        d.n_boards = nb
        d.max_chance_children = int(ft.n_children[ch].max()) if ch.any() else 0
        d.board_mask, d.board_prob = self.t_board_mask.data_ptr(), self.t_board_prob.data_ptr()
        d.board_mult = self.t_board_mult.data_ptr()
        d.board_gs, d.board_ge, d.board_pos = gs.data_ptr(), ge.data_ptr(), pos.data_ptr()
        d.board_row_order, d.board_row_pos = row_order.data_ptr(), row_pos.data_ptr()
        d.board_complete = self.t_board_complete.data_ptr()
        d.board_hand_rec = self.t_board_hand_rec.data_ptr() if self.t_board_hand_rec is not None else None
        # one 16-byte structure record per node (top-down sweep) and per work-list entry (bottom-up sweep over decision
        # nodes): see prl_tree_t.node_rec2 / work_rec2
        self.t_node_rec2 = self.t_work_rec2 = None
        if os.environ.get("PRL_NO_NODE_REC", "0") != "1":
            nrec, wrec = structure_records(ft, self.t_order.cpu().numpy())
            self.t_node_rec2, self.t_work_rec2 = up(nrec, np.int32), up(wrec, np.int32)
        self._level_nfold = np.ascontiguousarray(
            [int((ft.kind[int(ft.level_start[k]):int(ft.level_start[k + 1])] == nat.KIND_FOLD).sum())
             for k in range(ft.n_levels)], dtype=np.int64)
        d.level_nfold = self._level_nfold.ctypes.data
        d.node_rec2 = self.t_node_rec2.data_ptr() if self.t_node_rec2 is not None else None
        d.work_rec2 = self.t_work_rec2.data_ptr() if self.t_work_rec2 is not None else None
        d.n_sym = 0 if sp is None else int(sp.shape[0])
        d.sym_perm = self.t_sym_perm.data_ptr() if sp is not None else None
        n_deck, n_hole = rules.N_CARDS_IN_DECK, rules.N_HOLE_CARDS
        d.eq_const = comb(n_deck, n_hole) / comb(n_deck - n_hole, n_hole)
        self._init_allin(ft, d, complete)
        # scratch of the chance-node reductions (see prl_buffers_t.workspace)
        max_chance_per_level = max([int((ft.kind[int(ft.level_start[k]):int(ft.level_start[k + 1])] == nat.KIND_CHANCE).sum())
                                    for k in range(ft.n_levels)] + [0])
        chunks = -(-d.max_chance_children // 128)
        self.workspace_bytes = 4 * max(1, max_chance_per_level) * (chunks + 1) * self.ld * 4

    def _init_allin(self, ft, d, complete):
        """All-in showdowns before the board is complete (PRL_KIND_SHOWDOWN_ALLIN): per public board they occur on, the equity
        matrix of the boards it runs out over (ft.allin_completions()) as tensor-core operand tiles - csrc/allin_dense.cu;
        ValueFiller.py:160-175 is the one-card analogue."""
        from pokerrl_b200.allin import AllinEquity
        nodes = np.nonzero(ft.kind == nat.KIND_SHOWDOWN_ALLIN)[0]
        if nodes.size == 0:
            return
        self.allin = {}
        for key, (boards, w, sym) in ft.allin_completions().items():
            self.allin[key] = AllinEquity(ft.rules, device=self.device, boards=boards, weights=w, sym_perm=sym)
        first = next(iter(self.allin.values()))
        self._allin_nodes = np.ascontiguousarray(nodes, dtype=np.int32)
        self._allin_pot = np.ascontiguousarray(ft.pot[nodes], dtype=np.float32)
        self._allin_tiles = (C.c_void_p * nodes.size)(*[self.allin[int(ft.board[n])].tiles.data_ptr() for n in nodes])
        level_of = np.searchsorted(np.asarray(ft.level_start), nodes, side="right") - 1
        self._level_nallin = np.ascontiguousarray(np.bincount(level_of, minlength=ft.n_levels), dtype=np.int64)
        d.level_nallin = self._level_nallin.ctypes.data
        d.allin_nodes, d.allin_pot = self._allin_nodes.ctypes.data, self._allin_pot.ctypes.data
        d.allin_tiles = C.cast(self._allin_tiles, C.c_void_p)
        d.allin_partial = first.partial.data_ptr()

    @property
    def n_nodes(self):
        return self.ft.n_nodes

    @property
    def n_slots(self):
        return self.ft.n_slots


class TreeBuffers:
    """reach / ev / ev_br node vectors and regret / strategy / average tables (torch tensors in HBM)."""

    def __init__(self, dtree, with_tables=True, avg_dtype=torch.float32, share=None):
        dev, N, S, ld = dtree.device, dtree.n_nodes, dtree.n_slots, dtree.ld
        z = lambda *s, dtype=torch.float32: torch.zeros(*s, dtype=dtype, device=dev)  # noqa: E731
        self.reach = z(2, N, ld)
        if share is None:
            self.ev, self.ev_br = z(2, N, ld), z(2, N, ld)
            self.regret = z(S, ld) if with_tables else None
            self.strat = z(S, ld) if with_tables else None
            self.avg = z(S, ld, dtype=avg_dtype) if with_tables else None
        else:  # evaluation view: own reach, everything else shared with the training buffers
            self.ev, self.ev_br = share.ev, share.ev_br
            self.regret, self.strat, self.avg = share.regret, share.strat, share.avg
        d = nat.PrlBuffers()
        wb = getattr(dtree, "workspace_bytes", 0)
        if wb:
            self.workspace = share.workspace if share is not None else torch.zeros(wb // 4, dtype=torch.float32, device=dev)
            d.workspace, d.workspace_bytes = self.workspace.data_ptr(), wb
        d.reach, d.ev, d.ev_br = self.reach.data_ptr(), self.ev.data_ptr(), self.ev_br.data_ptr()
        d.regret = self.regret.data_ptr() if self.regret is not None else None
        d.strat = self.strat.data_ptr() if self.strat is not None else None
        d.avg = self.avg.data_ptr() if self.avg is not None else None
        self.desc = d


class TreeOps:
    """Thin wrappers over the C ABI passes for one (tree, buffers) pair."""

    def __init__(self, dtree, bufs):
        self.dtree, self.bufs = dtree, bufs
        self._expl = torch.zeros(2, dtype=torch.float32, device=dtree.device)

    def reach_pass(self, modes, player_mask=3):
        dev = self.dtree.device
        with _on(dev):
            nat.call("prl_reach_pass", C.byref(self.dtree.desc), C.byref(self.bufs.desc), player_mask,
                     nat.modes(*modes), _stream(dev))

    def value_pass(self, modes, player_mask=3, with_br=True):
        dev = self.dtree.device
        with _on(dev):
            nat.call("prl_value_pass", C.byref(self.dtree.desc), C.byref(self.bufs.desc), player_mask, int(with_br),
                     nat.modes(*modes), _stream(dev))

    def evaluate(self, modes, do_reach):
        """One persistent launch: [reach pass,] value pass with BR, root exploitability -> float32[2] chips."""
        dev = self.dtree.device
        with _on(dev):
            nat.call("prl_evaluate", C.byref(self.dtree.desc), C.byref(self.bufs.desc), nat.modes(*modes), int(do_reach),
                     C.c_void_p(self._expl.data_ptr()), _stream(dev))
        return self._expl.cpu().numpy()

    def root_exploitability(self):
        """float32[2] chips (device->host read)."""
        dev = self.dtree.device
        with _on(dev):
            nat.call("prl_root_exploitability", C.byref(self.dtree.desc), C.byref(self.bufs.desc),
                     C.c_void_p(self._expl.data_ptr()), _stream(dev))
        return self._expl.cpu().numpy()


class CFRSolver:
    """Iteration schedule of `_CFRBase` (reset :110-120, iteration :122-134) on the GPU.

    One `iteration()` = for p in (0, 1): fused half-iteration (value pass for p with regret update and regret
    matching, then reach pass for p with the average-strategy update).  Exploitability of the current / average
    strategy is a separate, optional evaluation (the reference does both every iteration).
    """

    def __init__(self, ft, algo="CFRPlus", delay=0, device=None, avg_f64=False, persistent=True, dcfr=_dcfr.DEFAULT,
                 pcfr_gamma=algorithm.PCFR_GAMMA):
        self.persistent = bool(persistent)  # one cooperative launch per call instead of one launch per tree level
        self.ft = ft
        self.alg = algorithm.Algorithm(algo, delay, dcfr, _require_cuda(device), pcfr_gamma)
        self.algo_name, self.algo, self.delay, self.dcfr = self.alg.name, self.alg.code, self.alg.delay, self.alg.dcfr
        self._factors = self.alg.factors  # DCFR's / PCFR+'s device table (None for the others), grown by factor_table
        self.avg_f64 = bool(avg_f64) and self.algo == nat.ALGO_CFR_PLUS
        self.dtree = DeviceTree(ft, device)
        self.bufs = TreeBuffers(self.dtree, avg_dtype=torch.float64 if self.avg_f64 else torch.float32)
        self.ops = TreeOps(self.dtree, self.bufs)
        self._eval_bufs = None
        self.ev_normalizer = ft.game_cls.EV_NORMALIZER
        self.reset()

    def reset(self):
        self.iter_counter = 0
        for t in (self.bufs.regret, self.bufs.strat, self.bufs.avg):
            t.zero_()
        self.modes = [nat.STRAT_UNIFORM64, nat.STRAT_UNIFORM64]  # StrategyFiller.py:61-62
        self.ops.reach_pass(self.modes)

    def iteration(self, n=1):
        with _on(self.dtree.device):
            self._iteration(n)

    def _bind_factors(self, n):
        """DCFR / PCFR+: the factor table covers the next n iterations"""
        self.bufs.desc.dcfr = self.alg.factor_table(self.iter_counter + n)

    def _iteration(self, n):
        self._bind_factors(n)
        tree, buf = C.byref(self.dtree.desc), C.byref(self.bufs.desc)
        _stream = lambda: C.c_void_p(torch.cuda.current_stream(self.dtree.device).cuda_stream)  # noqa: E731
        if self.persistent and n > 0:
            nat.call("prl_cfr_iterations", tree, buf, self.algo, self.iter_counter, n, self.delay,
                     int(self.avg_f64), nat.modes(*self.modes), _stream())
            self.modes = [nat.STRAT_F32, nat.STRAT_F32]
            self.iter_counter += n
            return
        for _ in range(n):
            for p in (0, 1):
                nat.call("prl_cfr_half_iteration", tree, buf, self.algo, p, self.iter_counter, self.delay,
                         int(self.avg_f64), nat.modes(*self.modes), _stream())
                self.modes[p] = nat.STRAT_F32
            self.iter_counter += 1

    # ---- checkpoint / resume (the reference's CFR classes keep regrets only inside node objects; WorkerBase.py:23-38 is
    #      a no-op skeleton) - SURVEY.md §8f N1
    def _identity(self):
        return {"engine": "levels", **self.alg.identity(), "avg_f64": self.avg_f64, "rank": getattr(self, "rank", 0),
                "world": getattr(self, "world", 1), "n_nodes": self.ft.n_nodes}

    def state_dict(self):
        return {**self._identity(), "iter_counter": self.iter_counter, "modes": list(self.modes),
                "regret": self.bufs.regret.cpu(), "strat": self.bufs.strat.cpu(), "avg": self.bufs.avg.cpu()}

    def load_state_dict(self, state):
        algorithm.check_identity(state, self._identity())
        if tuple(state["regret"].shape) != tuple(self.bufs.regret.shape) or state["avg"].dtype != self.bufs.avg.dtype:
            raise ValueError("checkpoint tables do not fit this solver (shape %s vs %s, avg dtype %s vs %s)" % (
                tuple(state["regret"].shape), tuple(self.bufs.regret.shape), state["avg"].dtype, self.bufs.avg.dtype))
        self.iter_counter, self.modes = int(state["iter_counter"]), list(state["modes"])
        self.bufs.regret.copy_(state["regret"])
        self.bufs.strat.copy_(state["strat"])
        self.bufs.avg.copy_(state["avg"].to(self.bufs.avg.dtype))
        self.ops.reach_pass(self.modes)  # reach rows are a function of the strategies

    # ---- evaluation (_CFRBase._log_curr_strat_expl :198-216, _evaluate_avg_strats :218-262)
    def _metric(self, expl):
        return algorithm.seat_averaged(expl, self.ev_normalizer)

    def exploitability_current(self):
        if self.persistent:
            return self._metric(self.ops.evaluate(self.modes, do_reach=False))
        self._value_pass_br(self.ops, self.modes)
        return self._metric(self.ops.root_exploitability())

    def average_modes(self):
        m = {algorithm.SUMS: nat.STRAT_AVG_SUM, algorithm.CURRENT: nat.STRAT_F32,
             algorithm.AVERAGE: nat.STRAT_AVG_F64 if self.avg_f64 else nat.STRAT_AVG_F32}[self.alg.average(self.iter_counter)]
        return [m, m]

    def _value_pass_br(self, ops, modes):
        """value pass with best responses of both seats over the buffers of `ops` (per-level launches)"""
        ops.value_pass(modes, 3, True)

    def exploitability_average(self):
        if self._eval_bufs is None:
            self._eval_bufs = TreeBuffers(self.dtree, share=self.bufs)
            self._eval_ops = TreeOps(self.dtree, self._eval_bufs)
        m = self.average_modes()
        if self.persistent:
            return self._metric(self._eval_ops.evaluate(m, do_reach=True))
        self._eval_ops.reach_pass(m)
        self._value_pass_br(self._eval_ops, m)
        return self._metric(self._eval_ops.root_exploitability())
