"""Board-resident CFR+ engine for two-card games with one chance layer (host side of csrc/cfr_board.cu).

`BoardCFRSolver` has the interface of `solver.CFRSolver` / `distributed.ShardedCFRSolver` (iteration / reset /
exploitability_current / exploitability_average / state_dict) and is what `pokerrl_b200.cfr.CFRPlus` runs for
Flop5Holdem (PokerRL/game/games.py:222-254).  The post-deal subtrees never exist as node vectors in HBM: one persistent
kernel walks (board, seat) units; only the pre-deal trunk (5 nodes in Flop5Holdem) is swept by the level kernels.

Sharding (SURVEY.md §8e): boards round-robin over the ranks, trunk replicated, ONE all-reduce per bottom-up sweep - of
the chance node's sums, which are 64-bit fixed point: integer addition is associative, so any number of ranks (and any
grouping inside a rank) produces bit-identical sums, hence bit-identical trajectories.
"""
import ctypes as C
import math
import os

import numpy as np
import torch

from pokerrl_b200 import _native as nat
from pokerrl_b200.game.flat_tree import FlatTree
from pokerrl_b200.game.holdem_boards import BoardSpec
from pokerrl_b200.solver import DeviceTree, TreeBuffers, TreeOps, _require_cuda

SRC_REGRET, SRC_AVG, SRC_AVG_SUM = 0, 1, 2
ALGOS = {"VanillaCFR": nat.ALGO_VANILLA, "CFRPlus": nat.ALGO_CFR_PLUS, "LinearCFR": nat.ALGO_LINEAR}


def board_layout():
    out = (C.c_int32 * 8)()
    nat.call("prl_board_layout", out)
    return dict(n_live=out[0], ldb=out[1], blob=out[2], sh_off=out[3], rows_off=out[4], live_cards=out[5],
                row_pad=out[6], n_local=out[7])


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def supports(game_cls, env_args, algo):
    """True iff the game's abstract tree is one pre-deal trunk + one chance layer + the compiled post-deal shape"""
    if algo not in ALGOS or game_cls.RULES.N_HOLE_CARDS != 2 or game_cls.RULES.N_CARDS_IN_DECK != 52:
        return False
    if game_cls.RULES.N_FLOP_CARDS != 5 or os.environ.get("PRL_ENGINE", "board") != "board":
        return False
    try:
        ft1 = FlatTree(game_cls, env_args, board_spec=_one_board_spec())
    except Exception:
        return False
    st = ft1.board_subtree()
    if st is None or sum(1 for n in ft1.abs_nodes if n.kind == nat.KIND_CHANCE) != 1:
        return False
    g = nat.PrlBoardGame()
    _fill_shape(g, st)
    return bool(nat.lib().prl_board_shape_ok(C.byref(g)))


def _one_board_spec():
    return BoardSpec(np.array([[0, 1, 2, 3, 4]], np.int8), np.ones(1), np.ones(1), None, "shape probe")


def _fill_shape(g, st):
    g.n_local = st["n_local"]
    for i in range(st["n_local"]):
        g.kind[i], g.parent[i], g.first_child[i] = st["kind"][i], st["parent"][i], st["first_child"][i]
        g.n_children[i], g.acted_last[i], g.pot[i] = st["n_children"][i], st["acted_last"][i], st["pot"][i]


class BoardCFRSolver:
    def __init__(self, game_cls, env_args, board_spec=None, algo="CFRPlus", delay=0, device=None, rank=0, world=1,
                 group=None, grid=0, reduce_fn=None):
        if algo not in ALGOS:
            raise ValueError("unknown algorithm %r" % (algo,))
        self.device = _require_cuda(device)
        self.rank, self.world, self.group = int(rank), int(world), group
        # cross-rank sum of the fixed-point chance sums, in place; default: torch.distributed all-reduce when world > 1
        self._reduce_fn = reduce_fn
        self.algo_name, self.algo = algo, ALGOS[algo]
        self.delay = int(delay) if algo == "CFRPlus" else 0
        # Vanilla / Linear CFR: weight of the average-strategy contribution of each seat's last update that the post-deal rows
        # have not received yet (it is added by the next sweep that walks those rows: csrc/cfr_board.cu, DEFER)
        self._pending = [0.0, 0.0]
        # CFR+: iteration of each seat's averaging step that is still pending (-1: none).  An update sweep with nothing pending
        # leaves its step pending; the seat's next update sweep applies it together with its own (csrc/cfr_board.cu, AVG):
        # every other sweep of a seat neither reads nor writes the average rows
        self._avg_due = [-1, -1]
        self.game_cls, self.env_args = game_cls, env_args
        rules = game_cls.RULES
        spec = board_spec if board_spec is not None else BoardSpec.full_game(rules)
        self.spec_full = spec
        self.L = board_layout()
        with torch.cuda.device(self.device):
            self._build(rules, spec, grid)
        self.ev_normalizer = game_cls.EV_NORMALIZER
        self.n_allreduce = 0
        self.reset()

    # ------------------------------------------------------------------------------------------------ construction
    def _build(self, rules, spec, grid):
        dev, L = self.device, self.L
        # structure: a one-board flat tree carries the trunk and the shape of the post-deal subtree
        self.ft1 = FlatTree(self.game_cls, self.env_args, board_spec=_one_board_spec())
        st = self.ft1.board_subtree()
        if st is None:
            raise ValueError("the game does not have ONE chance layer with a <= 16-node post-deal subtree")
        self.st = st
        self.chance_level = st["chance_level"]
        self.chance_node = st["chance_node"]
        sel = np.arange(self.rank, spec.boards.shape[0], self.world)
        self.board_ids = sel
        self.boards = np.ascontiguousarray(spec.boards[sel], np.int8)
        nb = self.n_boards = int(sel.size)
        self.n_boards_total = int(spec.boards.shape[0])
        self.R = rules.RANGE_SIZE
        # trunk: level sweeps over levels 0 .. chance_level of the one-board tree; the symmetrisation over the suit
        # permutations happens in prl_board_collect (integer sums), not in the level kernels
        self.trunk = DeviceTree(self.ft1, dev)
        self.trunk.desc.n_sym = 0
        self.trunk.desc.sym_perm = None
        self.bufs = TreeBuffers(self.trunk)
        self.ops = TreeOps(self.trunk, self.bufs)
        self._eval_bufs = None
        self.ld = self.trunk.ld
        sp = spec.sym_perm
        self.t_sym = None if sp is None else torch.from_numpy(np.ascontiguousarray(sp, np.int16)).to(dev)
        self.n_sym = 0 if sp is None else int(sp.shape[0])
        # per-board tables
        from pokerrl_b200.hand_eval import hand_rank_all_hands_on_given_boards
        self.t_blob = torch.empty((max(nb, 1), L["blob"]), dtype=torch.uint8, device=dev)
        lut = rules.get_lut_holder()
        t_hc = torch.from_numpy(np.ascontiguousarray(lut.LUT_IDX_2_HOLE_CARDS, np.int8)).to(dev)
        mask = np.zeros(nb, np.uint64)
        for k in range(self.boards.shape[1]):
            mask |= (np.uint64(1) << self.boards[:, k].astype(np.uint64))
        t_mask = torch.from_numpy(mask.view(np.int64)).to(dev)
        CH = 16384
        for i in range(0, nb, CH):
            n = min(CH, nb - i)
            ranks = hand_rank_all_hands_on_given_boards(self.boards[i:i + n], device=dev)
            nat.call("prl_board_build_tables", C.c_void_p(ranks.data_ptr()), C.c_void_p(t_mask[i:i + n].data_ptr()),
                     C.c_void_p(t_hc.data_ptr()), n, C.c_void_p(self.t_blob[i:i + n].data_ptr()), _stream(dev))
        torch.cuda.synchronize(dev)
        self.t_prob = torch.from_numpy(np.ascontiguousarray(spec.board_prob[sel], np.float32)).to(dev)
        self.t_mult = torch.from_numpy(np.ascontiguousarray(spec.board_mult[sel], np.float32)).to(dev)
        n_local = st["n_local"]
        dec = [i for i in range(n_local) if st["kind"][i] <= 1]
        self.rows_per_board = sum(st["n_children"][i] for i in dec)
        self.n_rows = nb * self.rows_per_board
        self.regret = torch.zeros((max(self.n_rows, 1), L["ldb"]), dtype=torch.float32, device=dev)
        self.avg = torch.zeros_like(self.regret)
        g = nat.PrlBoardGame()
        _fill_shape(g, st)
        g.n_boards, g.n_range, g.ld, g.n_deck = nb, self.R, self.ld, rules.N_CARDS_IN_DECK
        n_hole = rules.N_HOLE_CARDS
        g.eq_const = math.comb(g.n_deck, n_hole) / math.comb(g.n_deck - n_hole, n_hole)
        # fixed point: |sum| <= n_sym * K * max pot / 2 with headroom; 62 value bits
        bound = max(self.n_sym, 1) * g.eq_const * max(st["pot"]) * 0.5 * 4.0
        g.frac_bits = 62 - int(math.ceil(math.log2(bound)))
        # board-major rows: everything a (board, seat) unit touches is contiguous - row(i, j) = j * rows_per_board + row_of[i]
        row_of, rpb = (C.c_int32 * 16)(), C.c_int32(0)
        nat.call("prl_board_rows", row_of, C.byref(rpb))
        assert rpb.value == self.rows_per_board
        self.local_rows = {}  # local child node -> (row on board 0, stride per board)
        for i in range(n_local):
            g.row0[i], g.row_m[i] = -1, 0
        for d in dec:
            for a in range(st["n_children"][d]):
                c = st["first_child"][d] + a
                g.row0[c], g.row_m[c] = row_of[c], rpb.value
                self.local_rows[c] = (int(row_of[c]), rpb.value)
        g.grid = int(grid) if grid else int(nat.lib().prl_board_grid())
        g.tables, g.board_prob, g.board_mult = self.t_blob.data_ptr(), self.t_prob.data_ptr(), self.t_mult.data_ptr()
        g.regret, g.avg = self.regret.data_ptr(), self.avg.data_ptr()
        self.w_private = torch.zeros((g.grid, 2, self.R), dtype=torch.int64, device=dev)
        # chance sums: two generations of [4][R] int64 (a sweep writes one generation while slow peers may still read the other)
        self._symm = None
        self.collective = "none" if self.world == 1 else "nccl all_reduce(int64)"
        if (self.world > 1 and self._reduce_fn is None and os.environ.get("PRL_COLLECTIVE", "p2p") == "p2p"
                and os.environ.get("PRL_TRUNK", "fused") != "levels"):
            try:  # symmetric (peer-mapped) memory: the trunk kernel reads every rank's sums over NVLink itself
                import torch.distributed as dist
                import torch.distributed._symmetric_memory as symm_mem
                self.w_gens = symm_mem.empty((2, 4, self.R), dtype=torch.int64, device=dev)
                self.w_gens.zero_()
                self._symm = symm_mem.rendezvous(self.w_gens, group=self.group if self.group is not None else dist.group.WORLD)
                self._peer_ptrs = torch.tensor([int(x) for x in self._symm.buffer_ptrs], dtype=torch.int64, device=dev)
                self.collective = "one-shot NVLink sum inside trunk_kernel (symmetric memory, %d peers)" % self.world
            except Exception as e:  # noqa: BLE001 - any failure of the peer mapping leaves the NCCL path
                self._symm = None
                self.collective = "nccl all_reduce(int64) (symmetric memory unavailable: %s)" % type(e).__name__
        if self._symm is None:
            self.w_gens = torch.zeros((2, 4, self.R), dtype=torch.int64, device=dev)
        self._gen = 0
        self.w_total = self.w_gens[0]
        self.w_scratch = torch.zeros((4, self.R), dtype=torch.int64, device=dev)
        g.w_private, g.w_total = self.w_private.data_ptr(), self.w_total.data_ptr()
        self.g = g
        # the trunk in one launch (prl_board_trunk); PRL_TRUNK=levels keeps the level-kernel chain (A/B, cross-check)
        self.fused_trunk = os.environ.get("PRL_TRUNK", "fused") != "levels"
        self._expl = torch.zeros(2, dtype=torch.float32, device=dev)
        # where the level kernels expect the chance node's sums: prl_value_levels(chance_phase 1 / 2), one chance node,
        # one chunk -> W[arr] at float offset (4 + arr) * ld of the workspace
        self._w_off = 4 * self.ld
        self.n_nodes = int(self.ft1.level_start[self.chance_level + 1]) + self.n_boards_total * n_local
        self.n_nonterm = (int(((self.ft1.kind[:self.chance_node + 1] <= nat.KIND_CHANCE)).sum())
                          + self.n_boards_total * len(dec))

    # ------------------------------------------------------------------------------------------------ helpers
    def _trunk_desc(self, bufs, modes):
        ft, t = self.ft1, nat.PrlTrunk()
        n = self.chance_node + 1
        assert n <= 8 and int(ft.level_start[self.chance_level + 1]) == n, "the trunk must be the first nodes of the flat tree"
        t.n_nodes, t.chance_node, t.n_buf_nodes, t.ld, t.n_range = n, self.chance_node, self.trunk.n_nodes, self.ld, self.R
        t.mode[0], t.mode[1] = modes
        t.eq_const = self.g.eq_const
        for i in range(n):
            t.kind[i], t.first_child[i], t.n_children[i] = int(ft.kind[i]), int(ft.first_child[i]), int(ft.n_children[i])
            t.acted_last[i], t.pot[i] = int(ft.acted_last[i]), float(ft.pot[i])
            t.first_slot[i] = int(ft.first_slot[i]) if ft.first_slot[i] >= 0 else 0
        t.hand_cards = self.trunk.t_hand_cards.data_ptr()
        t.reach, t.ev, t.ev_br = bufs.reach.data_ptr(), bufs.ev.data_ptr(), bufs.ev_br.data_ptr()
        t.regret, t.strat, t.avg = bufs.regret.data_ptr(), bufs.strat.data_ptr(), bufs.avg.data_ptr()
        return t

    def _trunk(self, bufs, modes, evaluate, p):
        peers, n_peers, off = None, 0, 0
        if self._symm is not None:
            peers, n_peers, off = C.c_void_p(self._peer_ptrs.data_ptr()), self.world, self._gen * 4 * self.R
        nat.call("prl_board_trunk", C.byref(self.g), C.byref(self._trunk_desc(bufs, modes)), int(evaluate), p, self.n_sym,
                 C.c_void_p(self.t_sym.data_ptr()) if self.n_sym else None, self.iter_counter, self.delay,
                 C.c_void_p(self._expl.data_ptr()), peers, n_peers, off, C.c_void_p(self.w_scratch.data_ptr()), self.algo,
                 _stream(self.device))

    def _next_generation(self):
        """the next sweep(s) write the other generation of the chance sums"""
        self._gen ^= 1
        self.w_total = self.w_gens[self._gen]
        self.g.w_total = self.w_total.data_ptr()

    def _reduce(self, view):
        if self._symm is not None:
            # all ranks' sweeps are complete and visible before any trunk kernel reads the peers; the trunk kernel sums
            self._symm.barrier(channel=0)
            self.n_allreduce += 1
            return
        if self._reduce_fn is not None:
            self._reduce_fn(view)
        elif self.world > 1:  # the ONE collective of the path; int64 sums are exact in any order
            import torch.distributed as dist
            dist.all_reduce(view, op=dist.ReduceOp.SUM, group=self.group)
        self.n_allreduce += 1

    def _trunk_reach_row(self, bufs, seat):
        return C.c_void_p(bufs.reach.data_ptr() + 4 * (seat * self.trunk.n_nodes + self.chance_node) * self.ld)

    def _levels(self, bufs, mask, with_br, algo, upd_p, modes, hi, lo, phase):
        nat.call("prl_value_levels", C.byref(self.trunk.desc), C.byref(bufs.desc), mask, int(with_br), algo, upd_p,
                 self.iter_counter, self.delay, nat.modes(*modes), hi, lo, phase, _stream(self.device))

    def _reach_trunk(self, bufs, mask, algo, upd_p, modes):
        nat.call("prl_reach_levels", C.byref(self.trunk.desc), C.byref(bufs.desc), mask, algo, upd_p, self.iter_counter,
                 self.delay, nat.modes(*modes), 0, self.chance_level, _stream(self.device))

    def _sweep_begin(self, bufs, p, evaluate, src_own, src_opp):
        if not evaluate and self.algo == nat.ALGO_CFR_PLUS:
            t, due = self.iter_counter, self._avg_due[p]
            now = 1 if due >= 0 or t < self.delay else 0  # an iteration before delay has no step to leave pending
            self._avg_due[p] = -1 if now else t
            nat.call("prl_board_update_cfrp", C.byref(self.g), p, self._trunk_reach_row(bufs, 1 - p), t, self.delay, due, now,
                     _stream(self.device))
            return
        defer_w = 0.0
        if not evaluate and self.algo != nat.ALGO_CFR_PLUS:  # this sweep walks the opponent's rows: its pending average goes in
            defer_w, self._pending[1 - p] = self._pending[1 - p], 0.0
        nat.call("prl_board_sweep", C.byref(self.g), p, int(evaluate), src_own, src_opp, self._trunk_reach_row(bufs, 1 - p),
                 self.iter_counter, self.delay, self.algo, defer_w, 0, _stream(self.device))

    def flush_average(self):
        """Applies the average-strategy updates that are still pending: CFR+ averaging steps (prl_board_avg_flush), Vanilla /
        Linear CFR contributions (a light P1-only sweep per seat)"""
        with torch.cuda.device(self.device):
            for q in (0, 1):
                if self._avg_due[q] >= 0:
                    nat.call("prl_board_avg_flush", C.byref(self.g), q, self._avg_due[q], self.delay, _stream(self.device))
                    self._avg_due[q] = -1
                if self._pending[q] != 0.0:
                    nat.call("prl_board_sweep", C.byref(self.g), 1 - q, 0, 0, 0, self._trunk_reach_row(self.bufs, q),
                             self.iter_counter, self.delay, self.algo, self._pending[q], 1, _stream(self.device))
                    self._pending[q] = 0.0

    def _sweep_end(self, bufs, p, evaluate):
        """level-kernel trunk path: cross-rank sum, then the chance node's rows into the level kernels' workspace"""
        n_arr = 2 if evaluate else 1
        view = self.w_total[2 * p:2 * p + 2] if evaluate else self.w_total[:1]
        self._reduce(view)
        out = bufs.workspace.data_ptr() + 4 * (self._w_off + 2 * p * self.ld)
        g2 = self.g
        if evaluate and p == 1:  # collect reads w_total from its start: point it at this seat's arrays
            g2 = nat.PrlBoardGame.from_buffer_copy(self.g)
            g2.w_total = self.w_total.data_ptr() + 8 * 2 * self.R
        nat.call("prl_board_collect", C.byref(g2), n_arr, C.c_void_p(self.t_sym.data_ptr()) if self.n_sym else None,
                 self.n_sym, C.c_void_p(out), self.ld, _stream(self.device))

    def _sweep(self, bufs, p, evaluate, src_own, src_opp):
        self._sweep_begin(bufs, p, evaluate, src_own, src_opp)
        self._sweep_end(bufs, p, evaluate)

    def _update_begin(self, p):
        """first half of seat p's half-iteration: the board sweep (level path: the chance level's trunk terminals first)"""
        cl = self.chance_level
        if not self.fused_trunk:
            self._levels(self.bufs, 1 << p, False, self.algo, p, self.modes, cl, cl, 1)
        self._sweep_begin(self.bufs, p, False, SRC_REGRET, SRC_REGRET)

    def _update_end(self, p):
        """second half: cross-rank sum, chance node row, trunk regrets / matching / averaging, trunk reach of p"""
        cl = self.chance_level
        if self.algo != nat.ALGO_CFR_PLUS:  # VanillaCFR.py:56-59 / LinearCFR.py:55-58: weight of this update's strategy in the sums
            if not self.fused_trunk:
                raise RuntimeError("Vanilla / Linear CFR on the board engine need the fused trunk (unset PRL_TRUNK=levels)")
            self._pending[p] = float(self.iter_counter + 1) if self.algo == nat.ALGO_LINEAR else 1.0
        if self.fused_trunk:
            self._reduce(self.w_total[:1])
            self._trunk(self.bufs, self.modes, False, p)
            self.modes[p] = nat.STRAT_F32
            self._next_generation()
            return
        self._sweep_end(self.bufs, p, False)
        self._levels(self.bufs, 1 << p, False, self.algo, p, self.modes, cl, cl, 2)
        if cl > 0:
            self._levels(self.bufs, 1 << p, False, self.algo, p, self.modes, cl - 1, 0, 0)
        self.modes[p] = nat.STRAT_F32
        self._reach_trunk(self.bufs, 1 << p, self.algo, p, self.modes)

    # ------------------------------------------------------------------------------------------------ schedule
    def reset(self):
        with torch.cuda.device(self.device):
            self.iter_counter = 0
            for t in (self.regret, self.avg, self.bufs.regret, self.bufs.strat, self.bufs.avg):
                t.zero_()
            self._pending = [0.0, 0.0]
            self._avg_due = [-1, -1]
            self.modes = [nat.STRAT_UNIFORM64, nat.STRAT_UNIFORM64]
            self._reach_trunk(self.bufs, 3, -1, -1, self.modes)

    def iteration(self, n=1):
        with torch.cuda.device(self.device):
            for _ in range(n):
                for p in (0, 1):  # _CFRBase.py:122-128
                    self._update_begin(p)
                    self._update_end(p)
                self.iter_counter += 1

    def _evaluate(self, bufs, modes, src):
        cl = self.chance_level
        if self.fused_trunk:
            for p in (0, 1):
                self._sweep_begin(bufs, p, True, src, src)
            self._reduce(self.w_total)
            self._trunk(bufs, modes, True, -1)
            self._next_generation()
            e = self._expl.cpu().numpy()
            return sum(float(e[p]) * self.ev_normalizer for p in range(2)) / 2
        self._levels(bufs, 3, True, -1, -1, modes, cl, cl, 1)
        for p in (0, 1):
            self._sweep(bufs, p, True, src, src)
        self._levels(bufs, 3, True, -1, -1, modes, cl, cl, 2)
        if cl > 0:
            self._levels(bufs, 3, True, -1, -1, modes, cl - 1, 0, 0)
        ops = TreeOps(self.trunk, bufs) if bufs is not self.bufs else self.ops
        e = ops.root_exploitability()
        return sum(float(e[p]) * self.ev_normalizer for p in range(2)) / 2

    def exploitability_current(self):
        with torch.cuda.device(self.device):
            return self._evaluate(self.bufs, self.modes, SRC_REGRET)

    def exploitability_average(self):
        if self.iter_counter <= self.delay:
            raise RuntimeError("no average strategy before iteration delay+1 (CFRPlus.py:33-35)")
        with torch.cuda.device(self.device):
            if self._eval_bufs is None:
                self._eval_bufs = TreeBuffers(self.trunk, share=self.bufs)
            self.flush_average()
            if self.algo != nat.ALGO_CFR_PLUS:  # normalised reach-weighted sums (LinearCFR.py:64-71, VanillaCFR.py:65-72)
                modes, src = [nat.STRAT_AVG_SUM, nat.STRAT_AVG_SUM], SRC_AVG_SUM
            elif self.iter_counter == self.delay + 1:  # avg == copy of the current strategy (CFRPlus.py:83-84)
                modes, src = [nat.STRAT_F32, nat.STRAT_F32], SRC_REGRET
            else:
                modes, src = [nat.STRAT_AVG_F32, nat.STRAT_AVG_F32], SRC_AVG
            self._reach_trunk(self._eval_bufs, 3, -1, -1, modes)
            return self._evaluate(self._eval_bufs, modes, src)

    # ------------------------------------------------------------------------------------------------ interfaces
    def natural_tables(self, ft):
        """(regret, avg) as natural-order float32 [ft.n_slots, ld] tensors in the slot order of the flat tree `ft` built over
        THIS rank's boards (for agents, exports and parity tests on small instances)."""
        assert ft.board_spec.boards.shape[0] == self.n_boards
        self.flush_average()
        st = ft.board_subtree()
        out = []
        dev = self.device
        src, dst = [], []
        for i, (r0, m) in sorted(self.local_rows.items()):
            n0 = st["node_base"][i] + st["node_k"][i]
            src += [r0, m]
            dst += [int(ft.slot[n0]), st["node_m"][i]]
        t_src = torch.tensor(src, dtype=torch.int64, device=dev)
        t_dst = torch.tensor(dst, dtype=torch.int64, device=dev)
        n_trunk_slots = self.bufs.regret.shape[0] - self.rows_per_board  # slots of the one-board trunk tree before the board
        for tab, trunk_tab in ((self.regret, self.bufs.regret), (self.avg, self.bufs.avg)):
            nat_tab = torch.zeros((ft.n_slots, self.ld), dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                nat.call("prl_board_permute", C.byref(self.g), len(self.local_rows), C.c_void_p(t_src.data_ptr()),
                         C.c_void_p(t_dst.data_ptr()), C.c_void_p(tab.data_ptr()), C.c_void_p(nat_tab.data_ptr()), self.ld, 1,
                         _stream(dev))
            nat_tab[:n_trunk_slots] = trunk_tab[:n_trunk_slots]
            out.append(nat_tab)
        return out

    def load_natural_tables(self, ft, regret, avg):
        """inverse of natural_tables (teacher forcing in the parity tests, checkpoints written by the level engine)"""
        self._pending = [0.0, 0.0]  # the given average is complete
        self._avg_due = [-1, -1]
        st = ft.board_subtree()
        dev = self.device
        src, dst = [], []
        for i, (r0, m) in sorted(self.local_rows.items()):
            n0 = st["node_base"][i] + st["node_k"][i]
            src += [r0, m]
            dst += [int(ft.slot[n0]), st["node_m"][i]]
        t_src = torch.tensor(src, dtype=torch.int64, device=dev)
        t_dst = torch.tensor(dst, dtype=torch.int64, device=dev)
        n_trunk_slots = self.bufs.regret.shape[0] - self.rows_per_board
        for tab, trunk_tab, given in ((self.regret, self.bufs.regret, regret), (self.avg, self.bufs.avg, avg)):
            nat_tab = torch.zeros((ft.n_slots, self.ld), dtype=torch.float32, device=dev)
            nat_tab[:, :given.shape[1]] = torch.as_tensor(given, dtype=torch.float32).to(dev)
            with torch.cuda.device(dev):
                nat.call("prl_board_permute", C.byref(self.g), len(self.local_rows), C.c_void_p(t_src.data_ptr()),
                         C.c_void_p(t_dst.data_ptr()), C.c_void_p(tab.data_ptr()), C.c_void_p(nat_tab.data_ptr()), self.ld, 0,
                         _stream(dev))
            trunk_tab[:n_trunk_slots] = nat_tab[:n_trunk_slots]

    def set_trunk_strategy_from_regrets(self):
        """after load_natural_tables: the trunk's stored strategy rows = regret matching of its regret rows, reach rows
        refreshed (the post-deal rows need nothing: their strategy is never stored)"""
        ft = self.ft1
        n_trunk_slots = self.bufs.regret.shape[0] - self.rows_per_board
        r = torch.clamp(self.bufs.regret[:n_trunk_slots], min=0)
        for n in range(self.chance_node + 1):
            if ft.kind[n] <= 1 and ft.first_child[n] >= 0:
                fs, A = int(ft.first_slot[n]), int(ft.n_children[n])
                s = r[fs:fs + A].sum(dim=0, keepdim=True)
                self.bufs.strat[fs:fs + A] = torch.where(s > 0, r[fs:fs + A] / torch.where(s > 0, s, torch.ones_like(s)),
                                                         torch.full_like(s, 1.0 / A))
        self.modes = [nat.STRAT_F32, nat.STRAT_F32]
        with torch.cuda.device(self.device):
            self._reach_trunk(self.bufs, 3, -1, -1, self.modes)

    def state_dict(self):
        self.flush_average()
        return {"engine": "board", "algo": self.algo_name, "delay": self.delay, "iter_counter": self.iter_counter,
                "modes": list(self.modes), "rank": self.rank, "world": self.world, "n_boards": self.n_boards,
                "n_boards_total": self.n_boards_total, "regret": self.regret.cpu(), "avg": self.avg.cpu(),
                "trunk_regret": self.bufs.regret.cpu(), "trunk_strat": self.bufs.strat.cpu(), "trunk_avg": self.bufs.avg.cpu()}

    def load_state_dict(self, state):
        for k in ("engine", "algo", "delay", "rank", "world", "n_boards", "n_boards_total"):
            mine = {"engine": "board", "algo": self.algo_name}.get(k, getattr(self, k, None))
            if state.get(k) != mine:
                raise ValueError("checkpoint mismatch on %r: file has %r, this solver %r" % (k, state.get(k), mine))
        if tuple(state["regret"].shape) != tuple(self.regret.shape):
            raise ValueError("checkpoint table shape %s != %s" % (tuple(state["regret"].shape), tuple(self.regret.shape)))
        self.iter_counter, self.modes = int(state["iter_counter"]), list(state["modes"])
        self._pending = [0.0, 0.0]  # state_dict() flushes before it exports
        self._avg_due = [-1, -1]
        self.regret.copy_(state["regret"])
        self.avg.copy_(state["avg"])
        self.bufs.regret.copy_(state["trunk_regret"])
        self.bufs.strat.copy_(state["trunk_strat"])
        self.bufs.avg.copy_(state["trunk_avg"])
        with torch.cuda.device(self.device):
            self._reach_trunk(self.bufs, 3, -1, -1, self.modes)
