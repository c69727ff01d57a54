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
from pokerrl_b200 import algorithm
from pokerrl_b200 import dcfr as _dcfr
from pokerrl_b200.game.flat_tree import FlatTree
from pokerrl_b200.game.holdem_boards import BoardSpec
from pokerrl_b200.solver import DeviceTree, TreeBuffers, TreeOps, _require_cuda

SRC_REGRET, SRC_AVG, SRC_AVG_SUM = 0, 1, 2


def board_layout(g=None):
    """prl_board_layout: the per-board blob layout; n_local = nodes of the compiled shape the descriptor `g` names (0 without)"""
    out = (C.c_int32 * 8)()
    nat.call("prl_board_layout", C.byref(g) if g is not None else None, out)
    return dict(n_live=out[0], ldb=out[1], blob=out[2], sh_off=out[3], rows_off=out[4], live_cards=out[5],
                row_pad=out[6], n_local=out[7])


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def supports(game_cls, env_args, algo):
    """True iff the game's abstract tree is one pre-deal trunk + one chance layer + a compiled post-deal shape (Flop5Holdem:
    stacks of 301 chips and more; at 300 and below the preflop raise is all-in and there is no post-deal betting)"""
    if algo not in algorithm.ALL or game_cls.RULES.N_HOLE_CARDS != 2 or game_cls.RULES.N_CARDS_IN_DECK != 52:
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


def shape_rows(g):
    """(row_of[16], rows_per_board) of the compiled shape the descriptor `g` names (prl_board_rows): the board-major row layout"""
    row_of, rpb = (C.c_int32 * 16)(), C.c_int32(0)
    nat.call("prl_board_rows", C.byref(g), row_of, C.byref(rpb))
    return list(row_of), int(rpb.value)


def board_mask(boards):
    mask = np.zeros(boards.shape[0], np.uint64)
    for k in range(boards.shape[1]):
        mask |= (np.uint64(1) << boards[:, k].astype(np.uint64))
    return mask


def build_board_blobs(rules, boards, t_blob, dev):
    """per-board tables of `boards` (int8 [n, 5]) into t_blob[:n]: hand ranks (prl_hand_rank_boards), then
    prl_board_build_tables, 16 384 boards per launch"""
    from pokerrl_b200.hand_eval import hand_rank_all_hands_on_given_boards
    boards = np.ascontiguousarray(boards, np.int8)
    nb = boards.shape[0]
    lut = rules.get_lut_holder()
    t_hc = torch.from_numpy(np.ascontiguousarray(lut.LUT_IDX_2_HOLE_CARDS, np.int8)).to(dev)
    t_mask = torch.from_numpy(board_mask(boards).view(np.int64)).to(dev)
    CH = 16384
    for i in range(0, nb, CH):
        n = min(CH, nb - i)
        ranks = hand_rank_all_hands_on_given_boards(boards[i:i + n], device=dev)
        nat.call("prl_board_build_tables", C.c_void_p(ranks.data_ptr()), C.c_void_p(t_mask[i:i + n].data_ptr()),
                 C.c_void_p(t_hc.data_ptr()), n, C.c_void_p(t_blob[i:i + n].data_ptr()), _stream(dev))


def _decision_locals(st):
    """post-deal decision nodes, ascending local id (the columns of prl_board_policy_query's out_index)"""
    return [i for i in range(st["n_local"]) if st["kind"][i] <= 1 and st["n_children"][i] > 0]


def board_game(st, rules, n_boards, ld, n_sym, grid=0):
    """prl_board_game_t of a post-deal subtree `st` over n_boards boards, without buffers: shape, eq_const, the fixed-point
    format of the chance sums (which depends on n_sym, not on the boards) and the board-major row layout.
    Returns (g, rows_per_board, local_rows = {local child node: (row on board 0, stride per board)})."""
    g = nat.PrlBoardGame()
    _fill_shape(g, st)
    g.n_boards, g.n_range, g.ld, g.n_deck = n_boards, rules.RANGE_SIZE, ld, rules.N_CARDS_IN_DECK
    n_hole = rules.N_HOLE_CARDS
    g.eq_const = math.comb(g.n_deck, n_hole) / math.comb(g.n_deck - n_hole, n_hole)
    # fixed point: |sum| <= n_sym * K * max pot / 2 with headroom; 62 value bits
    bound = max(n_sym, 1) * g.eq_const * max(st["pot"]) * 0.5 * 4.0
    g.frac_bits = 62 - int(math.ceil(math.log2(bound)))
    n_local = st["n_local"]
    dec = _decision_locals(st)
    rows_per_board = sum(st["n_children"][i] for i in dec)
    # board-major rows: everything a (board, seat) unit touches is contiguous - row(i, j) = j * rows_per_board + row_of[i]
    row_of, rpb = shape_rows(g)
    assert rpb == rows_per_board
    local_rows = {}  # local child node -> (row on board 0, stride per board)
    for i in range(n_local):
        g.row0[i], g.row_m[i] = -1, 0
    for d in dec:
        for a in range(st["n_children"][d]):
            c = st["first_child"][d] + a
            g.row0[c], g.row_m[c] = row_of[c], rpb
            local_rows[c] = (int(row_of[c]), rpb)
    g.grid = int(grid) if grid else int(nat.lib().prl_board_grid())
    return g, rows_per_board, local_rows


def row_map(local_rows, ft=None):
    """(src, dst), the prl_board_permute descriptors: for every row of the post-deal decision nodes, {row on board 0, stride
    per board} in the strength-ordered table (src) and in the natural table (dst) - the slot table of the flat tree `ft` over
    a chunk of boards, or without `ft` [boards, rows] with each board's rows in ascending local node order"""
    st = None if ft is None else ft.board_subtree()
    src, dst = [], []
    for k, (i, (r0, m)) in enumerate(sorted(local_rows.items())):
        src += [r0, m]
        dst += [k, len(local_rows)] if ft is None else [int(ft.slot[st["node_base"][i] + st["node_k"][i]]), st["node_m"][i]]
    return src, dst


def _normalised(x, dim, matching):
    """x divided by its sums along `dim` (the actions), uniform where there is nothing to divide: regret matching
    (matching: x clamped at 0, sums > 0) or normalised reach-weighted sums (sums != 0)"""
    if matching:
        x = x.clamp(min=0)
    tot = x.sum(dim=dim, keepdim=True)
    ok = (tot > 0) if matching else (tot != 0)
    return torch.where(ok, x / torch.where(ok, tot, torch.ones_like(tot)), torch.full_like(x, 1.0 / x.shape[dim]))


def _sum_to_one(x, dim):
    """x divided by its sums along `dim` in float64, rounded to x's dtype; uniform where the sum is not positive (the
    fold identity of the restricted Nash response's sweep needs rows that sum to one)"""
    d = x.double()
    tot = d.sum(dim=dim, keepdim=True)
    ok = tot > 0
    return torch.where(ok, d / torch.where(ok, tot, torch.ones_like(tot)), torch.full_like(d, 1.0 / d.shape[dim])).to(x.dtype)


def _decision_row_groups(st, local_rows):
    """for every post-deal decision node, the row indices (on one board) of its children"""
    return [[local_rows[c][0] for c in range(st["first_child"][d], st["first_child"][d] + st["n_children"][d])]
            for d in _decision_locals(st)]


def _trunk_decisions(ft, chance_node):
    """(first slot, actions) of every trunk decision node of the flat tree `ft`"""
    return [(int(ft.first_slot[n]), int(ft.n_children[n])) for n in range(chance_node + 1)
            if ft.kind[n] <= 1 and ft.first_child[n] >= 0]


class _BoardEngine:
    """What the solver and the policy evaluator share: the pre-deal trunk, swept by prl_board_trunk / the level kernels over
    its own small buffers, the descriptor `g` of the post-deal subtrees of the boards, and the one call site of each board
    entry point.  A one-board flat tree carries the trunk and the shape of the post-deal subtree."""

    def _setup(self, game_cls, env_args, spec, n_boards, grid=0):
        """the one-board trunk tree, the suit-symmetry tables of `spec`, the descriptor `g` over n_boards boards with the
        buffers both engines bind, and the size of the game's tree over all the boards of `spec`"""
        dev = self.device
        self.rules = game_cls.RULES
        self.ev_normalizer = game_cls.EV_NORMALIZER
        self.L = board_layout()
        self.ft1 = FlatTree(game_cls, env_args, board_spec=_one_board_spec())
        st = self.ft1.board_subtree()
        if st is None:
            raise ValueError("the game does not have ONE chance layer with a <= 16-node post-deal subtree")
        self.st = st
        self.chance_level = st["chance_level"]
        self.chance_node = st["chance_node"]
        self.R = self.rules.RANGE_SIZE
        # trunk: level sweeps over levels 0 .. chance_level of the one-board tree; the symmetrisation over the suit
        # permutations happens in prl_board_collect / prl_board_trunk (integer sums), not in the level kernels
        self.trunk = DeviceTree(self.ft1, dev)
        self.trunk.desc.n_sym = 0
        self.trunk.desc.sym_perm = None
        self.bufs = TreeBuffers(self.trunk)
        self.ld = self.trunk.ld
        sp = spec.sym_perm
        self.n_sym = 0 if sp is None else int(sp.shape[0])
        self.t_sym = None if sp is None else torch.from_numpy(np.ascontiguousarray(sp, np.int16)).to(dev)
        g, self.rows_per_board, self.local_rows = board_game(st, self.rules, n_boards, self.ld, self.n_sym, grid)
        self.w_private = torch.zeros((g.grid, 2, self.R), dtype=torch.int64, device=dev)
        self._expl = torch.zeros(2, dtype=torch.float32, device=dev)
        g.w_private = self.w_private.data_ptr()
        self.g = g
        nb = self.n_boards_total = int(spec.boards.shape[0])
        self.n_nodes = int(self.ft1.level_start[self.chance_level + 1]) + nb * st["n_local"]
        self.n_nonterm = (int((self.ft1.kind[:self.chance_node + 1] <= nat.KIND_CHANCE).sum())
                          + nb * len(_decision_locals(st)))

    def _setup_boards(self, capacity):
        """the per-board tables, probabilities and multiplicities for `capacity` boards (at least one), bound to `g`"""
        dev, n = self.device, max(capacity, 1)
        self.t_blob = torch.empty((n, self.L["blob"]), dtype=torch.uint8, device=dev)
        self.t_prob = torch.zeros(n, dtype=torch.float32, device=dev)
        self.t_mult = torch.zeros(n, dtype=torch.float32, device=dev)
        g = self.g
        g.tables, g.board_prob, g.board_mult = self.t_blob.data_ptr(), self.t_prob.data_ptr(), self.t_mult.data_ptr()

    def _load_boards(self, boards, prob, mult):
        """`boards` with their probabilities and multiplicities into the first rows of t_blob / t_prob / t_mult, and `g`
        over them"""
        n = boards.shape[0]
        build_board_blobs(self.rules, boards, self.t_blob, self.device)
        self.t_prob[:n].copy_(torch.from_numpy(np.ascontiguousarray(prob, np.float32)))
        self.t_mult[:n].copy_(torch.from_numpy(np.ascontiguousarray(mult, np.float32)))
        self.g.n_boards = n

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

    def _trunk_reach_row(self, bufs, seat):
        return C.c_void_p(bufs.reach.data_ptr() + 4 * (seat * self.trunk.n_nodes + self.chance_node) * self.ld)

    def _reach_trunk(self, bufs, mask, algo, upd_p, modes, t, delay):
        nat.call("prl_reach_levels", C.byref(self.trunk.desc), C.byref(bufs.desc), mask, algo, upd_p, t, delay,
                 nat.modes(*modes), 0, self.chance_level, _stream(self.device))

    @property
    def n_trunk_slots(self):
        """table rows of the trunk: the first slots of every flat tree of the game (its children come before the deal)"""
        return self.ft1.n_slots - self.rows_per_board

    # ------------------------------------------------------------------------------------------------ board entry points
    def _board_sweep(self, bufs, p, evaluate, src_own, src_opp, t, delay, algo, defer_w=0.0, p1_only=0):
        """prl_board_sweep: seat p's update or evaluation sweep of the boards, against the opponent's trunk reach in `bufs`;
        p1_only: the Vanilla / Linear CFR flush of the opponent's pending average contribution of weight defer_w"""
        nat.call("prl_board_sweep", C.byref(self.g), p, int(evaluate), src_own, src_opp, self._trunk_reach_row(bufs, 1 - p),
                 t, delay, algo, defer_w, p1_only, _stream(self.device))

    def _board_trunk(self, bufs, modes, evaluate, p, t, delay, algo, peers=None, n_peers=0, peer_off=0, w_scratch=None):
        """prl_board_trunk: the trunk of seat p's half-iteration, or of an evaluation of both seats into _expl, from the
        chance sums `g` points at (peers: every rank's, summed in the kernel)"""
        nat.call("prl_board_trunk", C.byref(self.g), C.byref(self._trunk_desc(bufs, modes)), int(evaluate), p, self.n_sym,
                 C.c_void_p(self.t_sym.data_ptr()) if self.n_sym else None, t, delay, C.c_void_p(self._expl.data_ptr()), peers,
                 n_peers, peer_off, w_scratch, algo, _stream(self.device))

    def _board_permute(self, tab, nat_tab, to_natural, ft=None, lo=0, hi=None):
        """prl_board_permute: the post-deal rows of boards lo .. hi (default: the boards `g` covers) from the strength-ordered
        table `tab` to the natural table `nat_tab` (to_natural 1) or back (0); nat_tab's layout is that of row_map(ft)"""
        g = self.g
        if hi is not None:
            g = nat.PrlBoardGame.from_buffer_copy(self.g)
            g.n_boards, g.tables = hi - lo, self.t_blob[lo].data_ptr()
        src, dst = (torch.tensor(x, dtype=torch.int64, device=self.device) for x in row_map(self.local_rows, ft))
        nat.call("prl_board_permute", C.byref(g), len(self.local_rows), C.c_void_p(src.data_ptr()), C.c_void_p(dst.data_ptr()),
                 C.c_void_p(tab[lo * self.rows_per_board].data_ptr()), C.c_void_p(nat_tab.data_ptr()), self.ld, to_natural,
                 _stream(self.device))


class BoardCFRSolver(_BoardEngine):
    def __init__(self, game_cls, env_args, board_spec=None, algo="CFRPlus", delay=0, device=None, rank=0, world=1,
                 group=None, grid=0, reduce_fn=None, dcfr=_dcfr.DEFAULT, pcfr_gamma=algorithm.PCFR_GAMMA):
        self.device = _require_cuda(device)
        self.alg = algorithm.Algorithm(algo, delay, dcfr, self.device, pcfr_gamma)
        self.algo_name, self.algo, self.delay, self.dcfr = self.alg.name, self.alg.code, self.alg.delay, self.alg.dcfr
        self._factors = self.alg.factors  # DCFR's / PCFR+'s device table (None for the others), grown by factor_table
        self.rank, self.world, self.group = int(rank), int(world), group
        # cross-rank sum of the fixed-point chance sums, in place; default: torch.distributed all-reduce when world > 1
        self._reduce_fn = reduce_fn
        self.game_cls, self.env_args = game_cls, env_args
        spec = board_spec if board_spec is not None else BoardSpec.full_game(game_cls.RULES)
        self.spec_full = spec
        with torch.cuda.device(self.device):
            self._build(spec, grid)
        self.n_allreduce = 0
        self.reset()

    # ------------------------------------------------------------------------------------------------ construction
    def _build(self, spec, grid):
        dev = self.device
        sel = np.arange(self.rank, spec.boards.shape[0], self.world)
        self.board_ids = sel
        self.boards = np.ascontiguousarray(spec.boards[sel], np.int8)
        nb = self.n_boards = int(sel.size)
        self._setup(self.game_cls, self.env_args, spec, nb, grid)
        self.ops = TreeOps(self.trunk, self.bufs)
        self._eval_bufs = None
        self._setup_boards(nb)
        self._load_boards(self.boards, spec.board_prob[sel], spec.board_mult[sel])
        torch.cuda.synchronize(dev)
        g = self.g
        self.n_rows = nb * self.rows_per_board
        self.regret = torch.zeros((max(self.n_rows, 1), self.L["ldb"]), dtype=torch.float32, device=dev)
        self.avg = torch.zeros_like(self.regret)
        g.regret, g.avg = self.regret.data_ptr(), self.avg.data_ptr()
        # PCFR+ only: the predicted regrets max(R + d, 0) of the post-deal rows, laid out as `regret` (every strategy of its
        # sweeps is regret matching of these rows)
        self.pred = torch.zeros_like(self.regret) if self.algo == nat.ALGO_PCFR_PLUS else None
        g.pred = self.pred.data_ptr() if self.pred is not None else None
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
        g.w_total = self.w_total.data_ptr()
        # the trunk in one launch (prl_board_trunk); PRL_TRUNK=levels keeps the level-kernel chain (A/B, cross-check)
        self.fused_trunk = os.environ.get("PRL_TRUNK", "fused") != "levels"
        # where the level kernels expect the chance node's sums: prl_value_levels(chance_phase 1 / 2), one chance node,
        # one chunk -> W[arr] at float offset (4 + arr) * ld of the workspace
        self._w_off = 4 * self.ld

    # ------------------------------------------------------------------------------------------------ helpers
    def _clear_pending(self):
        """no average-strategy update pending on either seat.
        _pending (Vanilla / Linear CFR, DCFR): weight of the average-strategy contribution of each seat's last update that the
        post-deal rows have not received yet (it is added by the next sweep that walks those rows: csrc/cfr_board.cu, DEFER).
        _avg_due (CFR+): iteration of each seat's averaging step that is still pending (-1: none).  An update sweep with
        nothing pending leaves its step pending; the seat's next update sweep applies it together with its own
        (csrc/cfr_board.cu, AVG): every other sweep of a seat neither reads nor writes the average rows."""
        self._pending = [0.0, 0.0]
        self._avg_due = [-1, -1]

    def _trunk(self, bufs, modes, evaluate, p):
        peers, n_peers, off = None, 0, 0
        if self._symm is not None:
            peers, n_peers, off = C.c_void_p(self._peer_ptrs.data_ptr()), self.world, self._gen * 4 * self.R
        self._board_trunk(bufs, modes, evaluate, p, self.iter_counter, self.delay, self.algo, peers, n_peers, off,
                          C.c_void_p(self.w_scratch.data_ptr()))

    def _board_update_cfrp(self, p, due, now):
        """prl_board_update_cfrp: seat p's CFR+ update sweep of this iteration, writing its averaging step if `now` (else
        leaving it pending) together with the pending step of iteration `due` (-1: none)"""
        nat.call("prl_board_update_cfrp", C.byref(self.g), p, self._trunk_reach_row(self.bufs, 1 - p), self.iter_counter,
                 self.delay, due, now, _stream(self.device))

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

    def _levels(self, bufs, mask, with_br, algo, upd_p, modes, hi, lo, phase):
        nat.call("prl_value_levels", C.byref(self.trunk.desc), C.byref(bufs.desc), mask, int(with_br), algo, upd_p,
                 self.iter_counter, self.delay, nat.modes(*modes), hi, lo, phase, _stream(self.device))

    def _sweep_begin(self, bufs, p, evaluate, src_own, src_opp):
        if not evaluate and self.algo == nat.ALGO_CFR_PLUS:
            t, due = self.iter_counter, self._avg_due[p]
            now = 1 if due >= 0 or t < self.delay else 0  # an iteration before delay has no step to leave pending
            self._avg_due[p] = -1 if now else t
            self._board_update_cfrp(p, due, now)
            return
        defer_w = 0.0
        if not evaluate and self.algo != nat.ALGO_CFR_PLUS:  # this sweep walks the opponent's rows: its pending average goes in
            defer_w, self._pending[1 - p] = self._pending[1 - p], 0.0
        self._board_sweep(bufs, p, evaluate, src_own, src_opp, self.iter_counter, self.delay, self.algo, defer_w)

    def flush_average(self):
        """Applies the average-strategy updates that are still pending: CFR+ averaging steps (prl_board_avg_flush), Vanilla /
        Linear CFR contributions (a light P1-only sweep per seat)"""
        with torch.cuda.device(self.device):
            for q in (0, 1):
                if self._avg_due[q] >= 0:
                    nat.call("prl_board_avg_flush", C.byref(self.g), q, self._avg_due[q], self.delay, _stream(self.device))
                    self._avg_due[q] = -1
                if self._pending[q] != 0.0:
                    self._board_sweep(self.bufs, 1 - q, False, 0, 0, self.iter_counter, self.delay, self.algo,
                                      defer_w=self._pending[q], p1_only=1)
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
        self.g.dcfr = self.alg.factor_table(self.iter_counter + 1)  # DCFR: read by this update's sweep and trunk
        if not self.fused_trunk:
            self._levels(self.bufs, 1 << p, False, self.algo, p, self.modes, cl, cl, 1)
        self._sweep_begin(self.bufs, p, False, SRC_REGRET, SRC_REGRET)

    def _update_end(self, p):
        """second half: cross-rank sum, chance node row, trunk regrets / matching / averaging, trunk reach of p"""
        cl = self.chance_level
        if self.algo != nat.ALGO_CFR_PLUS:  # VanillaCFR.py:56-59 / LinearCFR.py:55-58: weight of this update's strategy in the sums
            if not self.fused_trunk:
                raise RuntimeError("Vanilla / Linear CFR, DCFR and PCFR+ on the board engine need the fused trunk (unset "
                                   "PRL_TRUNK=levels)")
            self._pending[p] = self.alg.sum_weight(self.iter_counter)  # THIS iteration's, whichever later sweep adds it
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
        self._reach_trunk(self.bufs, 1 << p, self.algo, p, self.modes, self.iter_counter, self.delay)

    # ------------------------------------------------------------------------------------------------ schedule
    def reset(self):
        with torch.cuda.device(self.device):
            self.iter_counter = 0
            for t in (self.regret, self.avg, self.bufs.regret, self.bufs.strat, self.bufs.avg):
                t.zero_()
            if self.pred is not None:
                self.pred.zero_()
            self._clear_pending()
            self.modes = [nat.STRAT_UNIFORM64, nat.STRAT_UNIFORM64]
            self._reach_trunk(self.bufs, 3, -1, -1, self.modes, self.iter_counter, self.delay)

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
        else:
            self._levels(bufs, 3, True, -1, -1, modes, cl, cl, 1)
            for p in (0, 1):
                self._sweep(bufs, p, True, src, src)
            self._levels(bufs, 3, True, -1, -1, modes, cl, cl, 2)
            if cl > 0:
                self._levels(bufs, 3, True, -1, -1, modes, cl - 1, 0, 0)
            e = (TreeOps(self.trunk, bufs) if bufs is not self.bufs else self.ops).root_exploitability()
        return algorithm.seat_averaged(e, self.ev_normalizer)

    def exploitability_current(self):
        with torch.cuda.device(self.device):
            return self._evaluate(self.bufs, self.modes, SRC_REGRET)

    def exploitability_average(self):
        # the board engine has no average before the first iteration for any algorithm; the level engine evaluates the
        # still-empty sums of Vanilla / Linear CFR and DCFR as the uniform strategy
        if self.iter_counter == 0:
            raise RuntimeError("no average strategy before the first iteration")
        m, src = {algorithm.SUMS: (nat.STRAT_AVG_SUM, SRC_AVG_SUM), algorithm.CURRENT: (nat.STRAT_F32, SRC_REGRET),
                  algorithm.AVERAGE: (nat.STRAT_AVG_F32, SRC_AVG)}[self.alg.average(self.iter_counter)]
        with torch.cuda.device(self.device):
            if self._eval_bufs is None:
                self._eval_bufs = TreeBuffers(self.trunk, share=self.bufs)
            self.flush_average()
            self._reach_trunk(self._eval_bufs, 3, -1, -1, [m, m], self.iter_counter, self.delay)
            return self._evaluate(self._eval_bufs, [m, m], src)

    # ------------------------------------------------------------------------------------------------ interfaces
    def natural_tables(self, ft):
        """(regret, avg) as natural-order float32 [ft.n_slots, ld] tensors in the slot order of the flat tree `ft` built over
        THIS rank's boards (for agents, exports and parity tests on small instances); PCFR+: (regret, avg, pred), whose trunk
        rows are the trunk's stored strategy (regret matching of its predictions, which the trunk does not keep)."""
        assert ft.board_spec.boards.shape[0] == self.n_boards
        self.flush_average()
        nts, out = self.n_trunk_slots, []
        pairs = [(self.regret, self.bufs.regret), (self.avg, self.bufs.avg)]
        if self.pred is not None:
            pairs.append((self.pred, self.bufs.strat))
        with torch.cuda.device(self.device):
            for tab, trunk_tab in pairs:
                nat_tab = torch.zeros((ft.n_slots, self.ld), dtype=torch.float32, device=self.device)
                self._board_permute(tab, nat_tab, 1, ft)
                nat_tab[:nts] = trunk_tab[:nts]
                out.append(nat_tab)
        return out

    def load_natural_tables(self, ft, regret, avg, pred=None):
        """inverse of natural_tables (teacher forcing in the parity tests, checkpoints written by the level engine); PCFR+
        takes the predictions `pred` too: post-deal rows into `self.pred`, and the trunk's stored strategy becomes regret
        matching of the given trunk rows"""
        if (pred is None) != (self.pred is None):
            raise ValueError("load_natural_tables: predictions are given exactly for PCFR+")
        self._clear_pending()  # the given average is complete
        nts, dev = self.n_trunk_slots, self.device
        triples = [(self.regret, self.bufs.regret, regret), (self.avg, self.bufs.avg, avg)]
        if pred is not None:
            triples.append((self.pred, None, pred))
        with torch.cuda.device(dev):
            for tab, trunk_tab, given in triples:
                nat_tab = torch.zeros((ft.n_slots, self.ld), dtype=torch.float32, device=dev)
                nat_tab[:, :given.shape[1]] = torch.as_tensor(given, dtype=torch.float32).to(dev)
                self._board_permute(tab, nat_tab, 0, ft)
                if trunk_tab is not None:
                    trunk_tab[:nts] = nat_tab[:nts]
                else:
                    self._set_trunk_strategy(nat_tab)

    def set_trunk_strategy_from_regrets(self):
        """after load_natural_tables: the trunk's stored strategy rows = regret matching of its regret rows, reach rows
        refreshed (the post-deal rows need nothing: their strategy is never stored).  PCFR+ sets the trunk's strategy from
        the predictions load_natural_tables was given instead."""
        if self.pred is not None:
            raise RuntimeError("PCFR+: the trunk strategy is regret matching of the predictions given to load_natural_tables")
        self._set_trunk_strategy(self.bufs.regret)

    def _set_trunk_strategy(self, rows):
        """the trunk's stored strategy rows = regret matching of the trunk rows of `rows` (natural slot order), reach rows
        refreshed"""
        ft = self.ft1
        for n in range(self.chance_node + 1):
            if ft.kind[n] <= 1 and ft.first_child[n] >= 0:
                fs, A = int(ft.first_slot[n]), int(ft.n_children[n])
                self.bufs.strat[fs:fs + A] = _normalised(rows[fs:fs + A], 0, True)
        self.modes = [nat.STRAT_F32, nat.STRAT_F32]
        with torch.cuda.device(self.device):
            self._reach_trunk(self.bufs, 3, -1, -1, self.modes, self.iter_counter, self.delay)

    def _identity(self):
        return {"engine": "board", **self.alg.identity(), "rank": self.rank, "world": self.world, "n_boards": self.n_boards,
                "n_boards_total": self.n_boards_total}

    def state_dict(self):
        self.flush_average()
        return {**self._identity(), "iter_counter": self.iter_counter, "modes": list(self.modes),
                "regret": self.regret.cpu(), "avg": self.avg.cpu(),
                "trunk_regret": self.bufs.regret.cpu(), "trunk_strat": self.bufs.strat.cpu(), "trunk_avg": self.bufs.avg.cpu(),
                **({"pred": self.pred.cpu()} if self.alg.code == nat.ALGO_PCFR_PLUS else {})}

    def load_state_dict(self, state):
        algorithm.check_identity(state, self._identity())
        if tuple(state["regret"].shape) != tuple(self.regret.shape):
            raise ValueError("checkpoint table shape %s != %s" % (tuple(state["regret"].shape), tuple(self.regret.shape)))
        self.iter_counter, self.modes = int(state["iter_counter"]), list(state["modes"])
        self._clear_pending()  # state_dict() flushes before it exports
        self.regret.copy_(state["regret"])
        self.avg.copy_(state["avg"])
        if self.alg.code == nat.ALGO_PCFR_PLUS:
            self.pred.copy_(state["pred"])
        self.bufs.regret.copy_(state["trunk_regret"])
        self.bufs.strat.copy_(state["trunk_strat"])
        self.bufs.avg.copy_(state["trunk_avg"])
        with torch.cuda.device(self.device):
            self._reach_trunk(self.bufs, 3, -1, -1, self.modes, self.iter_counter, self.delay)


def rnr_probability(p):
    """the model's probability of a restricted Nash response as float32, ValueError unless it is finite and in [0, 1]"""
    p = float(p)
    if not (math.isfinite(p) and 0.0 <= p <= 1.0):
        raise ValueError("the model's probability p must be a finite number in [0, 1], got %r" % p)
    return float(np.float32(p))


def rnr_identity(seat, p, model_digest):
    """the checkpoint keys a restricted Nash response game adds to CFR+'s"""
    return {"rnr_seat": int(seat), "rnr_p": float(p), "rnr_model": model_digest}


def device_digest(tensors):
    """an integer digest of the bits of float32 device tensors, computed on the device in chunks"""
    acc, mask = 0, (1 << 61) - 1
    for k, t in enumerate(tensors):
        flat = t.reshape(-1).view(torch.int32)
        for a in range(0, flat.numel(), 1 << 24):
            v = flat[a:a + (1 << 24)].to(torch.int64)
            w = torch.arange(a + 1, a + 1 + v.numel(), dtype=torch.int64, device=t.device) * 2654435761 + k
            acc = (acc * 1000003 + int((v * w).sum())) & mask
    return acc


class BoardRNRSolver(BoardCFRSolver):
    """One game of a restricted Nash response (Johanson, Zinkevich & Bowling, "Computing Robust Counter-Strategies", NIPS
    2007) on the board engine: seat `seat` (the exploiter) plays against an opponent that is, with probability p drawn before
    the deal and seen only by the opponent, a fixed model, and otherwise a free strategy.  Both learn by CFR+ (delay as
    CFRPlus).  The exploiter's values are linear in the opponent's reach, so its update is CFR+'s against the mixed reach
    (1 - p) * free + p * model:
      * the model's reach at every board's showdown terminals, trunk reach and deal included, is computed once
        (`model_reach`, float32 [n_boards * n_sd, 1088], BoardPolicyEvaluator.model_reach) and never changes; the sweep adds
        p times it to the free copy's, whose trunk reach row the host scales by 1 - p (prl_board_sweep, rnr_reach);
      * the trunk mixes the opponent's reach at its fold terminals with the model's trunk reach (`trunk_model`).
    The free copy's update is CFR+'s unchanged: its counterfactual values are 1 - p times those it computes, which scales its
    regrets by a constant and leaves regret matching as it is.  At p = 1 it is skipped; at p = 0 the exploiter runs the plain
    CFR+ sweep and trunk.  The model's tables are filled by the owner (RestrictedNashResponse) before the first iteration."""

    def __init__(self, game_cls, env_args, seat, p, board_spec=None, delay=0, device=None, grid=0, share_boards=None):
        """share_boards: another BoardRNRSolver over the same board spec and device whose per-board tables (blobs, deal
        probabilities, multiplicities; read-only after set-up) this one uses instead of building its own"""
        if seat not in (0, 1):
            raise ValueError("the exploiter's seat is 0 or 1")
        self.seat, self.p = int(seat), rnr_probability(p)
        if self.p > 0.0 and os.environ.get("PRL_TRUNK", "fused") == "levels":
            # the level-kernel trunk has no mixed form: the exploiter's trunk regrets would ignore the model
            raise ValueError("the restricted Nash response needs the fused trunk (unset PRL_TRUNK=levels)")
        self._q = float(np.float32(1.0) - np.float32(self.p))  # 1 - p as the trunk kernel computes it
        self._rnr_trunk = False
        self._share = share_boards
        super().__init__(game_cls, env_args, board_spec, algo="CFRPlus", delay=delay, device=device, grid=grid)
        dev = self.device
        self.n_sd = sum(1 for k in self.st["kind"][:self.st["n_local"]] if k == nat.KIND_SHOWDOWN)
        self.model_reach = torch.zeros((max(self.n_boards * self.n_sd, 1), self.L["ldb"]), dtype=torch.float32, device=dev)
        self.trunk_model = torch.zeros_like(self.bufs.reach)
        self.model_digest = None
        self._opp_row = torch.zeros(self.ld, dtype=torch.float32, device=dev)  # the free copy's trunk reach row times 1 - p
        self._expl = torch.zeros(6, dtype=torch.float32, device=dev)  # prl_trunk_t.reach_model: the evaluation's root values

    def _setup_boards(self, capacity):
        if self._share is None:
            return super()._setup_boards(capacity)
        sh = self._share
        if sh.n_boards != capacity or not np.array_equal(sh.boards, self.boards) or sh.device != self.device:
            raise ValueError("share_boards: another board spec or device")
        self.t_blob, self.t_prob, self.t_mult = sh.t_blob, sh.t_prob, sh.t_mult
        self.g.tables, self.g.board_prob, self.g.board_mult = sh.g.tables, sh.g.board_prob, sh.g.board_mult

    def _load_boards(self, boards, prob, mult):
        if self._share is None:
            return super()._load_boards(boards, prob, mult)
        self.g.n_boards = boards.shape[0]  # the shared tables are built

    def set_model(self, trunk_model):
        """after model_reach is filled: the model's trunk reach rows, and the digest that names the model in checkpoints"""
        self.trunk_model.copy_(trunk_model)
        with torch.cuda.device(self.device):
            self.model_digest = device_digest([self.model_reach, self.trunk_model])

    def _rnr_game(self, p):
        g = nat.PrlBoardGame.from_buffer_copy(self.g)
        g.rnr_reach, g.rnr_p = self.model_reach.data_ptr(), p
        return g

    def _skipped(self, p):
        return p != self.seat and self.p == 1.0  # the free copy never plays

    def _board_update_cfrp(self, p, due, now):
        if p != self.seat or self.p == 0.0:
            return super()._board_update_cfrp(p, due, now)
        free = self.bufs.reach.view(2, -1, self.ld)[1 - p, self.chance_node]
        torch.mul(free, self._q, out=self._opp_row)
        nat.call("prl_board_update_cfrp", C.byref(self._rnr_game(self.p)), p, C.c_void_p(self._opp_row.data_ptr()),
                 self.iter_counter, self.delay, due, now, _stream(self.device))

    def _trunk(self, bufs, modes, evaluate, p):
        self._rnr_trunk = not evaluate and p == self.seat and self.p > 0.0
        try:
            super()._trunk(bufs, modes, evaluate, p)
        finally:
            self._rnr_trunk = False

    def _trunk_desc(self, bufs, modes):
        t = super()._trunk_desc(bufs, modes)
        if self._rnr_trunk:
            t.reach_model, t.rnr_p = self.trunk_model.data_ptr(), self.p
        return t

    def _update_begin(self, p):
        if not self._skipped(p):
            super()._update_begin(p)

    def _update_end(self, p):
        if not self._skipped(p):
            super()._update_end(p)

    def rnr_values(self):
        """(exploitation, exploitability) of the exploiter's average strategy in chips: its value against the model, and the
        value of a best response of the other seat to it (prl_board_sweep with rnr_reach at rnr_p = 1 for the first, the
        plain evaluation sweep of the other seat for the second, one prl_board_trunk evaluation with reach_model for both)"""
        if self.model_digest is None:
            raise RuntimeError("the model's tables are not set")
        if self.iter_counter == 0:
            raise RuntimeError("no average strategy before the first iteration")
        m, src = {algorithm.CURRENT: (nat.STRAT_F32, SRC_REGRET),
                  algorithm.AVERAGE: (nat.STRAT_AVG_F32, SRC_AVG)}[self.alg.average(self.iter_counter)]
        s, o = self.seat, 1 - self.seat
        with torch.cuda.device(self.device):
            if self._eval_bufs is None:
                self._eval_bufs = TreeBuffers(self.trunk, share=self.bufs)
            self.flush_average()
            bufs = self._eval_bufs
            self._reach_trunk(bufs, 3, -1, -1, [m, m], self.iter_counter, self.delay)
            bufs.reach[o].copy_(self.trunk_model[o])  # the exploiter's opponent is the model
            self._opp_row.zero_()  # the model's reach is all in model_reach
            nat.call("prl_board_sweep", C.byref(self._rnr_game(1.0)), s, 1, src, src, C.c_void_p(self._opp_row.data_ptr()),
                     self.iter_counter, self.delay, nat.ALGO_CFR_PLUS, 0.0, 0, _stream(self.device))
            self._board_sweep(bufs, o, True, src, src, self.iter_counter, self.delay, nat.ALGO_CFR_PLUS)
            self._reduce(self.w_total)
            self._rnr_trunk = True
            try:
                self._board_trunk(bufs, [m, m], True, -1, self.iter_counter, self.delay, nat.ALGO_CFR_PLUS)
            finally:
                self._rnr_trunk = False
            self._next_generation()
            e = self._expl.cpu().numpy().astype(np.float64)
        return float(e[2 + s]), float(e[4 + o])

    def _identity(self):
        return {**super()._identity(), **rnr_identity(self.seat, self.p, self.model_digest)}


# ==================================================================================================================== policy evaluation
def board_keys(boards):
    """int64 key of each board: its sorted cards packed base 64 (holdem_boards.canonical_boards)"""
    b = np.sort(np.asarray(boards, np.int64), axis=1)
    key = np.zeros(b.shape[0], np.int64)
    for i in range(b.shape[1]):
        key = key * 64 + b[:, i]
    return key


def abstract_fingerprint(ft):
    """identity of the betting structure of a flat tree (any board spec): kinds, actions, pots and fan-outs of its abstract
    nodes - equal for every spec of one game and stack"""
    import hashlib
    a = np.array([(n.kind, n.action, n.pot, len(n.children), n.parent, n.acted_last) for n in ft.abs_nodes], np.int64)
    return hashlib.sha1(a.tobytes()).hexdigest()


class BoardPolicyEvaluator(_BoardEngine):
    """Exploitability of an agent's strategy on a game the board engine supports (single GPU), with the strategy supplied
    chunk by chunk over the boards of a BoardSpec, so that it never has to exist for the whole game at once.

    Spec: default = the game's suit-isomorphism classes, the semantics of PublicTree (the agent is queried on the
    representatives, which is exact for suit-symmetric agents); BoardSpec.full_game(rules, isomorphic=False) = every deal
    (2 598 960 boards in Flop5Holdem), exact for any agent.

    Per chunk of boards: a structure-only PublicTree over the chunk's slice of the spec is filled from the agent
    (PublicTree.agent_strategy_table: one batched get_a_probs_for_public_tree, or one get_a_probs_for_each_hand call per decision
    node - about 807 k calls over the 134 459 classes, slow but supported; float64 answers are rounded to float32), the boards'
    tables are built (build_board_blobs), the post-deal rows are moved into each board's strength order (prl_board_permute) and
    the evaluation sweep of each seat runs on them as they are (prl_board_sweep, src 1).  Its fixed-point chance sums are added
    into an int64 accumulator: integer addition makes the result independent of the chunking.  The trunk's rows come from the
    first chunk's answers (mode STRAT_AVG_F32) and its reach pass runs before the first sweep, which reads the opponent's reach
    at the chance node.  After the last chunk one prl_board_trunk evaluation gives the exploitability of each seat.

    Device memory is chunk-sized, allocated once:  chunk * bytes_per_board  with
        bytes_per_board = blob (15 392) + strength-ordered rows (rows_per_board * 1088 * 4)
                          + slot-table rows (rows_per_board * ld * 4) + the batched answers (n_dec * 1326 * N_ACTIONS * 4)
                          + hand ranks (1326 * 4)
    (Flop5Holdem, ld 1328, 3 actions: 245 KB per board at stacks of 901 chips and more - 14 rows, 6 decision nodes -, 158 KB
    at 301 to 900 chips - 8 rows, 4 decision nodes), plus the trunk and the chance sums.
    Default chunk = min(65 536, n_boards, free device memory / 2 / bytes_per_board)."""

    MAX_CHUNK = 65536

    def __init__(self, env_bldr, stack_size=None, board_spec=None, chunk=None, device=None):
        self.device = dev = _require_cuda(device)
        self.env_bldr, self.stack_size = env_bldr, stack_size
        game_cls = env_bldr.env_cls
        self.env_args = env_bldr.args_for_stack(stack_size)
        self.spec = board_spec if board_spec is not None else BoardSpec.full_game(game_cls.RULES)
        n_actions = env_bldr.N_ACTIONS
        with torch.cuda.device(dev):
            self._setup(game_cls, self.env_args, self.spec, 0)
            L, rpb, g = self.L, self.rows_per_board, self.g
            n_dec = len(_decision_locals(self.st))
            self.bytes_per_board = (L["blob"] + rpb * L["ldb"] * 4 + rpb * self.ld * 4 + n_dec * self.R * n_actions * 4
                                    + self.R * 4)
            if chunk is None:
                free, _ = torch.cuda.mem_get_info(dev)
                chunk = min(self.MAX_CHUNK, free // 2 // self.bytes_per_board)
            self.chunk = max(1, min(int(chunk), self.n_boards_total))
            n = self.chunk
            self._setup_boards(n)
            self.rows = torch.zeros((n * rpb, L["ldb"]), dtype=torch.float32, device=dev)
            self.nat_tab = torch.zeros((self.n_trunk_slots + n * rpb, self.ld), dtype=torch.float32, device=dev)
            self.w_total = torch.zeros((4, self.R), dtype=torch.int64, device=dev)
            self.w_acc = torch.zeros_like(self.w_total)
            # evaluation with src 1 reads the strategy rows as they are and never the regrets: one table serves both
            g.regret = g.avg = self.rows.data_ptr()
            g.w_total = self.w_total.data_ptr()
        self.times = {}

    def _chunk_tree(self, lo, hi):
        from pokerrl_b200.game.PublicTree import PublicTree
        s = self.spec
        spec = BoardSpec(s.boards[lo:hi], s.board_prob[lo:hi], s.board_mult[lo:hi], s.sym_perm,
                         "boards %d .. %d of: %s" % (lo, hi, s.note))
        pt = PublicTree(self.env_bldr, self.stack_size, stop_at_street=None, put_out_new_round_after_limit=True,
                        device=self.device, board_spec=spec)
        pt.build_structure()
        return pt

    def _chunks(self, agent, tick, normalise=False):
        """the agent's strategy over the spec, chunk by chunk: for the boards lo .. hi of each chunk (yielded with the time
        tick() last returned), their tables bound to `g` and the agent's post-deal rows in self.rows, strength order; from the
        first chunk on, the trunk's rows in bufs.avg and the reach of both seats in bufs.reach.  normalise: every decision
        node's rows divided by their sum in float64, then rounded to float32 (a model that the fold identity of the sweep
        holds for), where the sum is positive"""
        import time
        R, s, nts = self.R, self.spec, self.n_trunk_slots
        for lo in range(0, self.n_boards_total, self.chunk):
            hi = min(lo + self.chunk, self.n_boards_total)
            t0 = time.perf_counter()
            pt = self._chunk_tree(lo, hi)
            ft = pt.flat
            tab = self.nat_tab[:ft.n_slots]
            got = pt.agent_strategy_table(agent, out=tab)
            if not isinstance(got, torch.Tensor):  # answered node by node on the host
                tab[:, :R].copy_(torch.from_numpy(np.ascontiguousarray(got, np.float32)))
            t0 = tick("agent query", t0)
            self._load_boards(s.boards[lo:hi], s.board_prob[lo:hi], s.board_mult[lo:hi])
            self._board_permute(self.rows, tab, 0, ft)
            if normalise:
                rows = self.rows[:(hi - lo) * self.rows_per_board].view(hi - lo, self.rows_per_board, -1)[:, :, :self.L["n_live"]]
                for idx in _decision_row_groups(self.st, self.local_rows):
                    rows[:, idx] = _sum_to_one(rows[:, idx], 1)
            if lo == 0:  # the trunk's rows, then its reach: the sweeps read the opponent's reach at the chance node
                self.bufs.avg[:nts].copy_(tab[:nts])
                if normalise:
                    for fs, A in _trunk_decisions(self.ft1, self.chance_node):
                        self.bufs.avg[fs:fs + A, :R] = _sum_to_one(self.bufs.avg[fs:fs + A, :R], 0)
                self._reach_trunk(self.bufs, 3, -1, -1, [nat.STRAT_AVG_F32, nat.STRAT_AVG_F32], 0, 0)
            t0 = tick("table build", t0)
            yield lo, hi, t0
            del pt

    def model_reach(self, agent, tables):
        """restricted Nash response: for every {seat s: float32 [n_boards_total * n_sd, 1088] table}, the reach of `agent`
        playing seat 1 - s at the showdown terminals of every board of the spec (prl_board_sweep, p1_only with rnr_reach),
        in one pass over the agent's answers; returns the agent's trunk reach rows (float32 [2, nodes, ld], a copy)"""
        n_sd = sum(1 for k in self.st["kind"][:self.st["n_local"]] if k == nat.KIND_SHOWDOWN)
        with torch.cuda.device(self.device):
            for lo, hi, _ in self._chunks(agent, lambda key, t0: t0, normalise=True):
                for seat, F in tables.items():
                    g = nat.PrlBoardGame.from_buffer_copy(self.g)
                    g.rnr_reach, g.rnr_p = F[lo * n_sd].data_ptr(), 1.0
                    nat.call("prl_board_sweep", C.byref(g), seat, 0, SRC_AVG, SRC_AVG,
                             self._trunk_reach_row(self.bufs, 1 - seat), 0, 0, nat.ALGO_CFR_PLUS, 0.0, 1, _stream(self.device))
            return self.bufs.reach.clone()

    def evaluate(self, agent, profile=False):
        """exploitability of each seat in chips, numpy float64 [2] (the analogue of PublicTree's root.exploitability).
        profile=True synchronises between the phases and leaves their wall times (s) in self.times."""
        return self._evaluate(agent, profile)

    def best_response(self, agent, profile=False):
        """(exploitability, tables): evaluate(agent)'s numbers, bit for bit, and the best response to `agent` at both seats as a
        BoardPolicyTables (seat s's rows = seat s's best response).  Each evaluation sweep writes one-hot rows of its seat's
        best-response actions into one table over the whole spec (prl_board_sweep with br_out); the trunk's rows are one-hot
        rows of the best-response values the trunk evaluation leaves in bufs.ev_br.  At every node the action is the FIRST
        child in child order whose best-response value is the maximum (np.argmax; PublicTree's br_a_idx_in_child_arr_for_each_hand).
        Raises ValueError before allocating when the table and its position -> hand rows do not fit in free device memory
        (best_response_bytes: 8.19 GB + 291 MB for the 134 459 classes at stacks of 901 chips and more)."""
        import hashlib
        nb, rpb, L, dev = self.n_boards_total, self.rows_per_board, self.L, self.device
        need = best_response_bytes(nb, rpb)
        with torch.cuda.device(dev):
            free, _ = torch.cuda.mem_get_info(dev)
            check_best_response_fits(need, free + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev))
            rows = torch.empty((nb * rpb, L["ldb"]), dtype=torch.float32, device=dev)
            pos_hand = torch.empty((nb, L["n_live"]), dtype=torch.int16, device=dev)
            e = self._evaluate(agent, profile, rows, pos_hand)
            ft, nts, R = self.ft1, self.n_trunk_slots, self.R
            trunk = torch.zeros((nts, self.ld), dtype=torch.float32, device=dev)
            for n in range(self.chance_node + 1):
                if ft.kind[n] <= 1 and ft.first_child[n] >= 0:
                    fs, fc, A = int(ft.first_slot[n]), int(ft.first_child[n]), int(ft.n_children[n])
                    trunk[fs:fs + A, :R] = first_max_onehot(self.bufs.ev_br[int(ft.kind[n]), fc:fc + A, :R], 0)
            keys = board_keys(self.spec.boards)
            if np.any(np.diff(keys) <= 0):  # rows by ascending key, as BoardPolicyTables.from_solver
                perm = np.argsort(keys, kind="stable")
                t_perm = torch.from_numpy(perm).to(dev)
                rows = rows.view(nb, rpb, -1)[t_perm].reshape(nb * rpb, -1)
                pos_hand = pos_hand[t_perm]
                keys = keys[perm]
            t_keys = torch.from_numpy(keys).to(dev)
        spec_id = (int(nb), self.n_sym > 0, hashlib.sha1(keys.tobytes()).hexdigest())
        return e, BoardPolicyTables(rows, t_keys, pos_hand, trunk, self.n_sym > 0, _packed_actions(self.ft1, self.st),
                                    abstract_fingerprint(self.ft1), spec_id)

    def _evaluate(self, agent, profile, br_rows=None, pos_hand=None):
        """evaluate(); br_rows / pos_hand (best_response): the tables the sweeps export into, over the whole spec"""
        import time
        dev = self.device
        times = {"agent query": 0.0, "table build": 0.0, "sweeps": 0.0}
        modes = [nat.STRAT_AVG_F32, nat.STRAT_AVG_F32]

        def tick(key, t0):
            if profile:
                torch.cuda.synchronize(dev)
                t1 = time.perf_counter()
                times[key] += t1 - t0
                return t1
            return t0

        with torch.cuda.device(dev):
            self.w_acc.zero_()
            try:
                for lo, hi, t0 in self._chunks(agent, tick):
                    if br_rows is not None:
                        self.g.br_out = br_rows[lo * self.rows_per_board].data_ptr()
                        sh = self.L["sh_off"]
                        pos_hand[lo:hi] = self.t_blob[:hi - lo, sh:sh + 2 * self.L["n_live"]].contiguous().view(torch.int16)
                    for p in (0, 1):  # prl_board_sweep zeroes the arrays it writes at every launch: accumulate outside
                        self._board_sweep(self.bufs, p, True, SRC_AVG, SRC_AVG, 0, 0, nat.ALGO_CFR_PLUS)
                        self.w_acc[2 * p:2 * p + 2] += self.w_total[2 * p:2 * p + 2]
                    tick("sweeps", t0)
            finally:
                self.g.br_out = None
            t0 = time.perf_counter()
            self.w_total.copy_(self.w_acc)
            self._board_trunk(self.bufs, modes, True, -1, 0, 0, nat.ALGO_CFR_PLUS)
            e = self._expl.cpu().numpy().astype(np.float64)
            tick("sweeps", t0)
        self.times = times
        return e


def best_response_bytes(n_boards, rows_per_board):
    """device bytes of BoardPolicyEvaluator.best_response's tables: the strength-ordered rows (1088 floats per row) and the
    int16 position -> hand rows (1081 per board)"""
    return n_boards * rows_per_board * 1088 * 4 + n_boards * 1081 * 2


def check_best_response_fits(need, free):
    """ValueError, with the byte counts, when `need` bytes of best-response tables exceed `free` device bytes"""
    if need > free:
        raise ValueError("the best-response tables of this spec need %d bytes (%.2f GB) of device memory, %d bytes (%.2f GB) "
                         "are free" % (need, need / 1e9, free, free / 1e9))


def first_max_onehot(v, dim):
    """float32 one-hot of the FIRST index along `dim` whose entry equals the maximum (np.argmax's rule), same shape as v"""
    m = v.amax(dim=dim, keepdim=True)
    n = v.shape[dim]
    idx = torch.zeros_like(m, dtype=torch.int64)
    for c in reversed(range(n)):
        idx = torch.where(v.narrow(dim, c, 1) == m, c, idx)
    shape = [1] * v.dim()
    shape[dim] = n
    return (torch.arange(n, device=v.device).view(shape) == idx).to(torch.float32)


class BoardPolicyTables:
    """A board-engine strategy as an agent's own tables, independent of the solver that computed it:
      rows      float32 [n_cls * rows_per_board, 1088]  strength-ordered post-deal rows (the solver's board-major layout)
      keys      int64   [n_cls]                          ascending class keys (board_keys of the representatives)
      pos_hand  int16   [n_cls, 1081]                    strength position -> hand, cut from the boards' tables
      trunk     float32 [n_trunk_slots, ld]              trunk rows, natural hand order
    iso: the spec holds suit-isomorphism classes (queries are canonicalised), else raw boards.  Answers for the decision nodes
    of any flat tree of the game (any board spec, either engine) through prl_board_policy_query.  The post-deal shape is that of
    the game and stack the tables were computed on: rows_per_board = rows.shape[0] / n_cls tells it apart."""

    def __init__(self, rows, keys, pos_hand, trunk, iso, actions, fingerprint, spec_id):
        self.rows, self.keys, self.pos_hand, self.trunk = rows, keys, pos_hand, trunk
        self.iso, self.actions, self.fingerprint, self.spec_id = bool(iso), int(actions), fingerprint, spec_id
        self.n_cls = int(keys.shape[0])
        self.rows_per_board = int(rows.shape[0]) // self.n_cls

    @classmethod
    def from_solver(cls, s):
        """the average strategy of a single-GPU BoardCFRSolver: CFR+ after iteration delay + 1 the average rows as they are, at
        delay + 1 regret matching of the regret rows (CFRPlus.py:83-84); Vanilla / Linear CFR the normalised reach-weighted sums
        with the uniform fallback (LinearCFR.py:64-71)"""
        import hashlib
        if s.world != 1:
            raise ValueError("a sharded solver holds only its rank's boards")
        s.flush_average()
        avg = s.alg.average(s.iter_counter)
        nb, rpb, st = s.n_boards, s.rows_per_board, s.st
        groups = _decision_row_groups(st, s.local_rows)
        with torch.cuda.device(s.device):
            if avg == algorithm.AVERAGE:
                rows = s.avg.clone()
            else:
                matching = avg == algorithm.CURRENT  # regret matching at delay + 1, else normalised sums
                rows = torch.empty_like(s.avg)
                src = (s.regret if matching else s.avg).view(nb, rpb, -1)
                dst = rows.view(nb, rpb, -1)
                for lo in range(0, nb, 8192):
                    hi = min(lo + 8192, nb)
                    for idx in groups:
                        dst[lo:hi, idx] = _normalised(src[lo:hi, idx], 1, matching)
            nts, ft = s.n_trunk_slots, s.ft1
            if avg != algorithm.SUMS:
                trunk = (s.bufs.strat if avg == algorithm.CURRENT else s.bufs.avg)[:nts].clone()
            else:
                a = s.bufs.avg[:nts]
                trunk = torch.zeros_like(a)
                for n in range(s.chance_node + 1):
                    if ft.kind[n] <= 1 and ft.first_child[n] >= 0:
                        fs, A = int(ft.first_slot[n]), int(ft.n_children[n])
                        trunk[fs:fs + A] = _normalised(a[fs:fs + A], 0, False)
            L = s.L
            pos_hand = s.t_blob[:nb, L["sh_off"]:L["sh_off"] + 2 * L["n_live"]].contiguous().view(torch.int16)
            keys = board_keys(s.boards)
            if np.any(np.diff(keys) <= 0):  # a spec in another order: rows by ascending key
                perm = np.argsort(keys, kind="stable")
                t_perm = torch.from_numpy(perm).to(s.device)
                rows = rows.view(nb, rpb, -1)[t_perm].reshape(nb * rpb, -1)
                pos_hand = pos_hand[t_perm]
                keys = keys[perm]
            t_keys = torch.from_numpy(keys).to(s.device)
        spec_id = (int(nb), s.n_sym > 0, hashlib.sha1(keys.tobytes()).hexdigest())
        return cls(rows, t_keys, pos_hand, trunk, s.n_sym > 0, _packed_actions(s.ft1, st), abstract_fingerprint(s.ft1),
                   spec_id)

    # ---- queries
    def _check(self, ft):
        if abstract_fingerprint(ft) != self.fingerprint:
            raise ValueError("this agent's tables were computed on a different betting tree (game / stack / bet set)")

    def _query(self, st, boards, out_index, out, n_actions):
        g = nat.PrlBoardGame()
        _fill_shape(g, st)
        if shape_rows(g)[1] != self.rows_per_board:
            raise ValueError("this agent's tables hold %d rows per board, the queried tree's post-deal shape has %d"
                             % (self.rows_per_board, shape_rows(g)[1]))
        dev = out.device
        miss = torch.zeros(1, dtype=torch.int32, device=dev)
        t_b = torch.from_numpy(np.ascontiguousarray(boards, np.int8)).to(dev)
        t_i = torch.from_numpy(np.ascontiguousarray(out_index, np.int32)).to(dev)
        with torch.cuda.device(dev):
            nat.call("prl_board_policy_query", C.byref(g), C.c_void_p(self.rows.data_ptr()), C.c_void_p(self.keys.data_ptr()),
                     C.c_void_p(self.pos_hand.data_ptr()), self.n_cls, int(self.iso), C.c_void_p(t_b.data_ptr()), int(t_b.shape[0]),
                     C.c_void_p(t_i.data_ptr()), self.actions, n_actions, C.c_void_p(out.data_ptr()), C.c_void_p(miss.data_ptr()),
                     _stream(dev))
        if int(miss.item()):
            raise ValueError("a queried board is not in this agent's board spec (%s)"
                             % ("suit classes" if self.iso else "boards without isomorphism"))

    def answer_tree(self, ft, n_actions):
        """float32 [n_decision, R, n_actions] on the tables' device for every decision node of `ft` in flat order"""
        self._check(ft)
        dev = self.rows.device
        dec = np.nonzero((ft.kind <= nat.KIND_P1) & (ft.first_child >= 0))[0]
        dec_idx = np.full(ft.n_nodes, -1, np.int64)
        dec_idx[dec] = np.arange(dec.size)
        out = torch.empty((dec.size, ft.R, n_actions), dtype=torch.float32, device=dev)
        for n in dec[ft.cdepth[dec] == 0]:
            self._trunk_node(ft, n, out[dec_idx[n]])
        st = ft.board_subtree()
        nb = int(st["n_boards_local"])
        J = np.arange(nb, dtype=np.int64)
        locs = _decision_locals(st)
        idx = np.full((nb, len(locs)), -1, np.int64)
        for d, i in enumerate(locs):
            idx[:, d] = dec_idx[st["node_base"][i] + J * st["node_m"][i] + st["node_k"][i]]
        self._query(st, ft.board_spec.boards, idx, out, n_actions)
        return out

    def answer_node(self, ft, n, n_actions):
        """numpy float32 [R, n_actions] at decision node n of `ft` (the one-node form of answer_tree)"""
        self._check(ft)
        out = torch.empty((1, ft.R, n_actions), dtype=torch.float32, device=self.rows.device)
        if ft.cdepth[n] == 0:
            self._trunk_node(ft, n, out[0])
            return out[0].cpu().numpy()
        st = ft.board_subtree()
        j = int(ft.board[n]) - int(st["first_board"])
        locs = _decision_locals(st)
        idx = np.full((1, len(locs)), -1, np.int64)
        for d, i in enumerate(locs):
            if st["node_base"][i] + j * st["node_m"][i] + st["node_k"][i] == n:
                idx[0, d] = 0
        assert (idx == 0).sum() == 1, "not a post-deal decision node"
        self._query(st, ft.board_spec.boards[j:j + 1], idx, out, n_actions)
        return out[0].cpu().numpy()

    def _trunk_node(self, ft, n, out):
        fs, fc, A = int(ft.first_slot[n]), int(ft.first_child[n]), int(ft.n_children[n])
        out.zero_()
        out[:, torch.from_numpy(ft.action[fc:fc + A].astype(np.int64)).to(out.device)] = self.trunk[fs:fs + A, :ft.R].T

    # ---- state
    def state_dict(self):
        return {"rows": self.rows.cpu(), "keys": self.keys.cpu(), "pos_hand": self.pos_hand.cpu(), "trunk": self.trunk.cpu(),
                "iso": self.iso, "actions": self.actions, "fingerprint": self.fingerprint, "spec_id": self.spec_id}

    @classmethod
    def from_state(cls, state, device=None):
        dev = _require_cuda(device)
        return cls(*(state[k].to(dev) for k in ("rows", "keys", "pos_hand", "trunk")), state["iso"], state["actions"],
                   state["fingerprint"], state["spec_id"])


def _packed_actions(ft, st):
    """discrete action of every post-deal local node (as a child) in 4 bits per node, board 0 of `ft`"""
    act = 0
    for i in range(1, st["n_local"]):
        a = int(ft.action[st["node_base"][i] + st["node_k"][i]])
        assert 0 <= a < 16
        act |= a << (4 * i)
    return act
