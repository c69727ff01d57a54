"""Multi-GPU CFR for two-card games: public-chance subtrees (boards) sharded over the ranks of one node.

SURVEY.md §8(e): below a chance node the board subtrees are independent given the parent's reach rows
(`StrategyFiller.py:137-140`) and contribute additively to the parent's values (`ValueFiller.py:76-78`).  Every rank
(one process per GPU, `torch.distributed` / NCCL over NVLink) owns the regret / average tables and node vectors of ITS
boards and a replica of the tiny pre-deal trunk.  Top-down sweeps need no communication; in a bottom-up sweep each rank
reduces its boards into the per-chance-node sums W (board_mult-weighted) and ONE all-reduce(sum) of W - [4][n_chance][ld]
floats, 21 KB per chance node and seat - makes the trunk values identical on all ranks, which then update the trunk
regrets redundantly.  Nothing else crosses GPUs.
"""
import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from pokerrl_b200 import _native as nat
from pokerrl_b200 import algorithm
from pokerrl_b200 import dcfr as _dcfr
from pokerrl_b200.game.flat_tree import FlatTree
from pokerrl_b200.game.holdem_boards import BoardSpec
from pokerrl_b200.solver import CFRSolver, _on, _stream


def shard_board_spec(spec, rank, world):
    """boards rank, rank + world, ... of the FIRST chance layer of `spec` (every board subtree has the same cost, so
    round-robin balances); deeper layers follow their parents"""
    from pokerrl_b200.game.holdem_boards import MultiStreetBoards
    if isinstance(spec, MultiStreetBoards):
        boards, parents, prob, mult = [spec.boards[0]], [spec.parents[0]], [spec.prob[0]], [spec.mult[0]]
        keep = np.arange(rank, spec.boards[1].shape[0], world)
        new_parent = np.zeros(keep.size, np.int32)
        for c in range(1, spec.n_layers + 1):
            if c > 1:
                old = spec.parents[c]
                remap = np.full(spec.boards[c - 1].shape[0], -1, np.int64)
                remap[prev_keep] = np.arange(prev_keep.size)
                keep = np.nonzero(remap[old] >= 0)[0]
                new_parent = remap[old[keep]].astype(np.int32)
            boards.append(spec.boards[c][keep])
            parents.append(new_parent)
            prob.append(spec.prob[c][keep])
            mult.append(spec.mult[c][keep])
            prev_keep = keep
        return MultiStreetBoards(boards, parents, prob, mult, "%s; shard %d/%d" % (spec.note, rank, world))
    sel = np.arange(rank, spec.boards.shape[0], world)
    return BoardSpec(spec.boards[sel], spec.board_prob[sel], spec.board_mult[sel], spec.sym_perm,
                     "%s; shard %d/%d (%d boards)" % (spec.note, rank, world, sel.size))


class ShardedCFRSolver(CFRSolver):
    """CFRSolver whose bottom-up sweeps are split around an all-reduce of the chance-node sums.
    world == 1 (or no process group) runs the same split schedule without communication."""

    def __init__(self, game_cls, env_args, board_spec, algo="CFRPlus", delay=0, device=None, rank=0, world=1,
                 group=None, root_actions=None, dcfr=_dcfr.DEFAULT,
                 pcfr_gamma=algorithm.PCFR_GAMMA):
        self.rank, self.world, self.group = rank, world, group
        ft = FlatTree(game_cls, env_args, board_spec=shard_board_spec(board_spec, rank, world) if world > 1 else board_spec,
                      root_actions=root_actions)
        self.ft = ft
        if world > 1 and (ft.kind == nat.KIND_SHOWDOWN_ALLIN).any():
            raise NotImplementedError("all-in showdowns before the board is complete run out over ALL boards below them: "
                                      "not available with the boards sharded over ranks (run this tree on one GPU)")
        super().__init__(ft, algo=algo, delay=delay, device=device, avg_f64=False, persistent=False, dcfr=dcfr,
                         pcfr_gamma=pcfr_gamma)
        # levels holding BOUNDARY chance nodes: chance nodes right below the replicated trunk (no deal above them), whose
        # children - the boards of the first chance layer - are spread over the ranks.  Deeper chance nodes are local.
        self._n_chance, self._n_boundary = {}, {}
        for d in range(ft.n_levels):
            lo, hi = int(ft.level_start[d]), int(ft.level_start[d + 1])
            ch = ft.kind[lo:hi] == nat.KIND_CHANCE
            if ch.any():
                self._n_chance[d] = int(ch.sum())
                self._n_boundary[d] = int((ch & (ft.cdepth[lo:hi] == 0)).sum())
        self._chance_levels = [d for d in self._n_chance if self._n_boundary[d] > 0]
        self.n_allreduce = 0

    # ---- the one collective of the path
    def _allreduce_chance_sums(self, bufs, level, arrays):
        """all-reduce the per-node sums W of the boundary chance nodes of `level` (they come first in the work list);
        W is laid out [4][n_chance][ld] at float offset 4 * n_chance * chunks * ld of the workspace"""
        dt = self.dtree
        n_chance, n_b = self._n_chance[level], self._n_boundary[level]
        chunks = -(-dt.desc.max_chance_children // 128)
        w_off = 4 * n_chance * chunks * dt.ld
        for arr in arrays:
            o = w_off + arr * n_chance * dt.ld
            view = bufs.workspace[o:o + n_b * dt.ld]
            if self.world > 1:
                dist.all_reduce(view, op=dist.ReduceOp.SUM, group=self.group)
            self.n_allreduce += 1

    def _value_sweep(self, bufs, mask, with_br, algo, upd_p, modes, top=None):
        """bottom-up sweep from level `top` (default: the deepest) to the root"""
        tree, buf = C.byref(self.dtree.desc), C.byref(bufs.desc)

        def levels(hi, lo, phase):
            nat.call("prl_value_levels", tree, buf, mask, int(with_br), algo, upd_p, self.iter_counter, self.delay,
                     nat.modes(*modes), hi, lo, phase, _stream())

        arrays = [2 * p + k for p in (0, 1) if mask & (1 << p) for k in ((0, 1) if with_br else (0,))]
        hi = self.ft.n_levels - 1 if top is None else top
        for d in sorted(self._chance_levels, reverse=True):
            if d > hi:
                continue
            if hi > d:
                levels(hi, d + 1, 0)
            levels(d, d, 1)
            self._allreduce_chance_sums(bufs, d, arrays)
            levels(d, d, 2)
            hi = d - 1
        if hi >= 0:
            levels(hi, 0, 0)

    def iteration(self, n=1):
        with _on(self.dtree.device):
            self._iteration_sharded(n)

    def _iteration_sharded(self, n):
        self._bind_factors(n)
        tree, buf = C.byref(self.dtree.desc), C.byref(self.bufs.desc)
        for _ in range(n):
            for p in (0, 1):
                self._value_sweep(self.bufs, 1 << p, False, self.algo, p, self.modes)
                self.modes[p] = nat.STRAT_F32
                nat.call("prl_reach_update", tree, buf, self.algo, p, self.iter_counter, self.delay, _stream())
            self.iter_counter += 1

    def _value_pass_br(self, ops, modes):
        with _on(self.dtree.device):
            self._value_sweep(ops.bufs, 3, True, -1, -1, modes)
