"""`PublicTree` with the reference's API (`PokerRL/game/_/tree/PublicTree.py:30-158`) on top of the flat,
HBM-resident tree: build_tree / fill_uniform_random / fill_random_random / fill_with_agent_policy /
update_reach_probs / compute_ev / root / n_nodes / n_nonterm.

Nodes are *views* (`NodeView`) into the device arrays exposing the reference's node fields (nodes.py:8-62):
children, parent, p_id_acting_next, p_id_acted_last, action, allowed_actions, is_terminal, depth, strategy [R,A],
reach_probs / ev / ev_br [2,R], exploitability [2], env_state (public part).  Host copies are fetched lazily after
each pass.
"""
import os

import numpy as np
import torch

from pokerrl_b200 import _native as nat
from pokerrl_b200.game import tree_export
from pokerrl_b200.game.Poker import Poker
from pokerrl_b200.game.flat_tree import (FlatTree, KIND_CHANCE, KIND_FOLD, KIND_P1)
from pokerrl_b200.solver import DeviceTree, TreeBuffers, TreeOps


class NodeView:
    __slots__ = ("tree", "idx")

    def __init__(self, tree, idx):
        self.tree, self.idx = tree, int(idx)

    def __eq__(self, o):
        return isinstance(o, NodeView) and o.tree is self.tree and o.idx == self.idx

    def __hash__(self):
        return hash((id(self.tree), self.idx))

    # ---- structure
    @property
    def _ft(self):
        return self.tree.flat

    @property
    def children(self):
        ft, i = self._ft, self.idx
        fc = ft.first_child[i]
        return [NodeView(self.tree, fc + k) for k in range(ft.n_children[i])] if fc >= 0 else []

    @property
    def parent(self):
        p = self._ft.parent[self.idx]
        return None if p < 0 else NodeView(self.tree, p)

    @property
    def is_terminal(self):
        return self._ft.kind[self.idx] >= KIND_FOLD

    @property
    def depth(self):
        return int(np.searchsorted(self._ft.level_start, self.idx, side="right") - 1)

    @property
    def p_id_acting_next(self):
        k = self._ft.kind[self.idx]
        if k <= KIND_P1:
            return int(k)
        return PublicTree.CHANCE_ID if k == KIND_CHANCE else None

    @property
    def p_id_acted_last(self):
        a = self._ft.acted_last[self.idx]
        return None if a == -2 else (PublicTree.CHANCE_ID if a == -1 else int(a))

    @property
    def action(self):
        if self._ft.acted_last[self.idx] == -1 or self.idx == 0:
            return "CHANCE"
        return int(self._ft.action[self.idx])

    @property
    def allowed_actions(self):
        ft, i = self._ft, self.idx
        if ft.kind[i] > KIND_P1 or ft.first_child[i] < 0:
            return []
        fc = ft.first_child[i]
        return [int(a) for a in ft.action[fc:fc + ft.n_children[i]]]

    @property
    def env_state(self):
        """Public part of the reference's env state dict (PokerEnv.state_dict, PokerEnv.py:1161-1197)."""
        ft, i = self._ft, self.idx
        lut = self.tree.env_bldr.lut_holder
        return {
            "current_round": int(ft.round[i]), "main_pot": int(ft.pot[i]), "side_pots": [0, 0],
            "board_2d": lut.get_2d_cards(ft.node_board_cards()[i]) if lut is not None else None,
            "current_player": self.p_id_acting_next,
            "seats": [{"seat_id": p, "stack": int(ft.stack[i, p]), "current_bet": int(ft.bet[i, p])} for p in (0, 1)],
        }

    # ---- values
    def _vec(self, name):
        return self.tree._host(name)[:, self.idx, :self._ft.R]

    @property
    def reach_probs(self):
        return self._vec("reach")

    @property
    def ev(self):
        return self._vec("ev")

    @property
    def ev_br(self):
        return self._vec("ev_br")

    @property
    def ev_weighted(self):
        return self.ev * self.reach_probs

    @property
    def ev_br_weighted(self):
        return self.ev_br * self.reach_probs

    @property
    def epsilon(self):
        return self.ev_br_weighted - self.ev_weighted

    @property
    def exploitability(self):
        if self.idx == 0:
            return self.tree._root_expl  # computed on the device in the reference's summation order
        return np.sum(self.epsilon, axis=1)

    @property
    def strategy(self):
        """[R, A] strategy of the player (or chance) acting at this node; None at terminals."""
        return self.tree._node_strategy(self.idx)

    @property
    def br_a_idx_in_child_arr_for_each_hand(self):
        ft, i = self._ft, self.idx
        if ft.kind[i] > KIND_P1:
            return None
        fc, A = ft.first_child[i], ft.n_children[i]
        return np.argmax(self.tree._host("ev_br")[ft.kind[i], fc:fc + A, :ft.R], axis=0)


class PublicTree:
    CHANCE_ID = "Ch"

    def __init__(self, env_bldr, stack_size, stop_at_street, put_out_new_round_after_limit=False,
                 is_debugging=False, device=None, board_spec=None):
        """board_spec (extension, two-card games): the boards of the chance layer (holdem_boards.BoardSpec); default = all
        boards of the game as suit-isomorphism classes"""
        self._board_spec = board_spec
        self._env_bldr = env_bldr
        self._stack_size = stack_size
        self._is_debugging = is_debugging
        self._stop_at_street_arg = stop_at_street
        self._put_out_new_round_after_limit = put_out_new_round_after_limit
        self._device = device
        # optional PokerViz export: only into an installed viewer that carries the reference's marker file
        # (PublicTree.py:45-56); otherwise export_to_file() does nothing
        viz = os.path.join("C:\\" if os.name == "nt" else os.path.expanduser("~/"), "PokerRL_Viz")
        installed = os.path.isdir(viz) and os.path.isfile(os.path.join(viz, "ALLOWED_TO_WRITE_HERE.dontdelete"))
        self.dir_tree_vis_data = os.path.join(viz, "data") if installed else None
        self.root = None
        self.flat = None
        self._n_seats = env_bldr.N_SEATS

    # ---- properties of the reference
    stack_size = property(lambda s: s._stack_size)
    is_debugging = property(lambda s: s._is_debugging)
    n_seats = property(lambda s: s._n_seats)
    env_bldr = property(lambda s: s._env_bldr)
    put_out_new_round_after_limit = property(lambda s: s._put_out_new_round_after_limit)

    @property
    def stop_at_street(self):
        last = self._env_bldr.rules.ALL_ROUNDS_LIST[-1]
        return last + 1 if self._stop_at_street_arg is None else self._stop_at_street_arg

    @property
    def n_nodes(self):  # the reference does not count the root (PublicTree.py:161-166)
        return self.flat.n_nodes - 1

    @property
    def n_nonterm(self):
        return self.flat.n_nonterm - 1

    # ---- build
    def build_tree(self):
        args = self._env_bldr.args_for_stack(self._stack_size)
        self.flat = FlatTree(self._env_bldr.env_cls, args, stop_at_street=self._stop_at_street_arg, board_spec=self._board_spec)
        self.dtree = DeviceTree(self.flat, self._device)
        self.bufs = TreeBuffers(self.dtree, avg_dtype=torch.float64)
        self.ops = TreeOps(self.dtree, self.bufs)
        self.modes = [nat.STRAT_UNIFORM64, nat.STRAT_UNIFORM64]
        self._slot_maps = None
        self._cache = {}
        self._root_expl = None
        self._has_reach = self._has_ev = False
        self.root = NodeView(self, 0)

    def build_structure(self):
        """The flat tree and a device handle only: no node vectors, no strength tables.  Enough to query an agent
        (agent_strategy_table with an explicit `out`); the board engine's policy evaluation builds one per chunk of boards."""
        from types import SimpleNamespace
        from pokerrl_b200.solver import _require_cuda
        args = self._env_bldr.args_for_stack(self._stack_size)
        self.flat = FlatTree(self._env_bldr.env_cls, args, stop_at_street=self._stop_at_street_arg, board_spec=self._board_spec)
        R = self.flat.R
        self.dtree = SimpleNamespace(device=_require_cuda(self._device),
                                     ld=R if self.flat.rules.N_HOLE_CARDS == 1 else -(-R // 4) * 4)
        self.bufs = self.ops = None
        self.modes = [nat.STRAT_UNIFORM64, nat.STRAT_UNIFORM64]
        self._slot_maps = None
        self._cache = {}
        self._root_expl = None
        self._has_reach = self._has_ev = False
        self.root = NodeView(self, 0)

    # ---- strategy filling (StrategyFiller.py:17-46)
    def fill_uniform_random(self):
        self.modes = [nat.STRAT_UNIFORM64, nat.STRAT_UNIFORM64]
        self.update_reach_probs()

    def fill_random_random(self):
        ft = self.flat
        s = np.zeros((ft.n_slots, ft.R))
        for n in np.nonzero((ft.kind <= KIND_P1) & (ft.first_child >= 0))[0]:  # same visiting order not required
            A = ft.n_children[n]
            r = np.random.random(size=(ft.R, A))
            r /= np.expand_dims(np.sum(r, axis=1), axis=-1)
            s[ft.first_slot[n]:ft.first_slot[n] + A] = r.T
        self.set_strategy_table(s)

    def set_strategy_table(self, table):
        """table: [n_slots, R] float64 (reference math in double) or float32 (float math)."""
        t = torch.from_numpy(np.ascontiguousarray(table))
        if t.dtype == torch.float64:
            self.bufs.avg[:, :self.flat.R].copy_(t)
            self.modes = [nat.STRAT_AVG_F64, nat.STRAT_AVG_F64]
        else:
            self.bufs.strat[:, :self.flat.R].copy_(t.float())
            self.modes = [nat.STRAT_F32, nat.STRAT_F32]
        self.update_reach_probs()

    def decision_nodes(self):
        """flat ids of the decision nodes in flat order = the batch order of EvalAgentBase.get_a_probs_for_public_tree"""
        ft = self.flat
        return np.nonzero((ft.kind <= KIND_P1) & (ft.first_child >= 0))[0]

    def fill_with_agent_policy(self, agent):
        """StrategyFiller._fill_with_agent_policy (:88-116): the agent's strategy table (agent_strategy_table), then the
        reach pass."""
        tab = self.agent_strategy_table(agent)
        if isinstance(tab, torch.Tensor):
            self.modes = [nat.STRAT_F32, nat.STRAT_F32]
            self.update_reach_probs()
        else:
            self.set_strategy_table(tab)

    def agent_strategy_table(self, agent, out=None):
        """The agent's strategy table, one row per slot.  Agents that answer for the whole tree at once
        (`get_a_probs_for_public_tree(tree)` -> device float32 [n_decision, R, N_ACTIONS]) are gathered by ONE device launch
        into `out` (float32 [n_slots, ld] on the tree's device; default: the tree's `strat` buffer), which is returned.  Others
        are queried node by node like the reference does; the host table [n_slots, R] is returned (float64 if any answer
        was float64, else float32)."""
        ft = self.flat
        batched = getattr(agent, "get_a_probs_for_public_tree", None)
        probs = batched(self) if batched is not None else None
        if probs is not None:
            import ctypes as C
            from pokerrl_b200.solver import _on, _stream
            dev = self.dtree.device
            out = self.bufs.strat if out is None else out
            probs = torch.as_tensor(probs).to(device=dev, dtype=torch.float32).contiguous()
            dec = self.decision_nodes()
            assert probs.shape[0] == dec.size and probs.shape[1] == ft.R, probs.shape
            assert out.shape[0] >= ft.n_slots and out.shape[1] == self.dtree.ld and out.dtype == torch.float32, out.shape
            if getattr(self, "_slot_maps", None) is None:
                dec_idx = np.full(ft.n_nodes, -1, np.int64)
                dec_idx[dec] = np.arange(dec.size)
                child = np.nonzero(ft.slot >= 0)[0]  # flat order == slot order
                self._slot_maps = (torch.from_numpy(dec_idx[ft.parent[child]].astype(np.int32)).to(dev),
                                   torch.from_numpy(ft.action[child].astype(np.int32)).to(dev))
            d_of, a_of = self._slot_maps
            with _on(dev):
                nat.call("prl_gather_agent_policy", C.c_void_p(probs.data_ptr()), int(probs.shape[2]), C.c_void_p(d_of.data_ptr()),
                         C.c_void_p(a_of.data_ptr()), ft.n_slots, ft.R, self.dtree.ld, C.c_void_p(out.data_ptr()),
                         _stream(dev))
            return out
        rows, dt = np.zeros((ft.n_slots, ft.R)), None
        for n in np.nonzero((ft.kind <= KIND_P1) & (ft.first_child >= 0))[0]:
            node = NodeView(self, n)
            agent.set_to_public_tree_node_state(node=node)
            a_probs = np.asarray(agent.get_a_probs_for_each_hand())
            dt = a_probs.dtype if dt is None else np.promote_types(dt, a_probs.dtype)
            rows[ft.first_slot[n]:ft.first_slot[n] + ft.n_children[n]] = a_probs[:, node.allowed_actions].T
        return rows if dt == np.float64 else rows.astype(np.float32)

    def update_reach_probs(self):
        self.ops.reach_pass(self.modes)
        self._has_reach = True
        self._cache.pop("reach", None)

    def compute_ev(self):
        self.ops.value_pass(self.modes, 3, True)
        self._root_expl = self.ops.root_exploitability()
        self._has_ev = True
        self._cache.pop("ev", None)
        self._cache.pop("ev_br", None)

    def best_response_table(self):
        """after compute_ev: float32 [n_slots, R] on the tree's device, one-hot rows of the best response of the seat acting at
        each decision node - 1 on the FIRST child in child order whose ev_br is the maximum, the child
        br_a_idx_in_child_arr_for_each_hand names"""
        from pokerrl_b200.board_engine import first_max_onehot
        assert self._has_ev, "compute_ev() first"
        ft, dev, R = self.flat, self.dtree.device, self.flat.R
        dec = self.decision_nodes()
        n_ch = ft.n_children[dec].astype(np.int64)
        a_max = int(n_ch.max())
        k = np.arange(a_max)
        valid = k[None, :] < n_ch[:, None]
        child = np.where(valid, ft.first_child[dec][:, None] + k[None, :], 0)
        seat = np.broadcast_to(ft.kind[dec].astype(np.int64)[:, None], child.shape)
        t_valid = torch.from_numpy(valid).to(dev)
        v = self.bufs.ev_br[torch.from_numpy(seat).to(dev), torch.from_numpy(child).to(dev), :R]  # [n_dec, a_max, R]
        v = torch.where(t_valid[:, :, None], v, torch.full_like(v, -float("inf")))
        onehot = first_max_onehot(v, 1)
        out = torch.zeros((ft.n_slots, R), dtype=torch.float32, device=dev)
        slots = ft.first_slot[dec][:, None] + k[None, :]
        out[torch.from_numpy(slots[valid]).to(dev)] = onehot[t_valid]
        return out

    # ---- host access
    def _host(self, name):
        if name not in self._cache:
            self._cache[name] = getattr(self.bufs, name).cpu().numpy()
        return self._cache[name]

    def _node_strategy(self, n):
        ft = self.flat
        k = ft.kind[n]
        if k >= KIND_FOLD or ft.first_child[n] < 0:
            return None
        A = ft.n_children[n]
        if k == KIND_CHANCE:  # StrategyFiller.py:148-169
            bc = ft.node_board_cards()
            s = np.zeros((ft.R, A), np.float32)
            for c in range(A):
                mask = np.ones(ft.R, bool)
                mask[bc[ft.first_child[n] + c][bc[ft.first_child[n] + c] >= 0]] = False
                s[mask, c] = 1.0 / (ft.rules.N_CARDS_IN_DECK - 2)
            return s
        m = self.modes[k]
        fs = ft.first_slot[n]
        if m == nat.STRAT_UNIFORM64:
            return np.full((ft.R, A), 1.0 / float(A))
        tab = self.bufs.strat if m == nat.STRAT_F32 else self.bufs.avg
        return tab[fs:fs + A, :ft.R].cpu().numpy().T.copy()

    # ---- export hooks of the reference (PokerViz browser tool; not part of the compute path): PublicTree.py:143-149
    def get_tree_as_dict(self):
        reach = self._host("reach") if self._has_reach else None
        ev, ev_br = (self._host("ev"), self._host("ev_br")) if self._has_ev else (None, None)
        return tree_export.export_tree_dict(self.flat, reach, ev, ev_br, self._node_strategy if self._has_reach else None)

    def export_to_file(self, name="data"):
        if self.dir_tree_vis_data is not None:
            os.makedirs(self.dir_tree_vis_data, exist_ok=True)
            tree_export.write_tree_js(os.path.join(self.dir_tree_vis_data, str(name) + ".js"), self.get_tree_as_dict())
