"""Tabular CFR `EvalAgent` (SURVEY.md §8f N1): a concrete `EvalAgentBase` backed by the average-strategy table of a
`pokerrl_b200.cfr` solver, so that the solver's result can be handed to the evaluators (`LocalBRMaster`) and stored /
restored (`store_to_disk` / `load_from_disk`).  The reference ships no concrete tabular agent (EvalAgentBase.py is
abstract); the query contract is `StrategyFiller._fill_with_agent_policy` (StrategyFiller.py:88-116).

Solvers of the board engine (Flop5Holdem, pokerrl_b200.board_engine) hold no slot table: their agent keeps the strength-ordered
rows, class keys and position -> hand tables (board_engine.BoardPolicyTables, about 8.2 GB of rows + 290 MB for the full
game) and answers for any Flop5Holdem PublicTree - any board spec, either engine - with one kernel launch
(prl_board_policy_query)."""
import numpy as np

from pokerrl_b200 import algorithm
from pokerrl_b200.rl.base_cls.EvalAgentBase import EvalAgentBase


def tree_fingerprint(ft):
    """structural identity of a flat tree: slot count + hash of kinds / fan-outs / actions / pots"""
    import hashlib
    h = hashlib.sha1()
    for a in (ft.kind, ft.n_children, ft.action, ft.pot):
        h.update(np.ascontiguousarray(a).tobytes())
    return (int(ft.n_slots), h.hexdigest())


def average_strategy_table(solver):
    """float32 [n_slots, R] average strategy of a CFRSolver (host copy), normalised like the reference's `avg_strat`."""
    ft, R = solver.ft, solver.ft.R
    avg = solver.alg.average(solver.iter_counter)
    if avg != algorithm.SUMS:
        src = solver.bufs.strat if avg == algorithm.CURRENT else solver.bufs.avg
        return src[:, :R].float().cpu().numpy()
    s = solver.bufs.avg[:, :R].cpu().numpy()
    out = np.empty_like(s)
    for n in np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]:
        a, fs = ft.n_children[n], ft.first_slot[n]
        tot = s[fs:fs + a].sum(axis=0, keepdims=True)
        with np.errstate(divide="ignore", invalid="ignore"):
            out[fs:fs + a] = np.where(tot == 0, np.float32(1.0 / a), s[fs:fs + a] / tot)
    return out


class TabularCFREvalAgent(EvalAgentBase):
    EVAL_MODE_AVG = "AVG"
    ALL_MODES = [EVAL_MODE_AVG]

    def __init__(self, t_prof, mode=None, device=None):
        super().__init__(t_prof=t_prof, mode=mode or self.EVAL_MODE_AVG, device=device)
        self._table = None  # float32 [n_slots, R]: rows in the flat tree's slot order
        self._board = None  # board_engine.BoardPolicyTables of a board-engine solver
        self._n_actions = self.env_bldr.N_ACTIONS

    def update_weights(self, weights_for_eval_agent):
        """weights: float32 [n_slots, R] table, or (table, fingerprint) with the structural fingerprint of the tree the table
        belongs to (tree_fingerprint); with a fingerprint, querying the agent on a different tree raises"""
        fp = None
        if isinstance(weights_for_eval_agent, tuple):
            weights_for_eval_agent, fp = weights_for_eval_agent
        self._table = np.ascontiguousarray(weights_for_eval_agent, dtype=np.float32)
        self._fingerprint = fp
        self._board = None

    @classmethod
    def from_cfr(cls, t_prof, cfr, tree_idx=0):
        agent = cls(t_prof=t_prof)
        solver = cfr.solvers[tree_idx]
        if getattr(solver, "ft", None) is None and hasattr(solver, "ft1"):  # board engine: no slot table
            from pokerrl_b200.board_engine import BoardPolicyTables
            return cls.from_board_tables(t_prof, BoardPolicyTables.from_solver(solver))
        agent.update_weights((average_strategy_table(solver), tree_fingerprint(solver.ft)))
        return agent

    @classmethod
    def from_board_tables(cls, t_prof, tables):
        """the agent that plays a board_engine.BoardPolicyTables (a board-engine solver's average, a best response)"""
        agent = cls(t_prof=t_prof)
        agent._board = tables
        agent._fingerprint = (tables.fingerprint, tables.spec_id)
        return agent

    def can_compute_mode(self):
        return self._table is not None or self._board is not None

    def get_a_probs_for_each_hand(self):
        """[RANGE_SIZE, N_ACTIONS] with the node's probabilities at its allowed actions, 0 elsewhere"""
        node = self._node
        ft = node.tree.flat
        if self._board is not None:
            return self._board.answer_node(ft, node.idx, self._n_actions)
        if getattr(self, "_fingerprint", None) is not None and tree_fingerprint(ft) != self._fingerprint:
            raise ValueError("this agent's table was computed on a different public tree (stack / bet set / slot order): "
                             "build one agent per evaluated tree (TabularCFREvalAgent.from_cfr(..., tree_idx=...))")
        fs, a = ft.first_slot[node.idx], ft.n_children[node.idx]
        out = np.zeros((ft.R, self._n_actions), np.float32)
        out[:, node.allowed_actions] = self._table[fs:fs + a].T
        return out

    def get_a_probs_for_public_tree(self, tree):
        """all decision nodes at once: [n_decision, R, N_ACTIONS] on the tree's device (one scatter of the table rows)"""
        import torch
        ft = tree.flat
        if self._board is not None:
            return self._board.answer_tree(ft, self._n_actions)
        if getattr(self, "_fingerprint", None) is not None and tree_fingerprint(ft) != self._fingerprint:
            raise ValueError("this agent's table was computed on a different public tree")
        dev = tree.dtree.device
        dec = tree.decision_nodes()
        dec_idx = np.full(ft.n_nodes, -1, np.int64)
        dec_idx[dec] = np.arange(dec.size)
        child = np.nonzero(ft.slot >= 0)[0]
        out = torch.zeros((dec.size, ft.R, self._n_actions), dtype=torch.float32, device=dev)
        tab = torch.from_numpy(self._table).to(dev)  # [n_slots, R]
        out[torch.from_numpy(dec_idx[ft.parent[child]]).to(dev), :, torch.from_numpy(ft.action[child].astype(np.int64)).to(dev)] = tab
        return out

    def _state_dict(self):
        """board engine: CPU tensors (the full game's rows are about 8.2 GB)"""
        return {"table": self._table, "fingerprint": getattr(self, "_fingerprint", None),
                "board": None if self._board is None else self._board.state_dict()}

    def _load_state_dict(self, state):
        self._table = state["table"]
        self._fingerprint = state.get("fingerprint")
        self._board = None
        if state.get("board") is not None:  # back onto the device
            from pokerrl_b200.board_engine import BoardPolicyTables
            self._board = BoardPolicyTables.from_state(state["board"], self.device)
