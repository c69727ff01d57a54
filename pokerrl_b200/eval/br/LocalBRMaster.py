"""Exact best-response evaluator for any `EvalAgentBase` (`PokerRL/eval/br/LocalBRMaster.py:11-80`): one HBM-resident
`PublicTree` per evaluation stack size; `fill_with_agent_policy` -> reach pass -> value pass with BR on the GPU ->
`root.exploitability * EV_NORMALIZER` averaged over the two seats.

Games the board engine supports (Flop5Holdem; PRL_ENGINE unset) are evaluated by `board_engine.BoardPolicyEvaluator`
instead: the agent is queried chunk by chunk over the boards, so memory is bounded by the chunk, not by the game (a
PublicTree of the full game would need about 104 GB).  board_spec (extension, like CFRBase's): the boards of the chance layer;
default = the game's suit-isomorphism classes."""
import copy

from pokerrl_b200.eval._.EvaluatorMasterBase import EvaluatorMasterBase
from pokerrl_b200.game.PublicTree import PublicTree
from pokerrl_b200.rl.base_cls.TrainingProfileBase import get_env_builder


class LocalBRMaster(EvaluatorMasterBase):
    def __init__(self, t_prof, chief_handle, eval_agent_cls, device=None, board_spec=None):
        super().__init__(t_prof=t_prof, eval_env_bldr=get_env_builder(t_prof=t_prof), chief_handle=chief_handle,
                         eval_type="BR")
        self._env_bldr = get_env_builder(t_prof=t_prof)
        assert self._env_bldr.N_SEATS == 2
        self._eval_agent = eval_agent_cls(t_prof=t_prof)
        from pokerrl_b200 import board_engine
        env_cls = self._env_bldr.env_cls
        if all(board_engine.supports(env_cls, self._env_bldr.args_for_stack(s), "CFRPlus") for s in t_prof.eval_stack_sizes):
            self._game_trees = [board_engine.BoardPolicyEvaluator(self._env_bldr, stack_size=s, board_spec=board_spec, device=device)
                                for s in t_prof.eval_stack_sizes]
            for gt in self._game_trees:
                print("Tree with stack size", gt.stack_size, "has", gt.n_nodes - 1, "nodes out of which", gt.n_nonterm - 1,
                      "are non-terminal.")
            return
        self._game_trees = [PublicTree(env_bldr=self._env_bldr, stack_size=stack_size, stop_at_street=None,
                                       put_out_new_round_after_limit=True, is_debugging=t_prof.DEBUGGING, device=device,
                                       board_spec=board_spec)
                            for stack_size in t_prof.eval_stack_sizes]
        for gt in self._game_trees:
            gt.build_tree()
            print("Tree with stack size", gt.stack_size, "has", gt.n_nodes, "nodes out of which", gt.n_nonterm,
                  "are non-terminal.")

    @property
    def eval_agent(self):
        return self._eval_agent

    def evaluate(self, iter_nr):
        for mode in self._t_prof.eval_modes_of_algo:
            totals = []
            for stack_size_idx, stack_size in enumerate(self._t_prof.eval_stack_sizes):
                self._eval_agent.set_mode(mode)
                self._eval_agent.set_stack_size(stack_size=stack_size)
                if self._eval_agent.can_compute_mode():
                    e0, e1 = self._compute_br_heads_up(stack_size_idx=stack_size_idx, iter_nr=iter_nr)
                    self._log_results(iter_nr=iter_nr, agent_mode=mode, stack_size_idx=stack_size_idx,
                                      score=(e0 + e1) / 2)
                    totals.append((e0 + e1) / 2.0)
            if self._is_multi_stack and totals:
                self._log_multi_stack(agent_mode=mode, iter_nr=iter_nr, score_total=sum(totals) / float(len(totals)))

    def update_weights(self):
        self._eval_agent.update_weights(copy.deepcopy(self.pull_current_strat_from_chief()))

    def best_response_agent(self, stack_size_idx=0):
        """(e0, e1, agent): the exploitability of each seat of the current eval agent at evaluation stack stack_size_idx, in the
        game's metric (the numbers evaluate() logs the mean of), and its best response as a TabularCFREvalAgent - seat s's rows
        are seat s's best response.  At every node the action is the FIRST child in child order whose best-response value is
        the maximum (np.argmax).  Board engine: the agent holds the BoardPolicyTables of BoardPolicyEvaluator.best_response
        (for the full Flop5Holdem game about 8.5 GB of device memory besides the evaluated agent's); level engine: the
        one-hot slot table of PublicTree.best_response_table with the tree's fingerprint."""
        from pokerrl_b200.cfr.TabularCFREvalAgent import TabularCFREvalAgent, tree_fingerprint
        gt = self._game_trees[stack_size_idx]
        norm = self._env_bldr.env_cls.EV_NORMALIZER
        self._eval_agent.set_stack_size(stack_size=self._t_prof.eval_stack_sizes[stack_size_idx])
        if not isinstance(gt, PublicTree):  # board engine
            e, tables = gt.best_response(self._eval_agent)
            return float(e[0]) * norm, float(e[1]) * norm, TabularCFREvalAgent.from_board_tables(self._t_prof, tables)
        e0, e1 = self._compute_br_heads_up(stack_size_idx=stack_size_idx)
        agent = TabularCFREvalAgent(t_prof=self._t_prof)
        agent.update_weights((gt.best_response_table().cpu().numpy(), tree_fingerprint(gt.flat)))
        return e0, e1, agent

    def _compute_br_heads_up(self, stack_size_idx, iter_nr=None, do_export_tree=True):
        gt = self._game_trees[stack_size_idx]
        norm = self._env_bldr.env_cls.EV_NORMALIZER
        if not isinstance(gt, PublicTree):  # board engine
            e = gt.evaluate(self._eval_agent)
            return float(e[0]) * norm, float(e[1]) * norm
        gt.fill_with_agent_policy(agent=self._eval_agent)
        gt.compute_ev()
        return float(gt.root.exploitability[0]) * norm, float(gt.root.exploitability[1]) * norm
