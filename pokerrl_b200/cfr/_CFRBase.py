"""Base of the full-width tabular CFR variants with the reference's constructor, schedule and log names
(`PokerRL/cfr/_CFRBase.py:12-278`), driving the H100 engine (`pokerrl_b200.solver.CFRSolver`).

Differences to the reference, none of which changes a logged number:
  * one flat HBM-resident tree per stack size instead of Python node objects; the per-iteration rebuild of a fresh
    evaluation tree (`_CFRBase.py:222-227`, 23 % of the reference's iteration time) is replaced by a second set of
    reach vectors on the same device tree;
  * the regret update, regret matching, reach update and averaging of one player are two fused sweeps;
  * `eval_every` (extension, default 1 = the reference's behaviour) evaluates / logs exploitability only every
    k-th iteration (BASELINE.json config 2: "exact BR every 20 iters").
"""
import copy

from pokerrl_b200.game.flat_tree import FlatTree
from pokerrl_b200.game.games import get_env_cls_from_str
from pokerrl_b200.game.wrappers import HistoryEnvBuilder
from pokerrl_b200.solver import CFRSolver


class CFRBase:
    _SOLVER_ALGO = None  # "VanillaCFR" | "CFRPlus" | "LinearCFR" | "DCFR" | "PCFRPlus"

    def __init__(self, name, chief_handle, game_cls, agent_bet_set, algo_name, starting_stack_sizes=None,
                 delay=0, eval_every=1, device=None, avg_f64=False, board_spec=None, dcfr=None, pcfr_gamma=None):
        import os
        avg_f64 = bool(avg_f64) or os.environ.get("PRL_AVG_F64", "0") == "1"  # numpy >= 2 semantics of CFRPlus.py:69-73
        self._name = name
        self._n_seats = 2
        self._chief_handle = chief_handle
        self._starting_stack_sizes = ([game_cls.DEFAULT_STACK_SIZE] if starting_stack_sizes is None
                                      else copy.deepcopy(starting_stack_sizes))
        self._game_cls_str = game_cls.__name__
        self._env_args = [
            game_cls.ARGS_CLS(n_seats=self._n_seats, starting_stack_sizes_list=[s] * self._n_seats,
                              bet_sizes_list_as_frac_of_pot=agent_bet_set)
            for s in self._starting_stack_sizes]
        env_cls = get_env_cls_from_str(self._game_cls_str)
        self._env_bldrs = [HistoryEnvBuilder(env_cls=env_cls, env_args=a) for a in self._env_args]
        self._solvers = [self._make_solver(env_cls, a, delay, device, avg_f64, board_spec, dcfr, pcfr_gamma)
                         for a in self._env_args]
        self._flat_trees = [getattr(s, "ft", None) for s in self._solvers]  # None: board engine (no node arrays)
        for s, a in zip(self._solvers, self._env_args):
            ft = getattr(s, "ft", None) or s
            print("Tree with stack size", a.starting_stack_sizes_list, "has", ft.n_nodes - 1,
                  "nodes out of which", ft.n_nonterm - 1, "are non-terminal.")
        self._algo_name = algo_name
        self._eval_every = max(1, int(eval_every))
        ch, S = self._chief_handle, self._starting_stack_sizes
        self._exps_curr_total = [ch.create_experiment(self._name + "_Curr_S" + str(s) + "_total_" + algo_name)
                                 for s in S]
        self._exps_avg_total = [ch.create_experiment(self._name + "_Avg_total_S" + str(s) + "_" + algo_name)
                                for s in S]
        self._exp_all_averaged_curr_total = ch.create_experiment(self._name + "_Curr_total_averaged_" + algo_name)
        self._exp_all_averaged_avg_total = ch.create_experiment(self._name + "_Avg_total_averaged_" + algo_name)
        self._iter_counter = None

    def _make_solver(self, env_cls, env_args, delay, device, avg_f64, board_spec, dcfr=None, pcfr_gamma=None):
        """One engine per stack size.  Two-card games launched under torch.distributed (one process per GPU) shard their
        boards over the ranks (pokerrl_b200.distributed); everything else runs on this process's GPU.  dcfr: DCFR's
        (alpha, beta, gamma), pcfr_gamma: PCFR+'s gamma, handed to whichever engine runs it."""
        import torch.distributed as dist
        kw = {} if dcfr is None else {"dcfr": dcfr}
        if pcfr_gamma is not None:
            kw["pcfr_gamma"] = pcfr_gamma
        multi = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
        if device is None and multi:  # one process per GPU: this rank's device, not cuda:0
            import os
            device = "cuda:%d" % int(os.environ.get("LOCAL_RANK", "0"))
        from pokerrl_b200 import board_engine
        if board_engine.supports(env_cls, env_args, self._SOLVER_ALGO):
            # one chance layer with the compiled post-deal shape (Flop5Holdem): board-resident fused sweeps
            return board_engine.BoardCFRSolver(env_cls, env_args, board_spec, algo=self._SOLVER_ALGO, delay=delay,
                                               device=device, rank=dist.get_rank() if multi else 0,
                                               world=dist.get_world_size() if multi else 1, **kw)
        if env_cls.RULES.N_HOLE_CARDS == 2 and multi:
            from pokerrl_b200.distributed import ShardedCFRSolver
            from pokerrl_b200.game.holdem_boards import BoardSpec
            spec = board_spec if board_spec is not None else BoardSpec.full_game(env_cls.RULES)
            return ShardedCFRSolver(env_cls, env_args, spec, algo=self._SOLVER_ALGO, delay=delay, device=device,
                                    rank=dist.get_rank(), world=dist.get_world_size(), **kw)
        ft = FlatTree(env_cls, env_args, board_spec=board_spec)
        return CFRSolver(ft, algo=self._SOLVER_ALGO, delay=delay, device=device, avg_f64=avg_f64, **kw)

    name = property(lambda s: s._name)
    algo_name = property(lambda s: s._algo_name)
    iter_counter = property(lambda s: s._iter_counter)
    solvers = property(lambda s: s._solvers)

    def reset(self):
        self._iter_counter = 0
        for s in self._solvers:
            s.reset()
        self._log_curr_strat_expl()

    def iteration(self):
        for s in self._solvers:
            s.iteration()
        self._iter_counter += 1
        if self._iter_counter % self._eval_every == 0:
            self._log_curr_strat_expl()
            self._evaluate_avg_strats()

    # ---- checkpoint / resume (extension; the reference's CFR classes implement none, SURVEY.md §5)
    def state_dict(self):
        return {"iter_counter": self._iter_counter, "solvers": [s.state_dict() for s in self._solvers]}

    def load_state_dict(self, state):
        self._iter_counter = state["iter_counter"]
        for s, st in zip(self._solvers, state["solvers"]):
            s.load_state_dict(st)

    @staticmethod
    def _rank_path(path):
        """sharded runs: every rank owns different boards -> one file per rank"""
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            return "%s.rank%d_of_%d" % (path, dist.get_rank(), dist.get_world_size())
        return path

    def checkpoint(self, path):
        import torch
        torch.save(self.state_dict(), self._rank_path(path))

    def load_checkpoint(self, path):
        import torch
        # tensors, ints, strings and lists only: no pickled code is ever executed
        self.load_state_dict(torch.load(self._rank_path(path), weights_only=True))

    def _metric(self, t_idx):
        return "Evaluation/" + self._env_bldrs[t_idx].env_cls.WIN_METRIC

    def _log_scalars(self, per_tree_exps, averaged_exp, values):
        for t_idx, v in enumerate(values):
            self._chief_handle.add_scalar(per_tree_exps[t_idx], self._metric(t_idx), self._iter_counter, v)
        self._chief_handle.add_scalar(averaged_exp, self._metric(0), self._iter_counter,
                                      sum(values) / float(len(values)))

    def _log_curr_strat_expl(self):
        self._log_scalars(self._exps_curr_total, self._exp_all_averaged_curr_total,
                          [s.exploitability_current() for s in self._solvers])

    def _evaluate_avg_strats(self):
        self._log_scalars(self._exps_avg_total, self._exp_all_averaged_avg_total,
                          [s.exploitability_average() for s in self._solvers])
