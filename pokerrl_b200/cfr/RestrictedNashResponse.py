"""Restricted Nash response (Johanson, Zinkevich & Bowling, "Computing Robust Counter-Strategies", NIPS 2007) on the board
engine: a strategy that exploits a fixed agent (the model) while bounding its own exploitability.

Before the deal a coin seen only by the opponent makes it play the model with probability p and a free strategy otherwise; the
exploiter's equilibrium strategy of that game is the counter-strategy.  p = 0 gives an equilibrium, p = 1 a best response to the
model in the limit, and sweeping p traces the exploitation / exploitability trade-off.  A PokerRL agent plays both seats, so
one object solves two such games, one per exploiter seat s, each by CFR+ (`board_engine.BoardRNRSolver`).

Logged every `eval_every` iterations, per stack and seat-averaged, in the game's WIN_METRIC:
  <name>_Exploitation_S<stack>_RNR     the value of seat s's average strategy against the model's seat 1 - s
  <name>_Exploitability_S<stack>_RNR   the value of a best response of seat 1 - s to seat s's average
and <name>_Exploitation_averaged_RNR / <name>_Exploitability_averaged_RNR over the stacks."""
import copy

import numpy as np

from pokerrl_b200.game.games import get_env_cls_from_str
from pokerrl_b200.game.wrappers import HistoryEnvBuilder


class _TablesAgent:
    """BoardPolicyTables as an agent PublicTree.agent_strategy_table can query"""

    def __init__(self, tables, n_actions):
        self._tables, self._n_actions = tables, n_actions

    def get_a_probs_for_public_tree(self, tree):
        return self._tables.answer_tree(tree.flat, self._n_actions)


def _model_fingerprint(model, stack):
    """board_engine.abstract_fingerprint of the betting tree the model plays at `stack`: the tree its BoardPolicyTables were
    computed on, or the tree of its environment builder (EvalAgentBase.env_bldr); ValueError for a model with neither"""
    from pokerrl_b200 import board_engine
    from pokerrl_b200.game.flat_tree import FlatTree
    tables = model if isinstance(model, board_engine.BoardPolicyTables) else getattr(model, "_board", None)
    if isinstance(tables, board_engine.BoardPolicyTables):
        return tables.fingerprint
    bldr = getattr(model, "env_bldr", None)
    if bldr is None:
        raise ValueError("the model must be an EvalAgentBase or BoardPolicyTables (its betting tree is checked)")
    try:
        ft1 = FlatTree(bldr.env_cls, bldr.args_for_stack([stack, stack]), board_spec=board_engine._one_board_spec())
    except Exception as e:  # noqa: BLE001 - a game the board engine's trees cannot express is a different tree
        raise ValueError("the model plays a game the board engine does not run (%s)" % type(e).__name__) from e
    return board_engine.abstract_fingerprint(ft1)


class RestrictedNashResponse:
    def __init__(self, name, chief_handle, game_cls, agent_bet_set, model, p, starting_stack_sizes=None, delay=0,
                 eval_every=1, device=None, board_spec=None):
        import torch.distributed as dist
        from pokerrl_b200 import board_engine
        from pokerrl_b200.game.flat_tree import FlatTree
        self.p = board_engine.rnr_probability(p)
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            raise ValueError("the restricted Nash response runs on one GPU (torch.distributed world size %d)"
                             % dist.get_world_size())
        self._name, self._chief_handle, self.delay = name, chief_handle, int(delay)
        self._eval_every = max(1, int(eval_every))
        self._starting_stack_sizes = ([game_cls.DEFAULT_STACK_SIZE] if starting_stack_sizes is None
                                      else copy.deepcopy(starting_stack_sizes))
        env_cls = get_env_cls_from_str(game_cls.__name__)
        self._env_args = [game_cls.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[s, s], bet_sizes_list_as_frac_of_pot=agent_bet_set)
                          for s in self._starting_stack_sizes]
        self._env_bldrs = [HistoryEnvBuilder(env_cls=env_cls, env_args=a) for a in self._env_args]
        # every refusal before anything large is allocated
        for s, a in zip(self._starting_stack_sizes, self._env_args):
            if not board_engine.supports(env_cls, a, "CFRPlus"):
                raise ValueError("the restricted Nash response runs on the board engine: %s at stack %d is not a game it "
                                 "supports" % (game_cls.__name__, s))
        for s, a in zip(self._starting_stack_sizes, self._env_args):
            mine = board_engine.abstract_fingerprint(FlatTree(env_cls, a, board_spec=board_engine._one_board_spec()))
            if _model_fingerprint(model, s) != mine:
                raise ValueError("the model plays a different betting tree (game / stack / bet set) at stack %d" % s)
        if isinstance(model, board_engine.BoardPolicyTables):
            model = _TablesAgent(model, self._env_bldrs[0].N_ACTIONS)
        self._games = []
        for bldr, s, a in zip(self._env_bldrs, self._starting_stack_sizes, self._env_args):
            pair = [board_engine.BoardRNRSolver(env_cls, a, 0, self.p, board_spec, self.delay, device)]
            pair.append(board_engine.BoardRNRSolver(env_cls, a, 1, self.p, board_spec, self.delay, device, share_boards=pair[0]))
            ev = board_engine.BoardPolicyEvaluator(bldr, stack_size=[s, s], board_spec=pair[0].spec_full, device=pair[0].device)
            trunk = ev.model_reach(model, {g.seat: g.model_reach for g in pair})
            del ev
            for g in pair:
                g.set_model(trunk)
            self._games.append(pair)
        ch, S = chief_handle, self._starting_stack_sizes
        self._exps_exploitation = [ch.create_experiment("%s_Exploitation_S%d_RNR" % (name, s)) for s in S]
        self._exps_exploitability = [ch.create_experiment("%s_Exploitability_S%d_RNR" % (name, s)) for s in S]
        self._exp_exploitation_avg = ch.create_experiment(name + "_Exploitation_averaged_RNR")
        self._exp_exploitability_avg = ch.create_experiment(name + "_Exploitability_averaged_RNR")
        self._iter_counter = 0

    name = property(lambda s: s._name)
    iter_counter = property(lambda s: s._iter_counter)
    games = property(lambda s: s._games)  # [stack][exploiter seat] BoardRNRSolver

    def reset(self):
        self._iter_counter = 0
        for pair in self._games:
            for g in pair:
                g.reset()

    def iteration(self):
        """one CFR+ iteration of each game"""
        for pair in self._games:
            for g in pair:
                g.iteration()
        self._iter_counter += 1
        if self._iter_counter % self._eval_every == 0 and self._iter_counter > self.delay:
            self.evaluate()

    def values(self):
        """[stack] (exploitation, exploitability), seat-averaged, in the game's WIN_METRIC"""
        out = []
        for bldr, pair in zip(self._env_bldrs, self._games):
            v = np.array([g.rnr_values() for g in pair]) * bldr.env_cls.EV_NORMALIZER
            out.append((float(v[:, 0].sum() / 2), float(v[:, 1].sum() / 2)))
        return out

    def evaluate(self):
        vals = self.values()
        ch, it = self._chief_handle, self._iter_counter
        for k, (exploitation, exploitability) in enumerate(vals):
            metric = "Evaluation/" + self._env_bldrs[k].env_cls.WIN_METRIC
            ch.add_scalar(self._exps_exploitation[k], metric, it, exploitation)
            ch.add_scalar(self._exps_exploitability[k], metric, it, exploitability)
        metric = "Evaluation/" + self._env_bldrs[0].env_cls.WIN_METRIC
        ch.add_scalar(self._exp_exploitation_avg, metric, it, sum(v[0] for v in vals) / len(vals))
        ch.add_scalar(self._exp_exploitability_avg, metric, it, sum(v[1] for v in vals) / len(vals))
        return vals

    def counter_agent(self, stack_idx=0):
        """the counter-strategy as a BoardPolicyTables agent: seat s's post-deal and trunk rows from game s's average"""
        from pokerrl_b200 import board_engine
        pair = self._games[stack_idx]
        a = board_engine.BoardPolicyTables.from_solver(pair[0])
        b = board_engine.BoardPolicyTables.from_solver(pair[1])
        g, st = pair[1], pair[1].st
        seat1 = [g.local_rows[c][0] for c in g.local_rows if st["kind"][st["parent"][c]] == 1]
        rows = a.rows.view(a.n_cls, a.rows_per_board, -1)
        rows[:, seat1] = b.rows.view(b.n_cls, b.rows_per_board, -1)[:, seat1]
        ft = g.ft1
        for n in range(g.chance_node + 1):
            if ft.kind[n] == 1 and ft.first_child[n] >= 0:
                fs, A = int(ft.first_slot[n]), int(ft.n_children[n])
                a.trunk[fs:fs + A] = b.trunk[fs:fs + A]
        return a

    # ---- checkpoints, as the other algorithms (the identity of each game adds p, its seat and the model's digest)
    def state_dict(self):
        return {"iter_counter": self._iter_counter, "games": [[g.state_dict() for g in pair] for pair in self._games]}

    def load_state_dict(self, state):
        if len(state["games"]) != len(self._games):
            raise ValueError("checkpoint has %d stacks, this run %d" % (len(state["games"]), len(self._games)))
        from pokerrl_b200 import algorithm
        for pair, sts in zip(self._games, state["games"]):  # every game's identity before any table is touched
            for g, st in zip(pair, sts):
                algorithm.check_identity(st, g._identity())
        for pair, sts in zip(self._games, state["games"]):
            for g, st in zip(pair, sts):
                g.load_state_dict(st)
        self._iter_counter = state["iter_counter"]

    def checkpoint(self, path):
        import torch
        torch.save(self.state_dict(), path)

    def load_checkpoint(self, path):
        import torch
        self.load_state_dict(torch.load(path, weights_only=True))
