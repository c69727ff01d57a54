"""Short-stack Flop5Holdem on the board engine: the 9-node post-deal shape (stacks of 301 to 900 chips, where the flop's pot-size
bet is all-in; csrc/cfr_board.cu `ShapeFHPShort`) against the same oracles, at the same tolerances, as the 15-node shape.

The checks are those of test_gpu_board_engine, test_gpu_board_avg_pairing, test_gpu_board_br and test_gpu_board_full_game,
run at stack 600 (unless stated otherwise): each test rebinds the game constructors of those modules (`_engine`, `fhp_tree`,
`STACK`) to the short stack and calls their helpers and test bodies, so both shapes are held to one statement of each check."""
import ctypes as C
import functools
import time

import numpy as np
import pytest
import torch

import cfr2_c
import test_gpu_board_avg_pairing as pairing
import test_gpu_board_br as brt
import test_gpu_board_engine as eng
import test_gpu_board_full_game as full
from pokerrl_b200.game import games
from twocard_common import fhp_tree, oracle_tree, random_board_spec

pytestmark = pytest.mark.gpu
G = games.Flop5Holdem
STACK = 600
TOL = 1e-6


def _args(stack):
    return G.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[stack, stack], bet_sizes_list_as_frac_of_pot=[1.0])


def _engine(spec, stack=STACK, **kw):
    from pokerrl_b200.board_engine import BoardCFRSolver
    s = BoardCFRSolver(G, _args(stack), spec, **kw)
    assert s.st["n_local"] == 9 and s.rows_per_board == 8, "not the short shape"
    return s


@pytest.fixture
def at_stack(monkeypatch):
    """at_stack(s): the parity modules build their games at stack s"""
    pairing_engine = pairing._engine

    def bind(stack=STACK):
        monkeypatch.setattr(eng, "_engine", functools.partial(_engine, stack=stack))
        monkeypatch.setattr(eng, "fhp_tree", functools.partial(fhp_tree, stack=stack))
        monkeypatch.setattr(pairing, "_engine", functools.partial(pairing_engine, args=_args(stack)))
        monkeypatch.setattr(brt, "STACK", [stack, stack])
    bind()
    return bind


# ---------------------------------------------------------------------------------------------------------------- kernel parity
def test_root_rows_against_reference_anchored_golden_rows(at_stack):
    """root rows of every golden board with the short shape's own fold and showdown coefficients (derived from its subtree)"""
    eng.test_root_rows_against_reference_anchored_golden_rows()


@pytest.mark.parametrize("algo", ["CFRPlus", "LinearCFR", "VanillaCFR"])
@pytest.mark.parametrize("iso, grid", eng._with_grids([False, True]))
def test_teacher_forced_steps_match_float64_oracle(at_stack, algo, iso, grid):
    """every half-iteration at counters 0 .. 3 from the oracle's tables: 48 skewed random boards or the 57 suit classes of a
    12-card deck, at the default grid, 1 CTA and 7 CTAs"""
    spec = eng._iso_spec() if iso else eng._skewed(random_board_spec(48, 21))
    eng._print_errs("stack 600 %s grid %d" % (algo, grid), eng._teacher_forced(spec, algo, grid=grid))


@pytest.mark.parametrize("grid", [0, 7])
def test_cfr_plus_delay_teacher_forced(at_stack, grid):
    eng._print_errs("stack 600 CFRPlus delay 2 grid %d" % grid,
                    eng._teacher_forced(eng._skewed(random_board_spec(37, 5)), grid=grid, delay=2, warm=1, counters=range(1, 5)))


@pytest.mark.parametrize("algo", ["CFRPlus", "LinearCFR", "VanillaCFR"])
def test_teacher_forced_steps_late_in_a_run(at_stack, algo):
    eng._print_errs("stack 600 %s at iteration 997" % algo,
                    eng._teacher_forced(eng._skewed(random_board_spec(37, 5)), algo, grid=7, warm=3, counters=(997, 998)))


@pytest.mark.parametrize("stack", [301, 900])
def test_teacher_forced_at_the_ends_of_the_range(at_stack, stack):
    """the all-in calls' pot is 602 at stack 301 and 1800 at 900 (the fixed-point format follows the largest pot)"""
    at_stack(stack)
    eng._print_errs("stack %d CFRPlus" % stack, eng._teacher_forced(eng._skewed(random_board_spec(40, 23)), grid=7))


def test_fixed_point_sums_do_not_depend_on_the_grid(at_stack):
    eng.test_fixed_point_sums_do_not_depend_on_the_grid()


def test_shards_reproduce_the_single_device_run_bit_for_bit(at_stack):
    eng.test_shards_reproduce_the_single_device_run_bit_for_bit()


@pytest.mark.parametrize("delay, grid", [(0, 0), (2, 0), (0, 7), (2, 7)])
def test_paired_averaging_equals_the_immediate_form(at_stack, delay, grid):
    pairing.test_paired_averaging_equals_the_immediate_form(delay, grid)


def test_interrupted_pairs_equal_an_uninterrupted_run(at_stack):
    pairing.test_interrupted_pairs_equal_an_uninterrupted_run()


def test_shards_pair_like_one_device(at_stack):
    pairing.test_shards_pair_like_one_device()


@pytest.mark.parametrize("algo", ["LinearCFR", "VanillaCFR"])
def test_linear_and_vanilla_free_running_against_level_engine(at_stack, algo):
    """5 free-running iterations of the board engine, the level engine and the float64 oracle, board against level engine
    within the sanity bound of the deep-stack test (differences printed).  Unlike at deep stacks, the first iteration is not
    held to 1e-5: on this spec at stack 600 seat 0's first update already has hands whose actions tie, so both engines leave
    the oracle's trajectory after one iteration (measured on an H100: board engine 2.8e-4, level engine 1.5e-5, while every
    teacher-forced half-iteration from the same tables stays within 1e-6)."""
    from pokerrl_b200.solver import CFRSolver
    spec = random_board_spec(32, 6)
    ft = fhp_tree(spec, STACK)
    s, lv, orc = _engine(spec, algo=algo), CFRSolver(ft, algo), eng._oracle(ft, algo, lean=True)
    out = []
    for t in range(5):
        for x in (s, lv, orc):
            x.iteration(1)
        cur = [x.exploitability_current() for x in (s, lv, orc)]
        avg = [x.exploitability_average() for x in (s, lv, orc)]
        rel = [abs(v[i] - v[j]) / abs(v[j]) for v in (cur, avg) for i, j in ((0, 1), (0, 2), (1, 2))]
        out.append(rel)
        assert max(rel[0], rel[3]) <= 5e-2, (algo, t, rel)
    print(algo, "stack 600 (current: board-level, board-oracle, level-oracle; average: the same):",
          [" ".join("%.1e" % v for v in r) for r in out])


def test_free_running_trajectory_and_level_engine(at_stack):
    eng.test_free_running_trajectory_and_level_engine()


# ---------------------------------------------------------------------------------------------------------------- best response
def _oracle_expl(spec, agent):
    ft = fhp_tree(spec, STACK)
    orc = cfr2_c.Oracle2CSolver(ft, oracle_tree(ft).board_ranks, "CFRPlus", n_threads=8)
    dec = np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]
    pr = agent.probs(ft, dec)
    for d, n in enumerate(dec):
        fs, fc, A = int(ft.first_slot[n]), int(ft.first_child[n]), int(ft.n_children[n])
        orc.strat[fs:fs + A] = pr[d][:, ft.action[fc:fc + A]].T.astype(np.float64)
    orc.L.orc2_reach(C.byref(orc.t), orc.strat.ctypes.data)
    return orc.compute_ev()


@pytest.mark.parametrize("name", sorted(brt.SPECS))
def test_hash_agent_against_the_float64_oracle_and_the_level_engine(at_stack, name):
    from pokerrl_b200.board_engine import BoardPolicyEvaluator
    spec = brt.SPECS[name]()
    agent = brt.HashAgent(brt._bldr().N_ACTIONS)
    ev = BoardPolicyEvaluator(brt._bldr(), brt.STACK, spec)
    assert ev.rows_per_board == 8
    got = ev.evaluate(agent)
    for what, r in (("oracle", _oracle_expl(spec, agent)), ("level engine", brt._level_expl(spec, agent))):
        err = np.abs(got - r) / np.abs(r)
        print("stack 600 %s: board evaluator vs %s per-seat relative error %.2e %.2e" % (name, what, err[0], err[1]))
        assert np.all(err <= TOL), (name, what, got, r)


def test_chunking_gives_the_same_bits(at_stack):
    from pokerrl_b200.board_engine import BoardPolicyEvaluator
    spec = random_board_spec(300, 17)
    agent = brt.HashAgent(brt._bldr().N_ACTIONS)
    res = {c: BoardPolicyEvaluator(brt._bldr(), brt.STACK, spec, chunk=c).evaluate(agent) for c in (1, 7, None)}
    for c, e in res.items():
        assert np.array_equal(e, res[None]), (c, e, res[None])


def test_trained_agent_br_equals_the_solvers_average_evaluation(at_stack):
    """a CFR+ agent of the short shape (TabularCFREvalAgent.from_cfr): its BR equals the solver's logged _Avg_total bit for bit,
    also after a state_dict round trip; queried on a deep-stack tree it raises"""
    from pokerrl_b200.cfr.CFRPlus import CFRPlus
    from pokerrl_b200.cfr.TabularCFREvalAgent import TabularCFREvalAgent
    from pokerrl_b200.game.PublicTree import PublicTree
    from pokerrl_b200.game.wrappers import HistoryEnvBuilder
    spec = random_board_spec(300, 3)
    cfr, chief, avg = brt._train(CFRPlus, spec, 20, "short")
    assert type(cfr.solvers[0]).__name__ == "BoardCFRSolver"
    br, val, _ = brt._br(cfr, chief, spec, "short")
    print("stack 600 CFR+ 300 boards: _Avg_total %r, BR %r" % (avg, val))
    assert val == avg
    agent = br.eval_agent
    assert agent._board.rows_per_board == 8
    state = agent.state_dict()
    again = TabularCFREvalAgent(t_prof=agent.t_prof)
    again.load_state_dict(state)
    br._eval_agent = again
    br.evaluate(iter_nr=cfr.iter_counter + 1)
    got = [v for k, v in chief.get_experiments().items() if k.startswith("short ") and k.endswith(": BR Total")][0]
    assert got["Evaluation/" + G.WIN_METRIC][-1][1] == avg
    deep = PublicTree(HistoryEnvBuilder(env_cls=G, env_args=_args(20000)), [20000, 20000], None, board_spec=spec)
    deep.build_structure()
    with pytest.raises(ValueError, match="different betting tree"):
        again.get_a_probs_for_public_tree(deep)


def test_mixed_stacks_run_on_board_engines(at_stack):
    """starting_stack_sizes=[600, 20000]: both stacks on BoardCFRSolver (one 9-node, one 15-node shape), the S600 series equal
    to a standalone S600 run bit for bit, and LocalBRMaster over both stacks reproducing each stack's logged average"""
    from pokerrl_b200.cfr.CFRPlus import CFRPlus
    from pokerrl_b200.cfr.TabularCFREvalAgent import TabularCFREvalAgent
    from pokerrl_b200.eval.br.LocalBRMaster import LocalBRMaster
    from pokerrl_b200.rl.base_cls.TrainingProfileBase import TrainingProfileBase
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    spec = random_board_spec(300, 19)
    n_it = 6

    def run(name, stacks):
        chief = ChiefBase(t_prof=None)
        cfr = CFRPlus(name=name, chief_handle=chief, game_cls=G, agent_bet_set=[1.0], starting_stack_sizes=stacks,
                      board_spec=spec)
        for _ in range(n_it):
            cfr.iteration()
        return cfr, chief

    mixed, chief = run("mix", [600, 20000])
    assert [s.rows_per_board for s in mixed.solvers] == [8, 14]
    alone, chief1 = run("one", [600])
    exps, exps1 = chief.get_experiments(), chief1.get_experiments()
    for kind in ("Curr", "Avg"):
        pick = (lambda d, n: [v for k, v in d.items() if k.startswith(n) and "S600" in k and kind in k][0])
        assert pick(exps, "mix_")["Evaluation/" + G.WIN_METRIC] == pick(exps1, "one_")["Evaluation/" + G.WIN_METRIC], kind

    class PerStackAgent(TabularCFREvalAgent):
        """one tabular agent per solver, picked by the stack LocalBRMaster sets"""

        def set_stack_size(self, stack_size):
            super().set_stack_size(stack_size)
            self._board = self.per_stack[stack_size[0]]._board

    t_prof = TrainingProfileBase("mix", G, [1.0], eval_stack_sizes=[[600, 600], [20000, 20000]])
    br = LocalBRMaster(t_prof=t_prof, chief_handle=chief, eval_agent_cls=TabularCFREvalAgent, board_spec=spec)
    assert all(type(gt).__name__ == "BoardPolicyEvaluator" for gt in br._game_trees)
    agent = PerStackAgent(t_prof=t_prof)
    agent.per_stack = {s: TabularCFREvalAgent.from_cfr(t_prof, mixed, tree_idx=i) for i, s in enumerate((600, 20000))}
    br._eval_agent = agent
    br.evaluate(iter_nr=n_it)
    for s in (600, 20000):
        avg = [v for k, v in exps.items() if k.startswith("mix_Avg_total_S%d_" % s)][0]["Evaluation/" + G.WIN_METRIC][-1][1]
        got = [v for k, v in chief.get_experiments().items() if k.startswith("mix ") and "_stack_%d:" % s in k
               and k.endswith(": BR Total")][0]["Evaluation/" + G.WIN_METRIC][-1][1]
        print("mixed stacks: S%d _Avg_total %r, BR %r" % (s, avg, got))
        assert got == avg, s


# ---------------------------------------------------------------------------------------------------------------- full game
@pytest.fixture(scope="module")
def game():
    """test_gpu_board_full_game's engines, synthetic profiles and chunked oracle over all 134 459 classes at stack 600"""
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(full, "_engine", lambda spec, algo: _engine(spec, algo=algo))
        mp.setattr(full, "fhp_tree", functools.partial(fhp_tree, stack=STACK))
        g = full.game._get_wrapped_function()()
    assert g["eng"]["CFRPlus"].rows_per_board == 8
    yield g
    print("stack 600 full game module: %.0f s" % (time.time() - g["t0"]))


def test_full_game_evaluation(game):
    """exploitability of the uniform and the synthetic profile (current and average), chance-node ev / ev_br rows"""
    full.test_full_game_evaluation(game)


@pytest.mark.parametrize("p", [0, 1])
def test_full_game_half_iteration(game, p):
    """one CFR+ (seat 0: defer form, seat 1: paired form) and one Linear CFR half-iteration, every board against the oracle"""
    full.test_full_game_half_iteration(game, p)
