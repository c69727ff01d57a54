"""Restricted Nash response on the board engine (board_engine.BoardRNRSolver, cfr.RestrictedNashResponse) against the float64
restatement of tests/rnr_common.py.

  * p = 0 runs the plain CFR+ instantiations: both games equal a CFR+ BoardCFRSolver bit for bit.
  * Teacher-forced half-iterations (both seats of both games, p in {0.25, 0.5, 1}, both compiled shapes, several grids, CFR+
    with delay): the regrets and the conditioned average from the oracle's tables at 1e-6, as the other board-engine tests.
  * The chance sums are integers: every grid gives the same bits.
  * Exploitation and exploitability against the oracle; the counter-agent's best response (LocalBRMaster) against the logged
    seat-averaged exploitability; the exploitation never above the model's best-response value.
  * Checkpoints continue bit for bit and refuse another p or another model."""
import numpy as np
import pytest
import torch

from rnr_common import Oracle2RNR, TableAgent, random_model
from test_gpu_board_engine import _live_mask, _rel, _skewed
from twocard_common import fhp_tree, oracle_tree, random_board_spec

pytestmark = pytest.mark.gpu
TOL = 1e-6


def _args(stack):
    from pokerrl_b200.game import games
    g = games.Flop5Holdem
    return g, g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[stack, stack], bet_sizes_list_as_frac_of_pot=[1.0])


def _games(spec, model, p, stack=20000, delay=0, grid=0):
    """both games (exploiter seat 0, 1) with the model's tables filled"""
    from pokerrl_b200 import board_engine
    from pokerrl_b200.game.wrappers import HistoryEnvBuilder
    g, args = _args(stack)
    pair = [board_engine.BoardRNRSolver(g, args, s, p, spec, delay, grid=grid) for s in (0, 1)]
    bldr = HistoryEnvBuilder(env_cls=g, env_args=args)
    ev = board_engine.BoardPolicyEvaluator(bldr, stack_size=[stack, stack], board_spec=spec)
    trunk = ev.model_reach(TableAgent(fhp_tree(spec, stack), model, bldr.N_ACTIONS), {x.seat: x.model_reach for x in pair})
    for x in pair:
        x.set_model(trunk)
    return pair


@pytest.mark.parametrize("stack", [20000, 600])
def test_p0_equals_cfr_plus_bit_for_bit(stack):
    from pokerrl_b200.board_engine import BoardCFRSolver
    spec = _skewed(random_board_spec(48, 11))
    g, args = _args(stack)
    ref = BoardCFRSolver(g, args, spec, algo="CFRPlus")
    ref.iteration(6)
    ref.flush_average()
    for x in _games(spec, random_model(fhp_tree(spec, stack), 1), 0.0, stack):
        x.iteration(6)
        x.flush_average()
        for a, b in ((x.regret, ref.regret), (x.avg, ref.avg), (x.bufs.regret, ref.bufs.regret), (x.bufs.strat, ref.bufs.strat),
                     (x.bufs.avg, ref.bufs.avg)):
            assert torch.equal(a, b)


def _teacher_forced(spec, stack, p, grid=0, delay=0, counters=(2, 3), warm=2, paired=False):
    """paired: each update starts with a pending averaging step of the previous iteration, so that it runs the paired form
    (the step and its own in one pass over the average rows), else the deferred form and prl_board_avg_flush"""
    ft = fhp_tree(spec, stack)
    model = random_model(ft, 7)
    live = _live_mask(ft, spec.boards)
    worst = 0.0
    for x in _games(spec, model, p, stack, delay, grid):
        orc = Oracle2RNR(oracle_tree(ft), x.seat, p, model, delay)
        for _ in range(warm):
            orc.iteration()
        for t in counters:
            orc.iter_counter = t
            for q in (0, 1):
                if q != x.seat and p == 1.0:
                    continue
                x.load_natural_tables(ft, orc.regret, orc.avg)
                x.set_trunk_strategy_from_regrets()
                x.iter_counter = t
                if paired and t - 1 >= delay:
                    x._avg_due[q] = t - 1
                    orc.pending_step(q, t - 1)
                x._update_begin(q)
                x._update_end(q)
                orc.half_iteration(q)
                reg, avg = (y.cpu().numpy()[:, :ft.R].astype(np.float64) for y in x.natural_tables(ft))
                # the average step adds regret matching of the new regrets, which amplifies their round-off where a hand's
                # positive regret mass is small: its rows are weighted by that mass relative to the largest regret, as the
                # other board-engine tests weigh their averages
                cond = np.ones(orc.avg.shape)
                big = max(np.abs(orc.regret).max(), 1e-300)
                for n in orc.dec[ft.kind[orc.dec] == q]:
                    fs, A = int(ft.first_slot[n]), int(ft.n_children[n])
                    cond[fs:fs + A] = np.minimum(np.maximum(orc.regret[fs:fs + A], 0).sum(axis=0) / big, 1.0)
                e1 = _rel(reg * live, orc.regret * live)
                e2 = float((np.abs(avg - orc.avg) * cond * live).max() / max(np.abs(orc.avg).max(), 1e-300))
                worst = max(worst, e1, e2)
                print("RNR stack %d p %.2f grid %d delay %d paired %d exploiter %d counter %d seat %d: regret %.1e avg %.1e"
                      % (stack, p, grid, delay, paired, x.seat, t, q, e1, e2))
                assert max(e1, e2) <= TOL, (stack, p, grid, x.seat, t, q, e1, e2)
    return worst


@pytest.mark.parametrize("stack", [20000, 600])
@pytest.mark.parametrize("p", [0.25, 0.5, 1.0])
def test_teacher_forced_half_iterations(stack, p):
    _teacher_forced(_skewed(random_board_spec(48, 17)), stack, p)


@pytest.mark.parametrize("stack, p", [(20000, 0.5), (600, 0.5), (20000, 1.0)])
def test_teacher_forced_paired_average(stack, p):
    _teacher_forced(_skewed(random_board_spec(48, 19)), stack, p, paired=True)


@pytest.mark.parametrize("grid", [1, 7])
def test_teacher_forced_grids_and_suit_classes(grid):
    from test_gpu_board_engine import _iso_spec
    _teacher_forced(_iso_spec(), 20000, 0.5, grid=grid)


def test_teacher_forced_cfr_plus_delay():
    _teacher_forced(_skewed(random_board_spec(48, 23)), 20000, 0.5, delay=2, counters=(1, 2, 3, 4), warm=1)


def test_tables_do_not_depend_on_the_grid():
    spec = _skewed(random_board_spec(48, 29))
    model = random_model(fhp_tree(spec), 3)
    runs = []
    for grid in (0, 1, 7):
        out = []
        for x in _games(spec, model, 0.5, grid=grid):
            x.iteration(4)
            x.flush_average()
            out += [x.regret.clone(), x.avg.clone(), x.bufs.regret.clone(), x.bufs.avg.clone(), x.rnr_values()]
        runs.append(out)
    for r in runs[1:]:
        for a, b in zip(r, runs[0]):
            assert torch.equal(a, b) if isinstance(a, torch.Tensor) else a == b


@pytest.mark.parametrize("stack", [20000, 600])
def test_evaluation_against_the_oracle(stack):
    spec = _skewed(random_board_spec(48, 31))
    ft = fhp_tree(spec, stack)
    model = random_model(ft, 5)
    for x in _games(spec, model, 0.5, stack):
        orc = Oracle2RNR(oracle_tree(ft), x.seat, 0.5, model)
        for _ in range(3):
            orc.iteration()
        x.load_natural_tables(ft, orc.regret, orc.avg)
        x.set_trunk_strategy_from_regrets()
        x.iter_counter = 3
        got, want = x.rnr_values(), orc.exploitation_exploitability()
        err = [abs(a - b) / max(abs(b), 1e-12) for a, b in zip(got, want)]
        print("RNR evaluation stack %d exploiter %d: exploitation %.9g / %.9g, exploitability %.9g / %.9g, relative errors %.1e %.1e"
              % (stack, x.seat, got[0], want[0], got[1], want[1], *err))
        assert max(err) <= TOL, (got, want)


def _chief():
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    return ChiefBase(t_prof=None)


def _br_of(agent, spec, name, chief):
    from pokerrl_b200.cfr.TabularCFREvalAgent import TabularCFREvalAgent
    from pokerrl_b200.eval.br.LocalBRMaster import LocalBRMaster
    from pokerrl_b200.game import games
    from pokerrl_b200.rl.base_cls.TrainingProfileBase import TrainingProfileBase
    G = games.Flop5Holdem
    t_prof = TrainingProfileBase(name, G, [1.0], eval_stack_sizes=[[20000, 20000]])
    br = LocalBRMaster(t_prof=t_prof, chief_handle=chief, eval_agent_cls=TabularCFREvalAgent, board_spec=spec)
    br._eval_agent = TabularCFREvalAgent(t_prof=t_prof)
    br._eval_agent._board = agent
    br.evaluate(iter_nr=0)
    got = [v for k, v in chief.get_experiments().items() if k.startswith(name + " ") and k.endswith(": BR Total")][0]
    return got["Evaluation/" + G.WIN_METRIC][-1][1]


def _cfr_model(spec, iters=10):
    from pokerrl_b200.board_engine import BoardCFRSolver, BoardPolicyTables
    g, args = _args(20000)
    s = BoardCFRSolver(g, args, spec, algo="CFRPlus")
    s.iteration(iters)
    return BoardPolicyTables.from_solver(s)


def test_public_class_counter_agent_and_bounds(tmp_path):
    from pokerrl_b200.cfr import RestrictedNashResponse
    from pokerrl_b200.game import games
    G = games.Flop5Holdem
    spec = random_board_spec(200, 41)
    model = _cfr_model(spec)
    model_br = _br_of(model, spec, "m", _chief())
    chief = _chief()
    rnr = RestrictedNashResponse("r", chief, G, [1.0], model, 0.5, starting_stack_sizes=[20000], eval_every=5, board_spec=spec)
    for _ in range(20):
        rnr.iteration()
    exps = chief.get_experiments()
    metric = "Evaluation/" + G.WIN_METRIC
    exploitation = [v for _, v in exps["r_Exploitation_S20000_RNR"][metric]]
    exploitability = [v for _, v in exps["r_Exploitability_S20000_RNR"][metric]]
    assert len(exploitation) == len(exploitability) == 4
    assert [v for _, v in exps["r_Exploitation_averaged_RNR"][metric]] == exploitation
    counter = _br_of(rnr.counter_agent(), spec, "c", _chief())
    print("RNR p 0.5, 200 boards, 20 iterations: model BR %.6g, exploitation %s, exploitability %s, counter-agent BR %.9g mbb/g"
          % (model_br, exploitation, exploitability, counter))
    # the same quantity summed two ways: br_1(sigma_0) + br_0(sigma_1) from each game's root best-response value, and
    # LocalBRMaster's (br_0 - ev_0) + (br_1 - ev_1) of the combined profile, whose ev_0 + ev_1 cancels only up to rounding;
    # each is a float32 rounding of a double sum, so they may differ by about one float32 ulp (H100: 5.3e-8 relative)
    assert abs(counter - exploitability[-1]) <= 2.5e-7 * abs(counter), (counter, exploitability[-1])
    assert all(e <= model_br + 1e-6 * abs(model_br) for e in exploitation), (exploitation, model_br)
    # checkpoints: continue bit for bit; another p or another model is refused
    rnr.checkpoint(str(tmp_path / "ck.pt"))
    for _ in range(5):
        rnr.iteration()
    again = RestrictedNashResponse("r", _chief(), G, [1.0], model, 0.5, starting_stack_sizes=[20000], eval_every=5, board_spec=spec)
    again.load_checkpoint(str(tmp_path / "ck.pt"))
    for _ in range(5):
        again.iteration()
    for a, b in zip(again.games[0], rnr.games[0]):
        a.flush_average()
        b.flush_average()
        for t in ("regret", "avg"):
            assert torch.equal(getattr(a, t), getattr(b, t)), t
    with pytest.raises(ValueError, match="rnr_p"):
        RestrictedNashResponse("o", _chief(), G, [1.0], model, 0.25, starting_stack_sizes=[20000],
                               board_spec=spec).load_checkpoint(str(tmp_path / "ck.pt"))
    with pytest.raises(ValueError, match="rnr_model"):
        RestrictedNashResponse("o", _chief(), G, [1.0], _cfr_model(spec, 3), 0.5, starting_stack_sizes=[20000],
                               board_spec=spec).load_checkpoint(str(tmp_path / "ck.pt"))


def test_p1_exploitation_approaches_the_best_response():
    """p = 1: the exploiter learns a best response to the model, its exploitation rises towards the model's BR value (H100:
    the gap fell from 2.62 mbb/g after 20 iterations to 0.034 after 200; the bound asks for a tenth of the first gap)"""
    from pokerrl_b200.cfr import RestrictedNashResponse
    from pokerrl_b200.game import games
    G = games.Flop5Holdem
    spec = random_board_spec(100, 43)
    model = _cfr_model(spec)
    model_br = _br_of(model, spec, "m", _chief())
    chief = _chief()
    rnr = RestrictedNashResponse("q", chief, G, [1.0], model, 1.0, starting_stack_sizes=[20000], eval_every=20, board_spec=spec)
    for _ in range(200):
        rnr.iteration()
    got = [v for _, v in chief.get_experiments()["q_Exploitation_S20000_RNR"]["Evaluation/" + G.WIN_METRIC]]
    gaps = [model_br - v for v in got]
    print("RNR p 1, 100 boards: model BR %.6g mbb/g, gap after every 20 iterations %s" % (model_br, ["%.4g" % x for x in gaps]))
    assert all(g >= -1e-6 * abs(model_br) for g in gaps)
    assert gaps[-1] <= 0.1 * gaps[0]
