"""Predictive CFR+ on every engine against its oracles (tests/pcfr_common.py).

One-card games: bit for bit against the float32 oracle (the kernels evaluate in its dtypes and operation order), with the
persistent multi-iteration launch (the weights of many iterations inside one launch) and the per-iteration launch.
Two-card level engine: the float64 oracle, at the tolerances of the DCFR tests (test_gpu_dcfr.py) for the regrets and for the
first iteration.  The prediction max(R + d, 0) cancels where R is close to -d, so the float32 round-off of d (1e-7 of the
values) becomes a larger relative error of the prediction and of the strategy matched from it where a hand's prediction
mass is small (H100: 4.4e-5 on the unweighted strategy of 16 random boards after iteration 3, with the regrets at 2.4e-7).
The strategy rows are therefore compared weighted by that mass relative to the largest prediction, as the board engine tests
weigh their average sums (test_gpu_dcfr.py).  From the second iteration on the strategy and the exploitabilities, and from
the third the regrets, are held to 1e-5: the free-running strategies part where the weights are small and feed back into the
values (H100: 6.6e-6 on the current strategy's exploitability of the Limit Hold'em flop sub-game after iteration 2, 2.4e-6
on the regrets of the random boards after iteration 4).  The one-card kernels, which
run the same rules, match the float32 oracle bit for bit.  The level-split schedule of the sharded engine equals the plain
solver bit for bit.
Board engine: teacher-forced half-iterations against the float64 oracle at 1e-6 (R, Q and the conditioned sums), both
shapes, several grids, early and late counters; grid independence and shards bit for bit; best response and checkpoints."""
import numpy as np
import pytest
import torch

from common import make_flat_tree
from pcfr_common import Oracle2PCFR, OraclePCFR
from test_gpu_board_engine import _rel
from twocard_common import fhp_tree, oracle_tree, random_board_spec

pytestmark = pytest.mark.gpu
TOL = 1e-6
TOL_PRED = 1e-5  # strategies matched from predictions, from the second iteration on (see the module doc)
GAMMA = 2.0


def _slot_tables(ft, per_node):
    """oracle [R, A] per decision node -> float64 [n_slots, R]"""
    out = np.zeros((ft.n_slots, ft.R))
    for n in np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]:
        fs, A = int(ft.first_slot[n]), int(ft.n_children[n])
        out[fs:fs + A] = np.asarray(per_node[n], np.float64).T
    return out


def _gpu(t, ft):
    return t.cpu().numpy()[:, :ft.R].astype(np.float64)


@pytest.mark.parametrize("name", ["StandardLeduc", "NLLeduc_POT", "BigLeduc"])
def test_one_card_pcfr_bit_exact(name):
    """50 iterations along one oracle run: the per-iteration launch checked after every iteration, the persistent launch
    (ten iterations and their weights inside one launch) after every tenth; exploitability every tenth iteration"""
    from pokerrl_b200.solver import CFRSolver
    ft = make_flat_tree(name)
    per_it = CFRSolver(ft, "PCFRPlus", persistent=False, pcfr_gamma=GAMMA)
    pers = CFRSolver(ft, "PCFRPlus", persistent=True, pcfr_gamma=GAMMA)
    o = OraclePCFR(ft, GAMMA)
    assert per_it.exploitability_current() == pers.exploitability_current() == o.curr_series[0][1]
    for t in range(1, 51):
        per_it.iteration(1)
        if t % 10 == 0:
            pers.iteration(10)
        o.iteration(evaluate=False)
        ref = [_slot_tables(ft, x) for x in (o.regret, o.tree.strategy, o.avg_strat_sum)]
        for s in ((per_it, pers) if t % 10 == 0 else (per_it,)):
            for tab, r in zip((s.bufs.regret, s.bufs.strat, s.bufs.avg), ref):
                assert np.array_equal(_gpu(tab, ft), r), (t, s.persistent)
        if t % 10 == 0:
            o.tree.compute_ev()
            o._log_curr()
            avg = o.evaluate_avg()
            for s in (per_it, pers):
                assert s.exploitability_current() == o.curr_series[-1][1], (t, s.persistent)
                assert s.exploitability_average() == avg, (t, s.persistent)
    print("PCFR+ %s: 50 iterations bit for bit, average exploitability %.6g mbb/g" % (name, o.evaluate_avg()))


def _level_vs_oracle(ft, iters, regrets=True):
    """exploitability of the current and the average strategy after each iteration; regrets=True: the regret table and the
    strategy (regret matching of the predictions) too"""
    from pokerrl_b200.solver import CFRSolver
    s = CFRSolver(ft, "PCFRPlus", pcfr_gamma=GAMMA)
    c = Oracle2PCFR(oracle_tree(ft), GAMMA, ev_normalizer=ft.game_cls.EV_NORMALIZER)
    for t in range(iters):
        s.iteration(1)
        c.iteration()
        errs = []
        if regrets:
            errs.append(_rel(_gpu(s.bufs.regret, ft), c.regret))
            cond = np.zeros(c.pred.shape)  # per (node, hand): prediction mass / largest prediction, on the node's rows
            for n in c.dec:
                fs, A = int(ft.first_slot[n]), int(ft.n_children[n])
                cond[fs:fs + A] = np.minimum(c.pred[fs:fs + A].sum(axis=0) / max(c.pred.max(), 1e-300), 1.0)
            errs.append(float(np.abs(_gpu(s.bufs.strat, ft) - _slot_tables(ft, c.t.strategy)).__mul__(cond).max()))
            assert errs[0] <= (TOL if t < 2 else TOL_PRED), (t, errs)
            assert errs[1] <= (TOL if t == 0 else TOL_PRED), (t, errs)
        a, b = s.exploitability_current(), c.exploitability_current()
        errs.append(abs(a - b) / abs(b))
        a, b = s.exploitability_average(), c.exploitability_average()
        errs.append(abs(a - b) / abs(b))
        print("PCFR+ two-card iteration %d: relative errors %s" % (t, " ".join("%.1e" % e for e in errs)))
        assert max(errs[-2:]) <= (TOL if t == 0 else TOL_PRED), (t, errs)


def test_two_card_level_engine_random_boards():
    _level_vs_oracle(fhp_tree(random_board_spec(16, 2)), 4)


def test_two_card_level_engine_multi_street_subgame():
    """the Limit Hold'em flop sub-game of test_gpu_twocard.py, by exploitability, for two free-running iterations (as for
    DCFR: later, hands whose actions tie take a strategy decided by round-off)"""
    from twocard_common import hulh_flop_subgame
    _level_vs_oracle(hulh_flop_subgame([[20, 21, 22], [30, 31]]), 2, regrets=False)


def test_sharded_schedule_single_rank_equals_plain_solver():
    """the level-split sweeps of the sharded engine (prl_value_levels / prl_reach_levels) reproduce the plain solver"""
    from pokerrl_b200.distributed import ShardedCFRSolver
    from pokerrl_b200.game import games
    from pokerrl_b200.solver import CFRSolver
    spec = random_board_spec(20, 5)
    g = games.Flop5Holdem
    args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[20000, 20000], bet_sizes_list_as_frac_of_pot=[1.0])
    a = CFRSolver(fhp_tree(spec), "PCFRPlus", pcfr_gamma=GAMMA)
    b = ShardedCFRSolver(g, args, spec, "PCFRPlus", pcfr_gamma=GAMMA)
    for _ in range(3):
        a.iteration(1)
        b.iteration(1)
        assert a.exploitability_current() == b.exploitability_current()
        assert a.exploitability_average() == b.exploitability_average()
    for x, y in ((a.bufs.regret, b.bufs.regret), (a.bufs.strat, b.bufs.strat), (a.bufs.avg, b.bufs.avg)):
        assert torch.equal(x, y)


def test_checkpoint_round_trip_and_refusal(tmp_path):
    from pokerrl_b200.cfr import PredictiveCFRPlus
    from pokerrl_b200.game import bet_sets, games
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    G = games.StandardLeduc

    def make(name, chief, **kw):
        return PredictiveCFRPlus(name=name, chief_handle=chief, game_cls=G, agent_bet_set=bet_sets.POT_ONLY, **kw)

    chief = ChiefBase(t_prof=None)
    cfr = make("p", chief)
    for _ in range(10):
        cfr.iteration()
    cfr.checkpoint(str(tmp_path / "ck.pt"))
    for _ in range(10):
        cfr.iteration()
    key = "p_Avg_total_S%d_PCFRPlus" % G.DEFAULT_STACK_SIZE
    avg = chief.get_experiments()[key]["Evaluation/" + G.WIN_METRIC][-1][1]
    chief2 = ChiefBase(t_prof=None)
    again = make("p", chief2)
    again.load_checkpoint(str(tmp_path / "ck.pt"))
    for _ in range(10):
        again.iteration()
    assert again.iter_counter == 20
    for t in ("regret", "strat", "avg"):
        assert torch.equal(getattr(again.solvers[0].bufs, t), getattr(cfr.solvers[0].bufs, t))
    assert chief2.get_experiments()[key]["Evaluation/" + G.WIN_METRIC][-1][1] == avg
    with pytest.raises(ValueError, match="pcfr_gamma"):
        make("o", ChiefBase(t_prof=None), gamma=1.0).load_checkpoint(str(tmp_path / "ck.pt"))


def test_tabular_agent_best_response_equals_logged_average():
    """LocalBRMaster on the tabular agent of a trained PCFR+ (the SUMS path) gives the logged average exploitability"""
    from pokerrl_b200.cfr import PredictiveCFRPlus
    from pokerrl_b200.game import bet_sets, games
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    from pokerrl_b200.cfr.TabularCFREvalAgent import TabularCFREvalAgent
    from pokerrl_b200.eval.br.LocalBRMaster import LocalBRMaster
    from pokerrl_b200.rl.base_cls.TrainingProfileBase import TrainingProfileBase
    G = games.StandardLeduc
    S = G.DEFAULT_STACK_SIZE
    chief = ChiefBase(t_prof=None)
    cfr = PredictiveCFRPlus(name="b", chief_handle=chief, game_cls=G, agent_bet_set=bet_sets.POT_ONLY)
    for _ in range(20):
        cfr.iteration()
    avg = chief.get_experiments()["b_Avg_total_S%d_PCFRPlus" % S]["Evaluation/" + G.WIN_METRIC][-1][1]
    t_prof = TrainingProfileBase("b", G, bet_sets.POT_ONLY)
    br = LocalBRMaster(t_prof=t_prof, chief_handle=chief, eval_agent_cls=TabularCFREvalAgent)
    br._eval_agent = TabularCFREvalAgent.from_cfr(t_prof, cfr)
    br.evaluate(iter_nr=cfr.iter_counter)
    val = chief.get_experiments()["b AVG_stack_%d: BR Total" % S]["Evaluation/" + G.WIN_METRIC][-1][1]
    print("PCFR+ StandardLeduc, 20 iterations: logged average %.9g, LocalBRMaster %.9g mbb/g" % (avg, val))
    assert abs(val - avg) <= TOL * abs(avg), (val, avg)


# ---------------------------------------------------------------------------------------------------------- board engine
def _board_engine(spec, stack=20000, **kw):
    from pokerrl_b200.board_engine import BoardCFRSolver
    from pokerrl_b200.game import games
    g = games.Flop5Holdem
    args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[stack, stack], bet_sizes_list_as_frac_of_pot=[1.0])
    return BoardCFRSolver(g, args, spec, algo="PCFRPlus", pcfr_gamma=GAMMA, **kw)


def _board_teacher_forced(spec, stack=20000, grid=0, warm=0, counters=range(4)):
    """every half-iteration at the counters starts from the float64 oracle's tables (R, Q, S; the trunk's strategy = matching
    of its Q): exploitability of the current and the average strategy, then R, Q and the average sums after one seat's
    update, at 1e-6 (average sums weighted by the conditioning of the strategies above them, as in test_gpu_dcfr.py; Q and S
    of the post-deal rows, R everywhere)"""
    from test_gpu_board_engine import _live_mask, _skewed  # noqa: F401
    ft = fhp_tree(spec, stack)
    orc = Oracle2PCFR(oracle_tree(ft), GAMMA, ev_normalizer=ft.game_cls.EV_NORMALIZER)
    s = _board_engine(spec, stack, grid=grid)
    orc.iteration(warm)
    live = _live_mask(ft, spec.boards)
    post = np.zeros(ft.n_slots, bool)
    post[s.n_trunk_slots:] = True
    dec = orc.dec
    worst = 0.0
    for t in counters:
        orc.iter_counter = t
        for p in (0, 1):
            orc.set_strategies_from_predictions()
            s.load_natural_tables(ft, orc.regret, orc.avg, orc.pred)
            s.iter_counter = t
            e1 = e2 = 0.0
            if p == 0:
                a, b = s.exploitability_current(), orc.exploitability_current()
                e1 = abs(a - b) / abs(b)
                if t > 0:
                    a, b = s.exploitability_average(), orc.exploitability_average()
                    e2 = abs(a - b) / abs(b)
            s._update_begin(p)
            s._update_end(p)
            orc.half_iteration(p)
            reg, avg, pred = (x.cpu().numpy()[:, :ft.R].astype(np.float64) for x in s.natural_tables(ft))
            e3 = _rel(reg * live, orc.regret * live)
            e4 = _rel((pred * live)[post], (orc.pred * live)[post])
            cond = np.zeros(orc.pred.shape)
            node_cond = {}
            for n in dec[ft.kind[dec] == p]:
                fs, A = ft.first_slot[n], ft.n_children[n]
                c = np.minimum(orc.pred[fs:fs + A].sum(axis=0) / max(np.abs(orc.pred).max(), 1e-300), 1.0)
                a = ft.parent[n]
                while a >= 0 and a not in node_cond:
                    a = ft.parent[a]
                node_cond[n] = c * (node_cond[a] if a >= 0 else 1.0)
                cond[fs:fs + A] = node_cond[n]
            e5 = float((np.abs(avg - orc.avg) * cond * live).max() / max(np.abs(orc.avg).max(), 1e-300))
            # the trunk's stored strategy against matching of the oracle's predictions, weighted by the prediction mass as
            # the level-engine strategies above (matching a small mass amplifies the round-off of d)
            trunk = pred[:s.n_trunk_slots]
            want, wt = np.zeros_like(trunk), np.zeros_like(trunk)
            for n in dec:
                fs, A = int(ft.first_slot[n]), int(ft.n_children[n])
                if fs < s.n_trunk_slots:
                    want[fs:fs + A] = orc.matching(orc.pred[fs:fs + A], A).T
                    wt[fs:fs + A] = np.minimum(orc.pred[fs:fs + A].sum(axis=0) / max(orc.pred.max(), 1e-300), 1.0)
            e6 = float((np.abs(trunk - want) * wt).max())
            worst = max(worst, e1, e2, e3, e4, e5, e6)
            print("PCFR+ board stack %d grid %d counter %d seat %d: %.1e %.1e %.1e %.1e %.1e %.1e"
                  % (stack, grid, t, p, e1, e2, e3, e4, e5, e6))
            assert max(e1, e2, e3, e4, e5, e6) <= TOL, (stack, grid, t, p, e1, e2, e3, e4, e5, e6)
    return worst


@pytest.mark.parametrize("stack, grid", [(20000, 0), (20000, 1), (20000, 7), (600, 0), (600, 1), (600, 7)])
def test_board_engine_teacher_forced(stack, grid):
    from test_gpu_board_engine import _skewed
    _board_teacher_forced(_skewed(random_board_spec(40, 17)), stack, grid)


@pytest.mark.parametrize("stack", [20000, 600])
def test_board_engine_teacher_forced_late_counters(stack):
    """w_t about 1e6 in the sweep, the trunk and the pending average contribution"""
    from test_gpu_board_engine import _skewed
    _board_teacher_forced(_skewed(random_board_spec(37, 5)), stack, grid=7, warm=3, counters=(997, 998))


def test_board_engine_sums_independent_of_grid_and_shards_equal_one_device():
    from test_gpu_board_engine import _per_board, _skewed
    spec = _skewed(random_board_spec(64, 33))
    runs = []
    for grid in (0, 1, 7, 64):
        s = _board_engine(spec, grid=grid)
        s.iteration(3)
        cur = s.exploitability_current()
        s.flush_average()
        runs.append((s.regret.clone(), s.pred.clone(), s.bufs.regret.clone(), s.bufs.strat.clone(), s.avg.clone(),
                     s.bufs.avg.clone(), cur, s.exploitability_average()))
    for r in runs[1:]:
        assert all(torch.equal(x, y) for x, y in zip(r[:6], runs[0][:6])) and r[6:] == runs[0][6:]
    for n_boards in (3, 1):  # one rank with a single board / without any
        spec = random_board_spec(n_boards, 8)
        one = _board_engine(spec)
        parts = [_board_engine(spec, rank=r, world=2, reduce_fn=lambda t: None) for r in range(2)]
        for it in range(3):
            one.iteration(1)
            for p in (0, 1):
                for e in parts:
                    e._update_begin(p)
                tot = parts[0].w_total + parts[1].w_total
                for e in parts:
                    e.w_total.copy_(tot)
                    e._update_end(p)
            for e in parts:
                e.iter_counter += 1
        one.flush_average()
        for r, e in enumerate(parts):
            e.flush_average()
            for tab in ("regret", "pred", "avg"):
                assert torch.equal(_per_board(e, getattr(e, tab)), _per_board(one, getattr(one, tab))[r::2]), tab
            for tab in ("regret", "strat", "avg"):
                assert torch.equal(getattr(e.bufs, tab), getattr(one.bufs, tab)), tab


def test_board_engine_trained_agent_br_and_checkpoints(tmp_path):
    from pokerrl_b200.cfr import PredictiveCFRPlus
    from pokerrl_b200.game import games
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    from test_gpu_board_br import _br
    G = games.Flop5Holdem
    spec = random_board_spec(300, 3)

    def make(name, chief, **kw):
        return PredictiveCFRPlus(name=name, chief_handle=chief, game_cls=G, agent_bet_set=[1.0], starting_stack_sizes=[20000],
                                 eval_every=20, board_spec=spec, **kw)

    chief = ChiefBase(t_prof=None)
    cfr = make("d", chief)
    assert type(cfr.solvers[0]).__name__ == "BoardCFRSolver"
    for _ in range(10):
        cfr.iteration()
    cfr.checkpoint(str(tmp_path / "ck.pt"))
    for _ in range(10):
        cfr.iteration()
    avg = chief.get_experiments()["d_Avg_total_S20000_PCFRPlus"]["Evaluation/" + G.WIN_METRIC][-1][1]
    _, val, _ = _br(cfr, chief, spec, "d")
    print("PCFR+ board engine, 300 boards, 20 iterations: logged average %.9g, LocalBRMaster %.9g mbb/g" % (avg, val))
    assert abs(val - avg) <= TOL * abs(avg), (val, avg)
    chief2 = ChiefBase(t_prof=None)
    again = make("d", chief2)
    again.load_checkpoint(str(tmp_path / "ck.pt"))
    for _ in range(10):
        again.iteration()
    assert again.iter_counter == 20
    for tab in ("regret", "pred", "avg"):
        assert torch.equal(getattr(again.solvers[0], tab), getattr(cfr.solvers[0], tab)), tab
    assert chief2.get_experiments()["d_Avg_total_S20000_PCFRPlus"]["Evaluation/" + G.WIN_METRIC][-1][1] == avg
    with pytest.raises(ValueError, match="pcfr_gamma"):
        make("o", ChiefBase(t_prof=None), gamma=1.0).load_checkpoint(str(tmp_path / "ck.pt"))


def test_predictive_cfr_plus_picks_the_engine_and_names_the_experiments():
    from pokerrl_b200.cfr import PredictiveCFRPlus
    from pokerrl_b200.game import bet_sets, games
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    chief = ChiefBase(t_prof=None)
    fhp = PredictiveCFRPlus("f", chief, games.Flop5Holdem, [1.0], board_spec=random_board_spec(8, 1), gamma=3.0)
    assert type(fhp.solvers[0]).__name__ == "BoardCFRSolver" and fhp.solvers[0].alg.pcfr_gamma == 3.0
    assert fhp.solvers[0].pred is not None
    led = PredictiveCFRPlus("l", chief, games.StandardLeduc, bet_sets.POT_ONLY, gamma=1.5)
    assert type(led.solvers[0]).__name__ == "CFRSolver" and led.solvers[0].alg.pcfr_gamma == 1.5
    led.iteration()
    fhp.iteration()
    names = set(chief.get_experiments())
    S = games.Flop5Holdem.DEFAULT_STACK_SIZE
    for n in ("f_Curr_S%d_total_PCFRPlus" % S, "f_Avg_total_S%d_PCFRPlus" % S, "l_Curr_total_averaged_PCFRPlus",
              "l_Avg_total_averaged_PCFRPlus", "l_Avg_total_S%d_PCFRPlus" % games.StandardLeduc.DEFAULT_STACK_SIZE):
        assert n in names, (n, sorted(names))
