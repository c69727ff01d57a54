"""Discounted CFR on every engine against its oracles (tests/dcfr_common.py).

One-card games: bit for bit against the float32 oracle (the kernels evaluate in its dtypes and operation order), with the
persistent multi-iteration launch (factors of many iterations inside one launch) and the per-iteration launch.
Two-card level engine and board engine: the float64 oracle at the tolerances of the Linear CFR tests (test_gpu_twocard.py,
test_gpu_board_engine.py)."""
import numpy as np
import pytest
import torch

import cfr2_numpy as o2
from common import make_flat_tree
from dcfr_common import Oracle2DCFR, OracleDCFR
from test_gpu_board_engine import _live_mask, _natural, _per_board, _rel, _skewed
from twocard_common import fhp_tree, oracle_tree, random_board_spec

pytestmark = pytest.mark.gpu
TOL = 1e-6
PARAMS = (1.5, 0.0, 2.0)


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
def test_one_card_dcfr_bit_exact(name):
    """50 iterations along one oracle run: the per-iteration launch checked after every iteration, the persistent launch
    (ten iterations and their factors inside one launch) after every tenth; exploitability every tenth iteration"""
    from pokerrl_b200.solver import CFRSolver
    ft = make_flat_tree(name)
    per_it = CFRSolver(ft, "DCFR", persistent=False, dcfr=PARAMS)
    pers = CFRSolver(ft, "DCFR", persistent=True, dcfr=PARAMS)
    o = OracleDCFR(ft, PARAMS)
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


def _level_vs_oracle(ft, iters, regrets=True):
    """exploitability of the current and the average strategy after each iteration; regrets=True: the regret table too"""
    from pokerrl_b200.solver import CFRSolver
    s = CFRSolver(ft, "DCFR", dcfr=PARAMS)
    c = Oracle2DCFR(oracle_tree(ft), PARAMS, ev_normalizer=ft.game_cls.EV_NORMALIZER)
    for t in range(iters):
        s.iteration(1)
        c.iteration()
        if regrets:
            err = _rel(_gpu(s.bufs.regret, ft), c.regret)
            assert err <= (TOL if t < 2 else 2e-6), (t, err)
        a, b = s.exploitability_current(), c.exploitability_current()
        assert abs(a - b) <= TOL * abs(b), (t, a, b)
        a, b = s.exploitability_average(), c.exploitability_average()
        assert abs(a - b) <= TOL * abs(b), (t, a, b)


def test_two_card_level_engine_random_boards():
    _level_vs_oracle(fhp_tree(random_board_spec(16, 2)), 4)


def test_two_card_level_engine_multi_street_subgame():
    """the Limit Hold'em flop sub-game of test_gpu_twocard.py, checked like Linear CFR there, by exploitability, for two
    free-running iterations: from the third on, hands whose actions tie take a strategy decided by round-off (H100: 3.6e-6
    relative on the current strategy's exploitability after iteration 3)"""
    from twocard_common import hulh_flop_subgame
    _level_vs_oracle(hulh_flop_subgame([[20, 21, 22], [30, 31]]), 2, regrets=False)


def _board_engine(spec, stack=20000, **kw):
    from pokerrl_b200.board_engine import BoardCFRSolver
    from pokerrl_b200.game import games
    g = games.Flop5Holdem
    args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[stack, stack], bet_sizes_list_as_frac_of_pot=[1.0])
    return BoardCFRSolver(g, args, spec, algo="DCFR", dcfr=PARAMS, **kw)


def _teacher_forced(spec, stack=20000, grid=0, warm=0, counters=range(4)):
    """every half-iteration at the counters starts from the float64 oracle's tables: exploitability of the current and of the
    average strategy, then the regrets and average sums after one seat's update, at 1e-6 (masks and conditioning as in
    test_gpu_board_engine._teacher_forced for Linear CFR)"""
    ft = fhp_tree(spec, stack)
    orc = Oracle2DCFR(oracle_tree(ft), PARAMS, ev_normalizer=ft.game_cls.EV_NORMALIZER)
    s = _board_engine(spec, stack, grid=grid)
    orc.iteration(warm)
    live = _live_mask(ft, spec.boards)
    dec = orc.dec
    for t in counters:
        orc.iter_counter = t
        for p in (0, 1):
            orc.set_strategies_from_regrets()
            s.load_natural_tables(ft, orc.regret, orc.avg)
            s.set_trunk_strategy_from_regrets()
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
            reg, avg = _natural(s, ft)
            e3 = _rel(reg * live, orc.regret * live)
            rp = np.maximum(orc.regret, 0.0)
            cond = np.zeros(orc.regret.shape)
            node_cond = {}
            for n in dec[ft.kind[dec] == p]:
                fs, A = ft.first_slot[n], ft.n_children[n]
                c = np.minimum(rp[fs:fs + A].sum(axis=0) / np.abs(orc.regret).max(), 1.0)
                a = ft.parent[n]
                while a >= 0 and a not in node_cond:
                    a = ft.parent[a]
                node_cond[n] = c * (node_cond[a] if a >= 0 else 1.0)
                cond[fs:fs + A] = node_cond[n]
            e4 = float((np.abs(avg - orc.avg) * cond * live).max() / max(np.abs(orc.avg).max(), 1e-300))
            print("DCFR stack %d grid %d counter %d seat %d: %.1e %.1e %.1e %.1e" % (stack, grid, t, p, e1, e2, e3, e4))
            assert max(e1, e2, e3, e4) <= TOL, (stack, grid, t, p, e1, e2, e3, e4)


@pytest.mark.parametrize("stack, grid", [(20000, 0), (20000, 1), (20000, 7), (600, 0), (600, 7)])
def test_board_engine_teacher_forced(stack, grid):
    _teacher_forced(_skewed(random_board_spec(40, 17)), stack, grid)


@pytest.mark.parametrize("stack", [20000, 600])
def test_board_engine_teacher_forced_late_counters(stack):
    """a_t close to 1 and w_t about 1e6 in the sweep, the trunk and the pending average contribution"""
    _teacher_forced(_skewed(random_board_spec(37, 5)), stack, grid=7, warm=3, counters=(997, 998))


def test_board_engine_sums_independent_of_grid_and_shards_equal_one_device():
    spec = _skewed(random_board_spec(64, 33))
    runs = []
    for grid in (0, 1, 7, 64):
        s = _board_engine(spec, grid=grid)
        s.iteration(3)
        cur = s.exploitability_current()
        s.flush_average()
        runs.append((s.regret.clone(), s.bufs.regret.clone(), s.avg.clone(), s.bufs.avg.clone(), cur, s.exploitability_average()))
    for r in runs[1:]:
        assert all(torch.equal(x, y) for x, y in zip(r[:4], runs[0][:4])) and r[4:] == runs[0][4:]
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
            assert torch.equal(_per_board(e, e.regret), _per_board(one, one.regret)[r::2])
            assert torch.equal(_per_board(e, e.avg), _per_board(one, one.avg)[r::2])
            assert torch.equal(e.bufs.regret, one.bufs.regret) and torch.equal(e.bufs.avg, one.bufs.avg)


def test_trained_agent_br_and_checkpoints(tmp_path):
    from pokerrl_b200.cfr import DiscountedCFR
    from pokerrl_b200.game import games
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    from test_gpu_board_br import _br
    G = games.Flop5Holdem
    spec = random_board_spec(300, 3)

    def make(name, chief, **kw):
        return DiscountedCFR(name=name, chief_handle=chief, game_cls=G, agent_bet_set=[1.0], starting_stack_sizes=[20000],
                             eval_every=20, board_spec=spec, **kw)

    chief = ChiefBase(t_prof=None)
    cfr = make("d", chief)
    assert type(cfr.solvers[0]).__name__ == "BoardCFRSolver"
    for _ in range(10):
        cfr.iteration()
    cfr.checkpoint(str(tmp_path / "ck.pt"))
    for _ in range(10):
        cfr.iteration()
    avg = chief.get_experiments()["d_Avg_total_S20000_DCFR"]["Evaluation/" + G.WIN_METRIC][-1][1]
    _, val, _ = _br(cfr, chief, spec, "d")
    assert abs(val - avg) <= TOL * abs(avg), (val, avg)
    chief2 = ChiefBase(t_prof=None)
    again = make("d", chief2)
    again.load_checkpoint(str(tmp_path / "ck.pt"))
    for _ in range(10):
        again.iteration()
    assert again.iter_counter == 20
    assert torch.equal(again.solvers[0].regret, cfr.solvers[0].regret)
    assert torch.equal(again.solvers[0].avg, cfr.solvers[0].avg)
    assert chief2.get_experiments()["d_Avg_total_S20000_DCFR"]["Evaluation/" + G.WIN_METRIC][-1][1] == avg
    other = make("o", ChiefBase(t_prof=None), gamma=1.0)
    with pytest.raises(ValueError, match="dcfr"):
        other.load_checkpoint(str(tmp_path / "ck.pt"))


def test_discounted_cfr_picks_the_engine_and_names_the_experiments():
    from pokerrl_b200.cfr import DiscountedCFR
    from pokerrl_b200.game import bet_sets, games
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    chief = ChiefBase(t_prof=None)
    fhp = DiscountedCFR("f", chief, games.Flop5Holdem, [1.0], board_spec=random_board_spec(8, 1), alpha=1.0, beta=0.5,
                        gamma=3.0)
    assert type(fhp.solvers[0]).__name__ == "BoardCFRSolver" and fhp.solvers[0].dcfr == (1.0, 0.5, 3.0)
    led = DiscountedCFR("l", chief, games.StandardLeduc, bet_sets.POT_ONLY)
    assert type(led.solvers[0]).__name__ == "CFRSolver" and led.solvers[0].dcfr == (1.5, 0.0, 2.0)
    led.iteration()
    names = set(chief.get_experiments())
    S = games.Flop5Holdem.DEFAULT_STACK_SIZE
    for n in ("f_Curr_S%d_total_DCFR" % S, "f_Avg_total_S%d_DCFR" % S, "l_Curr_total_averaged_DCFR",
              "l_Avg_total_averaged_DCFR", "l_Avg_total_S%d_DCFR" % games.StandardLeduc.DEFAULT_STACK_SIZE):
        assert n in names, (n, sorted(names))
