"""Predictive CFR+ without a GPU: its host rules, and its oracles (tests/pcfr_common.py) pinned on the reference-pinned ones.

PCFR+'s step from tables (R, Q) is, piece by piece, a step of an algorithm whose oracle is pinned: its regrets are those of a
CFR+ step from regrets R played with the strategy matching(Q); its instantaneous regrets d are the regrets a Vanilla CFR step
writes from zero regrets under the same strategy, so Q' = max(R' + d, 0); and its addition to the average sums is DCFR's with
the same gamma from a state whose new regrets are R' + d.  Float32 bit for bit; float64 regrets bit for bit, sums to 1e-12."""
import math

import numpy as np
import pytest
import torch

import cfr2_numpy as o2
from common import make_flat_tree
from dcfr_common import OneSeat, Oracle2DCFR, OracleDCFR
from pcfr_common import Oracle2PCFR, OraclePCFR, step_weight
from pokerrl_b200 import _native as nat
from pokerrl_b200 import dcfr
from pokerrl_b200.algorithm import ALGOS, ALL, PREDICTIVE, SUMS, Algorithm, check_identity


# ---------------------------------------------------------------------------------------------------------- host rules
def test_pcfr_plus_is_registered_beside_the_four():
    assert PREDICTIVE == {"PCFRPlus": nat.ALGO_PCFR_PLUS} == {"PCFRPlus": 4}
    assert "PCFRPlus" not in ALGOS and ALL == {**ALGOS, **PREDICTIVE}
    a = Algorithm("PCFRPlus", delay=3, dcfr=(1.0, 0.5, 3.0), device="cpu")
    assert (a.name, a.code, a.delay, a.dcfr, a.pcfr_gamma) == ("PCFRPlus", 4, 0, None, 2.0)
    assert [a.average(t) for t in range(5)] == [SUMS] * 5
    assert a.factor_table(4) is not None
    for name in ALGOS:  # the other four keep their identity keys
        assert set(Algorithm(name, device="cpu").identity()) == {"algo", "delay", "dcfr"}
        assert Algorithm(name, pcfr_gamma=math.nan).pcfr_gamma is None  # not looked at


@pytest.mark.parametrize("gamma", [2.0, 1.0, 3.5])
def test_sum_weight_is_the_dcfr_statement_of_t_to_the_gamma(gamma):
    a = Algorithm("PCFRPlus", device="cpu", pcfr_gamma=gamma)
    f = dcfr.factors(1.5, 0.0, gamma, 998)
    for t in (0, 1, 2, 997):
        w = a.sum_weight(t)
        assert type(w) is float and w == float(f[t, 2]) == float(step_weight(gamma, t)), (gamma, t)


@pytest.mark.parametrize("bad", [math.nan, math.inf, -math.inf, "x", None])
def test_bad_gamma_is_refused_before_anything_is_built(bad):
    from pokerrl_b200.cfr import PredictiveCFRPlus
    from pokerrl_b200.game import bet_sets
    from pokerrl_b200.game.games import StandardLeduc
    with pytest.raises(ValueError, match="gamma"):
        Algorithm("PCFRPlus", pcfr_gamma=bad)
    with pytest.raises(ValueError, match="gamma"):
        PredictiveCFRPlus("x", chief_handle=None, game_cls=StandardLeduc, agent_bet_set=bet_sets.POT_ONLY, gamma=bad)


def test_a_weight_beyond_float32_is_refused():
    a = Algorithm("PCFRPlus", device="cpu", pcfr_gamma=40.0)
    assert a.sum_weight(8) == float(np.float32(9.0 ** 40))
    with pytest.raises(ValueError, match="t = 10"):
        a.sum_weight(9)


def test_identity_and_checkpoint_refusal():
    mine = {"engine": "levels", **Algorithm("PCFRPlus", device="cpu").identity()}
    assert mine == {"engine": "levels", "algo": "PCFRPlus", "delay": 0, "dcfr": None, "pcfr_gamma": 2.0}
    check_identity(dict(mine, iter_counter=5), mine)
    with pytest.raises(ValueError, match="'pcfr_gamma': file has 1.0"):
        check_identity(dict(mine, pcfr_gamma=1.0), mine)
    dcfr_file = {"engine": "levels", **Algorithm("DCFR", device="cpu").identity()}
    with pytest.raises(ValueError, match="'algo'"):
        check_identity(dcfr_file, mine)
    with pytest.raises(ValueError, match="'algo'"):  # and a PCFR+ checkpoint is no DCFR checkpoint
        check_identity(mine, dcfr_file)


def test_level_solver_checkpoint_header():
    import types
    from pokerrl_b200.solver import CFRSolver
    s = CFRSolver.__new__(CFRSolver)
    s.alg, s.avg_f64, s.ft, s.iter_counter, s.modes = Algorithm("PCFRPlus", device="cpu", pcfr_gamma=1.5), False, \
        types.SimpleNamespace(n_nodes=7), 3, [0, 0]
    s.bufs = types.SimpleNamespace(**{n: torch.zeros(2, 3) for n in ("regret", "strat", "avg")})
    st = s.state_dict()
    assert (st["algo"], st["pcfr_gamma"], st["dcfr"]) == ("PCFRPlus", 1.5, None)
    other = CFRSolver.__new__(CFRSolver)
    other.__dict__.update(s.__dict__, alg=Algorithm("PCFRPlus", device="cpu"))
    with pytest.raises(ValueError, match="pcfr_gamma"):
        other.load_state_dict(st)


def test_board_solver_checkpoint_carries_the_predictions():
    """PCFR+'s board checkpoint holds `pred` beside the other tables; the other algorithms' hold no such key"""
    import types
    from pokerrl_b200.board_engine import BoardCFRSolver

    def board(alg):
        s = BoardCFRSolver.__new__(BoardCFRSolver)
        s.alg, s.algo, s.delay, s.device, s.iter_counter, s.modes = alg, alg.code, 0, -1, 3, [0, 0]
        s.rank, s.world, s.n_boards, s.n_boards_total = 0, 1, 5, 5
        s.regret, s.avg = torch.zeros(2, 3), torch.zeros(2, 3)
        s.bufs = types.SimpleNamespace(**{n: torch.zeros(2, 3) for n in ("regret", "strat", "avg")})
        s._pending, s._avg_due = [0.0, 0.0], [-1, -1]
        return s

    s = board(Algorithm("PCFRPlus", device="cpu", pcfr_gamma=1.5))
    s.pred = torch.arange(6, dtype=torch.float32).view(2, 3)
    st = s.state_dict()
    assert torch.equal(st["pred"], s.pred) and st["pcfr_gamma"] == 1.5
    s2 = board(Algorithm("PCFRPlus", device="cpu", pcfr_gamma=1.5))
    s2.pred = torch.zeros(2, 3)
    s2._reach_trunk = lambda *a: None
    s2.load_state_dict(st)
    assert torch.equal(s2.pred, s.pred)
    assert "pred" not in board(Algorithm("DCFR", device="cpu")).state_dict()


# ---------------------------------------------------------------------------------------------------------- float32 oracle
def _cfrp_state(k=3):
    from cfr_numpy import OracleCFR
    ft = make_flat_tree("StandardLeduc")
    o = OracleCFR(ft, "CFRPlus")
    for _ in range(k):
        o.iteration(evaluate=False)
    return ft, o


def test_float32_pcfr_regrets_are_cfr_plus_regrets_under_the_predicted_strategy():
    """from regrets R and a strategy (playing matching(Q)), OraclePCFR's new regrets are the pinned CFR+ oracle's, bit for bit;
    its predictions are max(R' + d) with d the pinned Vanilla oracle's first regrets from the same values"""
    from cfr_numpy import OracleCFR
    ft, cp = _cfrp_state()
    k = cp.iter_counter
    for p in (0, 1):
        pc = OraclePCFR(ft)
        pc.iter_counter = k
        pc.tree.strategy, pc.tree.reach, pc.tree.ev = list(cp.tree.strategy), cp.tree.reach.copy(), cp.tree.ev.copy()
        pc.regret = [None if r is None else r.copy() for r in cp.regret]
        van = OracleCFR(ft, "VanillaCFR")  # counter 0: regrets = d, from the same values
        van.tree.ev = cp.tree.ev.copy()
        keep = [None if r is None else r.copy() for r in cp.regret]
        cp._compute_regrets(p)
        pc._compute_regrets(p)
        van._compute_regrets(p)
        nodes = cp._nodes_of(p)
        assert len(nodes)
        for n in nodes:
            assert np.array_equal(pc.regret[n], cp.regret[n]), (p, n)
            assert np.array_equal(pc.pred[n], np.maximum(cp.regret[n] + van.regret[n], np.float32(0))), (p, n)
        cp.regret = keep


@pytest.mark.parametrize("gamma", [2.0, 1.25])
def test_float32_pcfr_sum_increment_is_dcfrs(gamma):
    ft, cp = _cfrp_state()
    k = cp.iter_counter
    w = step_weight(gamma, k)
    for p in (0, 1):
        pc = OraclePCFR(ft, gamma)
        dc = OracleDCFR(ft, (1.5, 0.0, gamma))
        for o in (pc, dc):
            o.iter_counter = k
            o.tree.strategy, o.tree.reach = list(cp.tree.strategy), cp.tree.reach.copy()
            o.avg_strat_sum = [None if s is None else s.copy() for s in cp.avg_strat]  # some non-zero sums
        old = [None if s is None else s.copy() for s in pc.avg_strat_sum]
        pc._add_strategy_to_average(p)
        dc._add_strategy_to_average(p)
        for n in cp._nodes_of(p):
            assert np.array_equal(pc.avg_strat_sum[n], dc.avg_strat_sum[n]), (p, n)
            want = old[n] + (cp.tree.strategy[n] * cp.tree.reach[n, p][:, None]) * w
            assert np.array_equal(pc.avg_strat_sum[n], want)


# ---------------------------------------------------------------------------------------------------------- float64 oracle
def _leduc_tree():
    from test_oracle_cfr2 import leduc_oracle2
    ft = make_flat_tree("StandardLeduc")
    return ft, lambda: leduc_oracle2(ft)


def _twocard_tree():
    from twocard_common import fhp_tree, oracle_tree, random_board_spec
    ft = fhp_tree(random_board_spec(4, 3))
    t = oracle_tree(ft)
    return ft, lambda: o2.Oracle2Tree(ft, t.hand_cards, t.board_ranks, t.board_prob, t.board_mult, t.sym_perm)


def _flat(ft, per_node, R):
    out = np.zeros((ft.n_slots, R))
    for n in np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]:
        if per_node[n] is not None:
            fs, A = int(ft.first_slot[n]), int(ft.n_children[n])
            out[fs:fs + A] = per_node[n].T
    return out


def _per_node(ft, flat):
    out = [None] * ft.n_nodes
    for n in np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]:
        fs, A = int(ft.first_slot[n]), int(ft.n_children[n])
        out[n] = flat[fs:fs + A].T.copy()
    return out


@pytest.mark.parametrize("game", ["StandardLeduc", "Flop5Holdem 4 boards"])
def test_float64_pcfr_step_is_pinned(game):
    """from (R, Q, S) of a PCFR+ run after k = 3 iterations, one half-iteration of each seat: R' = the pinned CFR+ oracle's
    step from R played with matching(Q), Q' = max(R' + d) with d the pinned Vanilla oracle's step from zero regrets, and
    S' - S = DCFR's increment (gamma alike, a_t = b_t = 1) from a state whose new regrets are R' + d"""
    ft, make_tree = _leduc_tree() if game == "StandardLeduc" else _twocard_tree()
    k, gamma = 3, 2.0
    run = Oracle2PCFR(make_tree(), gamma)
    run.iteration(k)
    errs = []
    for p in (0, 1):
        pc = Oracle2PCFR(make_tree(), gamma)
        pc.iter_counter, pc.regret, pc.pred, pc.avg = k, run.regret.copy(), run.pred.copy(), run.avg.copy()
        pc.set_strategies_from_predictions()
        strat = list(pc.t.strategy)
        mine = np.zeros(ft.n_slots, bool)
        for n in pc.dec[ft.kind[pc.dec] == p]:
            mine[int(ft.first_slot[n]):int(ft.first_slot[n]) + int(ft.n_children[n])] = True

        cp = OneSeat(make_tree(), "CFRPlus")
        cp.iter_counter, cp.regret = k, _per_node(ft, run.regret)
        cp.avg = [None if s is None else s.copy() for s in strat]  # CFR+'s own average: not compared
        cp.t.strategy = list(strat)
        cp.t.update_reach()
        van = OneSeat(make_tree(), "VanillaCFR")
        van.t.strategy = list(strat)
        van.t.update_reach()

        pc.half_iteration(p)
        cp.half_iteration(p)
        van.half_iteration(p)
        r_cp, d = _flat(ft, cp.regret, ft.R), _flat(ft, van.regret, ft.R)
        assert np.array_equal(pc.regret[mine], r_cp[mine]), (game, p)
        assert np.array_equal(pc.regret[~mine], run.regret[~mine]) and np.array_equal(pc.pred[~mine], run.pred[~mine])
        assert np.array_equal(pc.pred[mine], np.maximum(r_cp + d, 0.0)[mine]), (game, p)

        dc = Oracle2DCFR(make_tree(), (400.0, 400.0, gamma))
        assert tuple(dcfr.factors(400.0, 400.0, gamma, k + 1)[k, :2]) == (1.0, 1.0)
        dc.iter_counter, dc.regret, dc.avg = k, np.where(mine[:, None], pc.regret, run.regret), run.avg.copy()
        dc.t.strategy = list(strat)
        dc.t.update_reach()
        dc.half_iteration(p)
        inc_p, inc_d = pc.avg - run.avg, dc.avg - run.avg
        err = float(np.abs(inc_p - inc_d).max() / np.abs(inc_d).max())
        errs.append(err)
        assert err <= 1e-12, (game, p, err)
    print("PCFR+ float64 pinning on %s: sum increments within %.1e of DCFR's" % (game, max(errs)))


def test_float64_average_exploitability_on_standard_leduc():
    """deterministic sanity run: 200 iterations of the float64 oracle; the average strategy's exploitability decreases over
    the run (printed beside CFR+'s)"""
    ft, make_tree = _leduc_tree()
    pc = Oracle2PCFR(make_tree(), 2.0, ev_normalizer=ft.game_cls.EV_NORMALIZER)
    cp = o2.Oracle2CFR(make_tree(), "CFRPlus", ev_normalizer=ft.game_cls.EV_NORMALIZER)
    marks, rows = (1, 10, 50, 100, 200), []
    for t in range(1, 201):
        pc.iteration()
        cp.iteration()
        if t in marks:
            rows.append((t, pc.exploitability_average(), cp.exploitability_average()))
    for t, a, b in rows:
        print("StandardLeduc iteration %3d: average-strategy exploitability PCFR+ %.4f  CFR+ %.4f mbb/g" % (t, a, b))
    vals = [a for _, a, _ in rows]
    assert all(x > y for x, y in zip(vals, vals[1:])), vals
    assert vals[-1] < 0.05 * vals[0]
