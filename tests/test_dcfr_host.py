"""Discounted CFR without a GPU: the factor table, parameter checks, and DCFR(1, 1, 1) against the pinned Linear CFR oracle.

The DCFR oracles of tests/dcfr_common.py are pinned on the reference-pinned oracles in two ways.  Any (alpha, beta, gamma):
from the same tables, a DCFR half-iteration is a Vanilla CFR half-iteration whose new regrets x are then multiplied by a_t
where x > 0 and by b_t elsewhere, with the same strategies (regret matching ignores the positive factor a_t) and w_t times
Vanilla's addition to the average sums - exactly in float32, to round-off in float64.  And DCFR(1, 1, 1) regrets are Linear
CFR's divided by t + 1 and its average sums are Linear CFR's (pokerrl_b200/dcfr.py).  Both comparisons are teacher-forced: from the tables of a Linear CFR oracle run after k iterations, with the DCFR regrets set to
R_L / (k + 1) and the same strategies, one half-iteration of each seat.  Free-running runs would drift apart where actions
tie: there regret matching turns round-off into a pure strategy (DESIGN.md §2)."""
import math

import numpy as np
import pytest

import cfr2_numpy as o2
from common import make_flat_tree
from dcfr_common import OneSeat, Oracle2DCFR, OracleDCFR
from pokerrl_b200 import dcfr


def test_factors_at_t_1_and_the_float32_rounding():
    f = dcfr.factors(1.5, 0.0, 2.0, 1000)
    assert f.dtype == np.float32 and f.shape == (1000, 3)
    assert tuple(f[0]) == (0.5, 0.5, 1.0)
    for alpha, beta, gamma in ((1.5, 0.0, 2.0), (1.0, 1.0, 1.0), (-0.5, 3.0, 0.5), (400.0, -400.0, 3.0)):
        f = dcfr.factors(alpha, beta, gamma, 1000)
        for i in (0, 1, 2, 9, 996, 997, 999):
            t = float(i + 1)
            for k, e in ((0, alpha), (1, beta)):
                x = t ** e if e * math.log(t) < 700 else math.inf
                want = 1.0 if math.isinf(x) else x / (x + 1.0)
                assert f[i, k] == np.float32(want), (alpha, beta, gamma, i, k)
            assert f[i, 2] == np.float32(t ** gamma)
    lin = dcfr.factors(1, 1, 1, 5)
    assert np.array_equal(lin[:, 2], np.arange(1, 6, dtype=np.float32))
    assert np.array_equal(lin[:, 0], (np.arange(1, 6) / np.arange(2, 7)).astype(np.float32))


@pytest.mark.parametrize("bad", [(math.nan, 0, 2), (1.5, math.inf, 2), (1.5, 0, -math.inf), ("x", 0, 2), (None, 0, 2)])
def test_non_finite_parameters_are_refused(bad):
    with pytest.raises(ValueError):
        dcfr.check_params(*bad)
    with pytest.raises(ValueError):
        dcfr.factors(*bad, 4)


def test_a_weight_beyond_float32_is_refused():
    assert dcfr.factors(1.5, 0.0, 40.0, 9)[8, 2] == np.float32(9.0 ** 40)  # 1.5e38: still finite
    with pytest.raises(ValueError, match="t = 10"):
        dcfr.factors(1.5, 0.0, 40.0, 10)
    tab = dcfr.FactorTable((1.5, 0.0, 40.0), "cpu")
    assert tab.w(8) == float(np.float32(9.0 ** 40))  # grows only as far as asked when the weights leave float32 early
    with pytest.raises(ValueError):
        tab.w(9)


def test_discounted_cfr_refuses_bad_parameters_before_building_anything():
    from pokerrl_b200.cfr import DiscountedCFR
    from pokerrl_b200.game import bet_sets
    from pokerrl_b200.game.games import StandardLeduc
    with pytest.raises(ValueError, match="finite"):
        DiscountedCFR("x", chief_handle=None, game_cls=StandardLeduc, agent_bet_set=bet_sets.POT_ONLY, gamma=math.inf)


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


@pytest.mark.parametrize("game", ["StandardLeduc", "Flop5Holdem 4 boards"])
def test_dcfr_111_is_linear_cfr_rescaled_teacher_forced(game):
    ft, make_tree = _leduc_tree() if game == "StandardLeduc" else _twocard_tree()
    lin = OneSeat(make_tree(), "LinearCFR")
    checked = 0
    for k in (0, 1, 2, 5):
        while lin.iter_counter < k:
            lin.iteration()
        for p in (0, 1):
            base_reg = [None if r is None else r.copy() for r in lin.regret]
            base_sum = [None if s is None else s.copy() for s in lin.avg_sum]
            base_strat = list(lin.t.strategy)
            d = Oracle2DCFR(make_tree(), (1.0, 1.0, 1.0))
            d.iter_counter = k
            d.regret = _flat(ft, base_reg, ft.R) / (k + 1)
            d.avg = _flat(ft, base_sum, ft.R)
            d.t.strategy = list(base_strat)
            d.t.update_reach()
            lin.half_iteration(p)
            d.half_iteration(p)
            reg_l, sum_l = _flat(ft, lin.regret, ft.R), _flat(ft, lin.avg_sum, ft.R)
            scale = np.abs(reg_l).max()
            # seat p's rows: R_D = (d + R_L(k) / (k + 1)) * a with a = float32((k + 1) / (k + 2)), so R_D * (k + 1) / a = R_L;
            # the other seat's rows are those of counter k: R_D * (k + 1) = R_L
            mult = np.full(ft.n_slots, float(k + 1))
            ok = np.ones_like(reg_l, bool)  # average sums: where regret matching is well conditioned (see the module doc)
            rp = np.maximum(reg_l, 0)
            a = float(dcfr.factors(1, 1, 1, k + 1)[k, 0])
            for n in d.dec[ft.kind[d.dec] == p]:
                fs, A = int(ft.first_slot[n]), int(ft.n_children[n])
                mult[fs:fs + A] = (k + 1) / a
                ok[fs:fs + A] = rp[fs:fs + A].sum(axis=0) > 1e-9 * scale
            assert np.abs(d.regret * mult[:, None] - reg_l).max() <= 1e-12 * scale, (game, k, p)
            assert ok.mean() > 0.5
            assert np.abs((d.avg - sum_l) * ok).max() <= 1e-12 * np.abs(sum_l).max(), (game, k, p)
            checked += 1
            # restore the Linear oracle's tables of counter k for the other seat
            lin.regret, lin.avg_sum, lin.t.strategy = base_reg, base_sum, base_strat
            lin.t.update_reach()
    assert checked == 8


def _vanilla_state(make_tree, k):
    van = OneSeat(make_tree(), "VanillaCFR")
    for _ in range(k):
        van.iteration()
    return van


@pytest.mark.parametrize("params", [(1.5, 0.0, 2.0), (0.5, 3.0, 1.25)])
@pytest.mark.parametrize("game", ["StandardLeduc", "Flop5Holdem 4 boards"])
def test_float64_dcfr_step_is_a_vanilla_step_discounted_by_sign(game, params):
    ft, make_tree = _leduc_tree() if game == "StandardLeduc" else _twocard_tree()
    k = 3
    van = _vanilla_state(make_tree, k)
    a, b, w = (float(x) for x in dcfr.factors(*params, k + 1)[k])
    assert a != b and w not in (1.0, float(k + 1))
    for p in (0, 1):
        base_reg = [None if r is None else r.copy() for r in van.regret]
        base_sum = [None if x is None else x.copy() for x in van.avg_sum]
        base_strat = list(van.t.strategy)
        d = Oracle2DCFR(make_tree(), params)
        d.iter_counter = k
        d.regret, d.avg = _flat(ft, base_reg, ft.R), _flat(ft, base_sum, ft.R)
        d.t.strategy = list(base_strat)
        d.t.update_reach()
        van.half_iteration(p)
        d.half_iteration(p)
        x, s_v, s0 = _flat(ft, van.regret, ft.R), _flat(ft, van.avg_sum, ft.R), _flat(ft, base_sum, ft.R)
        mine = np.zeros(ft.n_slots, bool)
        for n in d.dec[ft.kind[d.dec] == p]:
            mine[int(ft.first_slot[n]):int(ft.first_slot[n]) + int(ft.n_children[n])] = True
        assert (x[mine] > 0).any() and (x[mine] < 0).any()
        want = np.where(mine[:, None], x * np.where(x > 0, a, b), x)  # the other seat's rows stay as they were
        assert np.array_equal(d.regret, want), (game, params, p)
        assert np.abs((d.avg - s0) - w * (s_v - s0)).max() <= 1e-12 * w * np.abs(s_v - s0).max(), (game, params, p)
        van.regret, van.avg_sum, van.t.strategy = base_reg, base_sum, base_strat
        van.t.update_reach()


@pytest.mark.parametrize("params", [(1.5, 0.0, 2.0), (0.5, 3.0, 1.25)])
def test_float32_dcfr_rules_are_vanilla_rules_discounted_by_sign(params):
    """OracleDCFR (the bit-exact target of the one-card kernels) against the pinned float32 Vanilla CFR oracle of
    oracle/cfr_numpy.py, from the same state: regrets = Vanilla's new regrets x times a_t / b_t by the sign of x, and the
    average sums = the old sums + (Vanilla's contribution) * w_t, bit for bit"""
    from cfr_numpy import OracleCFR
    ft = make_flat_tree("StandardLeduc")
    van = OracleCFR(ft, "VanillaCFR")
    for _ in range(3):
        van.iteration(evaluate=False)
    k = van.iter_counter
    a, b, w = dcfr.factors(*params, k + 1)[k]
    d = OracleDCFR(ft, params)
    d.iter_counter = k
    d.tree.strategy, d.tree.reach, d.tree.ev = list(van.tree.strategy), van.tree.reach.copy(), van.tree.ev.copy()
    for p in (0, 1):
        nodes = van._nodes_of(p)
        d.regret = [None if r is None else r.copy() for r in van.regret]
        d.avg_strat_sum = [None if x is None else x.copy() for x in van.avg_strat_sum]
        old = [None if x is None else x.copy() for x in van.avg_strat_sum]
        van_reg = [None if r is None else r.copy() for r in van.regret]
        van._compute_regrets(p)
        d._compute_regrets(p)
        van._add_strategy_to_average(p)
        d._add_strategy_to_average(p)
        for n in nodes:
            x = van.regret[n]
            assert np.array_equal(d.regret[n], x * np.where(x > 0, a, b)), (p, n)
            contrib = van.avg_strat_sum[n] - old[n]  # exact: Vanilla added its contribution to these sums
            assert np.array_equal(d.avg_strat_sum[n], old[n] + (van.tree.strategy[n] * van.tree.reach[n, p][:, None]) * w)
            assert np.allclose(d.avg_strat_sum[n] - old[n], contrib * w, rtol=1e-5, atol=0)
        van.regret, van.avg_strat_sum = van_reg, old
