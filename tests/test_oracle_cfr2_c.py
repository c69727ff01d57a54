"""oracle/cfr2_oracle.c (float64, O(R) sorted-sweep showdowns, OpenMP) against oracle/cfr2_numpy.py (dense sign
matrices) on whole sweeps and CFR iterations - two independent formulations of the same statements.  DCFR and PCFR+
against their numpy restatements on the same trees (tests/dcfr_common.py, tests/pcfr_common.py)."""
import numpy as np
import pytest

import cfr2_c
import cfr2_numpy as o2
from twocard_common import fhp_tree, hulh_flop_subgame, oracle_tree, random_board_spec


def _pair(ft, algo, lean=False):
    orc = oracle_tree(ft)
    return o2.Oracle2CFR(orc, algo, ev_normalizer=ft.game_cls.EV_NORMALIZER), \
        cfr2_c.Oracle2CSolver(ft, orc.board_ranks, algo, n_threads=4, lean=lean)


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize("algo", ["CFRPlus", "LinearCFR", "VanillaCFR"])
def test_iterations_match_numpy_oracle(algo):
    ft = fhp_tree(random_board_spec(6, 3))
    a, b = _pair(ft, algo)
    ea, eb = a.t.compute_ev(), b.compute_ev()
    assert _rel(b.reach, a.t.reach) < 1e-13 and _rel(b.ev, a.t.ev) < 1e-12 and _rel(b.ev_br, a.t.ev_br) < 1e-12
    assert _rel(eb, ea) < 1e-12
    for t in range(3):
        a.iteration()
        b.iteration()
        ref = np.zeros_like(b.regret)
        for n in a.t.decision_nodes():
            ref[ft.first_slot[n]:ft.first_slot[n] + ft.n_children[n]] = a.regret[n].T
        assert _rel(b.regret, ref) < 1e-10, t
        x, y = a.exploitability_current(), b.exploitability_current()
        assert abs(x - y) <= 1e-10 * abs(x), (t, x, y)
        x, y = a.exploitability_average(), b.exploitability_average()
        assert abs(x - y) <= 1e-10 * abs(x), (t, x, y)


def test_lean_schedule_is_the_same_trajectory():
    """computing only ev[p] without BR in the update sweeps (the GPU's schedule, bench.py's CPU arm) changes nothing"""
    ft = fhp_tree(random_board_spec(5, 9))
    orc = oracle_tree(ft)
    a = cfr2_c.Oracle2CSolver(ft, orc.board_ranks, "CFRPlus", n_threads=2, lean=False)
    b = cfr2_c.Oracle2CSolver(ft, orc.board_ranks, "CFRPlus", n_threads=2, lean=True)
    a.iteration(3)
    b.iteration(3)
    assert np.array_equal(a.regret, b.regret) and np.array_equal(a.avg, b.avg)
    assert a.exploitability_average() == b.exploitability_average()


def test_multi_street_and_isomorphic_trees():
    ft = hulh_flop_subgame([[20, 21, 22], [30, 31]])
    a, b = _pair(ft, "LinearCFR")
    a.iteration()
    b.iteration()
    x, y = a.exploitability_average(), b.exploitability_average()
    assert abs(x - y) <= 1e-10 * abs(x)
    # from the second iteration on, regrets that are exactly 0 in exact arithmetic come out as +-1e-17 depending on the
    # summation order and regret matching turns them into pure strategies (the reference's own sensitivity, SURVEY.md
    # headline 5): two float64 implementations then agree to ~1e-7, not to round-off
    a.iteration()
    b.iteration()
    x, y = a.exploitability_average(), b.exploitability_average()
    assert abs(x - y) <= 1e-6 * abs(x)
    from pokerrl_b200.game.games import FlopHoldemRules
    from pokerrl_b200.game.holdem_boards import BoardSpec
    iso = fhp_tree(BoardSpec.full_game(FlopHoldemRules, isomorphic=True, deck_subset=[0, 1, 2, 3, 48, 49, 50, 51]))
    a, b = _pair(iso, "CFRPlus")
    a.iteration()
    b.iteration()
    x, y = a.exploitability_current(), b.exploitability_current()
    assert abs(x - y) <= 1e-10 * abs(x)


@pytest.mark.parametrize("stack", [20000, 600])
@pytest.mark.parametrize("algo", ["DCFR", "PCFRPlus"])
def test_dcfr_and_pcfr_iterations_match_numpy_oracles(algo, stack):
    """DCFR and PCFR+ iterations of the C oracle against the numpy restatements (tests/dcfr_common.py, tests/pcfr_common.py),
    both seats' half-iterations at counters 0 .. 3 and at 997 (w_t about 1e6): values, regrets, predictions, sums and
    both exploitabilities; both sides take the float32 factors of pokerrl_b200.dcfr"""
    from dcfr_common import Oracle2DCFR
    from pcfr_common import Oracle2PCFR
    ft = fhp_tree(random_board_spec(6, 3), stack)
    orc = oracle_tree(ft)
    norm = ft.game_cls.EV_NORMALIZER
    a = Oracle2DCFR(orc, ev_normalizer=norm) if algo == "DCFR" else Oracle2PCFR(orc, 2.0, ev_normalizer=norm)
    b = cfr2_c.Oracle2CSolver(ft, orc.board_ranks, algo, n_threads=4)
    for t in (0, 1, 2, 3, 997):
        a.iter_counter = b.iter_counter = t
        for p in (0, 1):
            a.half_iteration(p)
            b.half_iteration(p)
            errs = [_rel(b.ev, a.t.ev), _rel(b.reach, a.t.reach), _rel(b.regret, a.regret), _rel(b.avg, a.avg)]
            if algo == "PCFRPlus":
                errs.append(_rel(b.pred, a.pred))
                assert (b.regret >= 0).all() and (b.pred >= 0).all()
            assert max(errs) <= 1e-12, (t, p, errs)
        x, y = a.exploitability_current(), b.exploitability_current()
        assert abs(x - y) <= 1e-12 * abs(x), (t, x, y)
        x, y = a.exploitability_average(), b.exploitability_average()
        assert abs(x - y) <= 1e-12 * abs(x), (t, x, y)
        print("%s stack %d counter %d: relative errors %s" % (algo, stack, t, " ".join("%.1e" % e for e in errs)))
