"""GPU parity of the two-card (Hold'em family) LEVEL-engine sweeps against the float64 oracle (oracle/cfr2_numpy.py, whose
terminal rows are pinned on the reference's hand strengths, tests/test_oracle_twocard_rows.py).

Tolerances (achieved errors are printed with -s): BASELINE.json's bar, 1e-6 of the largest
magnitude of the compared array / relative for exploitability; regrets of free-running iterations 2 and 3 and the trunk
regrets of the isomorphism test get 2e-6 / 5e-6 (float32 round-off decides ties in regret matching, SURVEY headline 5)."""
import numpy as np
import pytest

import cfr2_numpy as o2
from pokerrl_b200.game.holdem_boards import BoardSpec
from pokerrl_b200.game.games import FlopHoldemRules
from twocard_common import fhp_tree, oracle_tree, random_board_spec

pytestmark = pytest.mark.gpu


ACHIEVED = {}


def _close(name, mine, ref, tol=1e-6):
    scale = np.abs(ref).max()
    err = np.abs(mine - ref).max()
    ACHIEVED[name] = max(ACHIEVED.get(name, 0.0), float(err / scale))
    print("level engine vs float64 oracle: %-14s relative error %.2e (tolerance %.0e)" % (name, err / scale, tol))
    assert err <= tol * scale, (name, err, scale)


def _expl_close(name, a, b, tol=1e-6):
    err = abs(a - b) / abs(b)
    ACHIEVED[name] = max(ACHIEVED.get(name, 0.0), float(err))
    print("level engine vs float64 oracle: %-14s relative error %.2e (tolerance %.0e)" % (name, err, tol))
    assert err <= tol, (name, a, b)


def _node_vec(s_t, ft):  # torch [2, N, ld] -> [N, 2, R]
    return s_t.cpu().numpy()[:, :, :ft.R].transpose(1, 0, 2).astype(np.float64)


def test_uniform_profile_values_random_boards():
    from pokerrl_b200.solver import CFRSolver
    ft = fhp_tree(random_board_spec(24, 1))
    orc = oracle_tree(ft)
    orc.fill_uniform()
    expl = orc.compute_ev()
    s = CFRSolver(ft, "CFRPlus")
    m = s.exploitability_current()
    _close("reach", _node_vec(s.bufs.reach, ft), orc.reach)
    _close("ev", _node_vec(s.bufs.ev, ft), orc.ev)
    _close("ev_br", _node_vec(s.bufs.ev_br, ft), orc.ev_br)
    ref_m = float(sum(expl) / 2 * ft.game_cls.EV_NORMALIZER)
    _expl_close("expl uniform", m, ref_m, tol=1e-6)
    # zero-sum check of the reference (ValueFiller.py:98) at the root
    assert abs((orc.ev[0] * orc.reach[0]).sum()) < 1e-6 * np.abs(orc.ev[0]).max()


@pytest.mark.parametrize("algo", ["CFRPlus", "LinearCFR", "VanillaCFR"])
def test_cfr_iterations_match_oracle(algo):
    from pokerrl_b200.solver import CFRSolver
    ft = fhp_tree(random_board_spec(16, 2))
    s = CFRSolver(ft, algo)
    c = o2.Oracle2CFR(oracle_tree(ft), algo, ev_normalizer=ft.game_cls.EV_NORMALIZER)
    for t in range(4):
        s.iteration(1)
        c.iteration()
        reg = s.bufs.regret.cpu().numpy()[:, :ft.R].astype(np.float64)
        ref = np.zeros_like(reg)
        for n in c.t.decision_nodes():
            ref[ft.first_slot[n]:ft.first_slot[n] + ft.n_children[n]] = c.regret[n].T
        _close("regret it%d" % t, reg, ref, tol=1e-6 if t < 2 else 2e-6)
        a, b = s.exploitability_current(), c.exploitability_current()
        _expl_close("expl cur it%d" % t, a, b, tol=1e-6)
        a, b = s.exploitability_average(), c.exploitability_average()
        _expl_close("expl avg it%d" % t, a, b, tol=1e-6)


def test_suit_isomorphism_equals_full_enumeration():
    """Representatives + orbit weights + symmetrisation reproduce the evaluation over every board of a
    suit-closed deck subset (ranks 2 and A in four suits: 56 boards)."""
    from pokerrl_b200.solver import CFRSolver
    deck = [0, 1, 2, 3, 48, 49, 50, 51]
    full = fhp_tree(BoardSpec.full_game(FlopHoldemRules, isomorphic=False, deck_subset=deck))
    iso = fhp_tree(BoardSpec.full_game(FlopHoldemRules, isomorphic=True, deck_subset=deck))
    assert iso.board_spec.boards.shape[0] < full.board_spec.boards.shape[0] == 56
    s_full, s_iso = CFRSolver(full, "CFRPlus"), CFRSolver(iso, "CFRPlus")
    orc = o2.Oracle2CFR(oracle_tree(full), "CFRPlus", ev_normalizer=full.game_cls.EV_NORMALIZER)
    for t in range(3):
        a, b, c = s_full.exploitability_current(), s_iso.exploitability_current(), orc.exploitability_current()
        _expl_close("expl full-enum it%d" % t, a, c, tol=1e-6)
        _expl_close("expl iso it%d" % t, b, c, tol=1e-6)
        # trunk (pre-deal) regrets agree between the two GPU trees and with the oracle
        ra = s_full.bufs.regret[:4, :full.R].cpu().numpy()
        rb = s_iso.bufs.regret[:4, :iso.R].cpu().numpy()
        _close("trunk regret", rb, ra.astype(np.float64), tol=5e-6) if t else None
        s_full.iteration(1)
        s_iso.iteration(1)
        orc.iteration()
    a, b, c = s_full.exploitability_average(), s_iso.exploitability_average(), orc.exploitability_average()
    _expl_close("expl avg full-enum", a, c, tol=1e-6)
    _expl_close("expl avg iso", b, c, tol=1e-6)


def test_sharded_schedule_single_rank_equals_plain_solver():
    """The level-split sweep used for multi-GPU runs (world = 1: no communication) reproduces the plain solver."""
    from pokerrl_b200.distributed import ShardedCFRSolver
    from pokerrl_b200.game import games
    from pokerrl_b200.solver import CFRSolver
    spec = random_board_spec(20, 5)
    ft = fhp_tree(spec)
    g = games.Flop5Holdem
    args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[20000, 20000], bet_sizes_list_as_frac_of_pot=[1.0])
    a, b = CFRSolver(ft, "CFRPlus"), ShardedCFRSolver(g, args, spec, "CFRPlus")
    for _ in range(3):
        a.iteration(1)
        b.iteration(1)
        assert a.exploitability_current() == b.exploitability_current()
        assert a.exploitability_average() == b.exploitability_average()
    assert torch_equal(a.bufs.regret, b.bufs.regret)
    assert b.n_allreduce > 0


def torch_equal(x, y):
    import torch
    return bool(torch.equal(x, y))


def test_multi_street_subgame_matches_oracle():
    """Limit Hold'em sub-game rooted at a flop (two chance layers: turn and river, cards restricted to keep the oracle
    fast): values under the uniform profile and three Linear CFR iterations (BASELINE.json configs[3] structure)."""
    from pokerrl_b200.solver import CFRSolver
    from twocard_common import hulh_flop_subgame
    ft = hulh_flop_subgame([[20, 21, 22], [30, 31]])
    orc = oracle_tree(ft)
    orc.fill_uniform()
    expl = orc.compute_ev()
    s = CFRSolver(ft, "LinearCFR")
    m = s.exploitability_current()
    _close("reach", _node_vec(s.bufs.reach, ft), orc.reach)
    _close("ev", _node_vec(s.bufs.ev, ft), orc.ev)
    _close("ev_br", _node_vec(s.bufs.ev_br, ft), orc.ev_br)
    ref_m = float(sum(expl) / 2 * ft.game_cls.EV_NORMALIZER)
    _expl_close("expl uniform (multi-street)", m, ref_m, tol=1e-6)
    c = o2.Oracle2CFR(orc, "LinearCFR", ev_normalizer=ft.game_cls.EV_NORMALIZER)
    for t in range(3):
        s.iteration(1)
        c.iteration()
        a, b = s.exploitability_current(), c.exploitability_current()
        _expl_close("expl multi-street it%d" % t, a, b, tol=1e-6)
        a, b = s.exploitability_average(), c.exploitability_average()
        _expl_close("expl multi-street it%d" % t, a, b, tol=1e-6)


@pytest.mark.parametrize("algo", ["CFRPlus", "LinearCFR"])
def test_kernel_variants_agree(algo, monkeypatch):
    """The record-free fallbacks of the C ABI (NULL node_rec2 / work_rec2 / board_hand_rec: tiled row kernels with
    pointer chains, table-reading terminal kernel) follow the same trajectory as the default kernels."""
    from pokerrl_b200.solver import CFRSolver
    ft = fhp_tree(random_board_spec(6, 11))
    ref = None
    for env in ({}, {"PRL_NO_HAND_REC": "1"}, {"PRL_NO_NODE_REC": "1", "PRL_NO_HAND_REC": "1"}):
        for k in ("PRL_NO_NODE_REC", "PRL_NO_HAND_REC"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        s = CFRSolver(ft, algo)
        assert (s.dtree.desc.node_rec2 is None) == ("PRL_NO_NODE_REC" in env)
        s.iteration(3)
        got = (s.bufs.regret.cpu().numpy().astype(np.float64), s.exploitability_current(), s.exploitability_average())
        if ref is None:
            ref = got
        else:
            _close("regret %s" % env, got[0], ref[0], tol=2e-6)
            _expl_close("expl cur %s" % env, got[1], ref[1], tol=1e-6)
            _expl_close("expl avg %s" % env, got[2], ref[2], tol=1e-6)
