"""GPU parity of the two-card (Hold'em family) LEVEL-engine sweeps against the float64 oracle (oracle/cfr2_numpy.py, whose
terminal rows are pinned on the reference's hand strengths, tests/test_oracle_twocard_rows.py).

Tolerances (achieved errors are printed with -s): BASELINE.json's bar, 1e-6 of the largest
magnitude of the compared array / relative for exploitability; regrets of free-running iterations 2 and 3 and the trunk
regrets of the isomorphism test get 2e-6 / 5e-6 (float32 round-off decides ties in regret matching, SURVEY headline 5)."""
import numpy as np
import pytest

import cfr2_c
import cfr2_numpy as o2
from pokerrl_b200.game.holdem_boards import BoardSpec
from pokerrl_b200.game.games import FlopHoldemRules
from twocard_common import fhp_tree, oracle_tree, random_board_spec

pytestmark = pytest.mark.gpu


ACHIEVED = {}
# Flop5Holdem trees whose chance node has more than 128 children: the level engine reduces it in chunks of 128
# (csrc/cfr_twocard.cu, chance_partial_kernel / chance_sum_kernel) - 128 + 128 + 44 boards, and 128 + 128 + 16 suit classes
# of a 16-card deck (ranks 2 .. 5) followed by the symmetrisation over the 24 suit permutations
BIG_CHANCE = {
    "300boards": lambda: random_board_spec(300, 3),
    "iso272": lambda: BoardSpec.full_game(FlopHoldemRules, isomorphic=True, deck_subset=list(range(16))),
}


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


def test_cfr_plus_delay_matches_oracle():
    """CFR+ with delay 2 (CFRPlus.py:68-84): no averaging step at iterations 0 and 1, the copy of the strategy at iteration 2,
    mixed steps after it - free-running against the float64 C oracle with the same delay"""
    from pokerrl_b200.solver import CFRSolver
    ft = fhp_tree(random_board_spec(16, 2))
    s = CFRSolver(ft, "CFRPlus", delay=2)
    c = cfr2_c.Oracle2CSolver(ft, oracle_tree(ft).board_ranks, "CFRPlus", delay=2)
    for t in range(4):
        s.iteration(1)
        c.iteration(1)
        reg = s.bufs.regret.cpu().numpy()[:, :ft.R].astype(np.float64)
        _close("delay regret it%d" % t, reg, c.regret, tol=1e-6 if t < 2 else 2e-6)
        _expl_close("delay cur it%d" % t, s.exploitability_current(), c.exploitability_current(), tol=1e-6)
        if s.iter_counter > 2:  # iteration 3: the average is the copy of the current strategy
            _expl_close("delay avg it%d" % t, s.exploitability_average(), c.exploitability_average(), tol=1e-6)


def _chance_error_bound(ft, rows):
    """[N, 2, R] bound on the float32 rounding of the chance-node sums in `rows` (ev or ev_br), from the kernels' order:
    sequential sums of <= 128 products mult_b * v_b[h] per chunk, a sequential sum of the chunks, then (suit classes) a
    sequential sum over the n_sym permutations.  With u = 2^-24 each term of a sum of k terms carries at most k u of
    relative error, so a chance node's error is at most (128 + n_chunks + n_sym) u sum_s sum_b |mult_b v_b[perm_s(h)]|, plus
    the bounds of its children.  A decision node sums (or maximises over) its children with weights <= 1: its bound is the
    sum of theirs.  Zero below the chance layer."""
    from pokerrl_b200 import _native as nat
    sp = ft.board_spec.sym_perm
    perms = np.arange(ft.R)[None] if sp is None else np.asarray(sp, np.int64)
    bound = np.zeros_like(rows)
    for n in range(ft.n_nodes - 1, -1, -1):  # level order: children after parents
        fc, A = int(ft.first_child[n]), int(ft.n_children[n])
        if fc < 0 or A <= 0:
            continue
        kids = np.arange(fc, fc + A)
        if ft.kind[n] == nat.KIND_CHANCE:
            k = 128 + -(-A // 128) + perms.shape[0]
            mult = np.asarray(ft.board_mult, np.float64)[ft.board[kids]][:, None, None]
            terms = (mult * (np.abs(rows[kids]) * k * 2.0 ** -24 + bound[kids])).sum(axis=0)
            bound[n] = terms[:, perms].sum(axis=1)
        else:
            bound[n] = bound[kids].sum(axis=0)
    return bound


def _close_with_bound(name, mine, ref, bound, tol=1e-6):
    """|mine - ref| <= tol * max|ref| + bound, per entry; prints the relative error and the share of the allowance used"""
    scale = np.abs(ref).max()
    err = np.abs(mine - ref)
    used = float((err / (tol * scale + bound)).max())
    ACHIEVED[name] = max(ACHIEVED.get(name, 0.0), float(err.max() / scale))
    print("level engine vs float64 oracle: %-22s relative error %.2e, %.0f%% of the allowance (%.0e + chance-sum bound, "
          "largest %.1e relative)" % (name, err.max() / scale, 100 * used, tol, bound.max() / scale))
    assert used <= 1.0, (name, used)


@pytest.mark.parametrize("spec", sorted(BIG_CHANCE))
def test_chance_nodes_over_128_boards_match_oracle(spec):
    """Chance nodes reduced in several chunks: reach, ev and ev_br of the uniform profile at every node, then the four
    half-iterations of two CFR+ and two Linear CFR iterations, each from the oracle's tables, against the float64 C oracle.  Nodes below the chance node at 1e-6; at and above it the float32
    sum depends on its order, so the allowance adds the bound of `_chance_error_bound`."""
    import ctypes as C
    import torch
    from pokerrl_b200 import _native as nat
    from pokerrl_b200.solver import CFRSolver
    ft = fhp_tree(BIG_CHANCE[spec]())
    ch = np.nonzero(ft.kind == nat.KIND_CHANCE)[0]
    assert ch.size > 0 and ft.n_children[ch].min() > 256  # three chunks at every chance node
    ranks = oracle_tree(ft).board_ranks
    orc = cfr2_c.Oracle2CSolver(ft, ranks, "CFRPlus")
    ref_m = orc.exploitability_current()  # uniform profile
    s = CFRSolver(ft, "CFRPlus")
    m = s.exploitability_current()
    _close("reach %s" % spec, _node_vec(s.bufs.reach, ft), orc.reach)
    _close_with_bound("ev %s" % spec, _node_vec(s.bufs.ev, ft), orc.ev, _chance_error_bound(ft, orc.ev))
    _close_with_bound("ev_br %s" % spec, _node_vec(s.bufs.ev_br, ft), orc.ev_br, _chance_error_bound(ft, orc.ev_br))
    _expl_close("expl uniform %s" % spec, m, ref_m, tol=1e-6)
    for algo in ("CFRPlus", "LinearCFR"):
        s = CFRSolver(ft, algo, persistent=False)
        c = cfr2_c.Oracle2CSolver(ft, ranks, algo)
        for t in range(2):
            for p in (0, 1):
                # teacher-forced: the oracle's tables, its strategy included (a hand whose actions tie has float64 regrets of
                # round-off size, and their regret matching decides the other seat's values, SURVEY.md headline 5)
                for dst, src in ((s.bufs.regret, c.regret), (s.bufs.strat, c.strat), (s.bufs.avg, c.avg)):
                    dst[:, :ft.R] = torch.from_numpy(src).to(dst)
                s.iter_counter, s.modes = c.iter_counter, [nat.STRAT_F32, nat.STRAT_F32]
                s.ops.reach_pass(s.modes)
                if p == 0:
                    _expl_close("%s cur it%d" % (algo, t), s.exploitability_current(), c.exploitability_current(), tol=1e-6)
                    if t > 0:
                        _expl_close("%s avg it%d" % (algo, t), s.exploitability_average(), c.exploitability_average(), tol=1e-6)
                nat.call("prl_cfr_half_iteration", C.byref(s.dtree.desc), C.byref(s.bufs.desc), s.algo, p, s.iter_counter, 0, 0,
                         nat.modes(*s.modes), C.c_void_p(torch.cuda.current_stream().cuda_stream))
                c.half_iteration(p)
                # seat p's regret rows take in ev[child] - ev[node] (times the weight iter + 1 of Linear CFR)
                w = c.iter_counter + 1.0 if algo == "LinearCFR" else 1.0
                bound = _chance_error_bound(ft, c.ev)
                allow = np.zeros(c.regret.shape)
                for n in np.nonzero((ft.kind == p) & (ft.first_child >= 0))[0]:
                    fs, fc, A = ft.first_slot[n], ft.first_child[n], ft.n_children[n]
                    allow[fs:fs + A] = w * (bound[fc:fc + A, p] + bound[n, p])
                reg = s.bufs.regret.cpu().numpy()[:, :ft.R].astype(np.float64)
                _close_with_bound("%s regret it%d seat %d" % (algo, t, p), reg, c.regret, allow)
            c.iter_counter += 1


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
    """The level-split sweep used for multi-GPU runs (world = 1: no communication) reproduces the plain solver, also where
    the chance node's sums run over several chunks (chance_phase 1, then 2)."""
    from pokerrl_b200.distributed import ShardedCFRSolver
    from pokerrl_b200.game import games
    from pokerrl_b200.solver import CFRSolver
    spec = random_board_spec(20, 5)
    g = games.Flop5Holdem
    args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[20000, 20000], bet_sizes_list_as_frac_of_pot=[1.0])
    for spec in (spec, ) + tuple(BIG_CHANCE[k]() for k in sorted(BIG_CHANCE)):
        ft = fhp_tree(spec)
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


@pytest.mark.parametrize("algo, spec", [pytest.param(a, None, id=a) for a in ("CFRPlus", "LinearCFR")]
                         + [pytest.param(a, k, id="%s-%s" % (a, k)) for k in sorted(BIG_CHANCE) for a in ("CFRPlus", "LinearCFR")])
def test_kernel_variants_agree(algo, spec, monkeypatch):
    """The record-free fallbacks of the C ABI (NULL node_rec2 / work_rec2 / board_hand_rec: tiled row kernels with
    pointer chains, table-reading terminal kernel) follow the same trajectory as the default kernels - on 6 boards and
    where the chance node has more than 128 children."""
    from pokerrl_b200.solver import CFRSolver
    ft = fhp_tree(random_board_spec(6, 11) if spec is None else BIG_CHANCE[spec]())
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
