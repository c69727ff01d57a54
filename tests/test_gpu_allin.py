"""GPU parity of the all-in showdown before the deal (csrc/allin_dense.cu: equity matrix, wgmma GEMM) through the C ABI.

Oracle: float64 brute force (oracle/cfr2_numpy.allin_equity_matrix) on hand strengths of the REFERENCE's lib_hand_eval.so
(tests/golden/twocard_rows.npz `ranks`) - the one-card analogue in the reference is ValueFiller.py:160-175.
Tolerance 1e-6 of the row's largest magnitude (BASELINE.json north_star); achieved errors are printed."""
import os

import numpy as np
import pytest

import cfr2_numpy as o2
from gen_golden_twocard_common import make_reach
from pokerrl_b200.game.holdem_boards import BoardSpec
from twocard_common import fhp_tree, nl_flop_subgame, oracle_tree, random_board_spec

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "twocard_rows.npz"))
TOL = 1e-6


def _rules():
    from pokerrl_b200.game import games
    return games.Flop5Holdem.RULES


def _rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-300))


def test_equity_matrix_and_dense_rows_on_reference_ranks():
    """E from the GPU evaluator + accumulate / finish kernels == float64 E from the reference's ranks (exactly, before the
    bf16 split: integer multiples of 1/64), and 20 value rows (two tensor-core launches: 16 + 4 columns) within 1e-6"""
    import torch
    from pokerrl_b200.allin import AllinEquity
    rules = _rules()
    hc = np.asarray(rules.get_lut_holder().LUT_IDX_2_HOLE_CARDS).astype(np.int64)
    boards, ranks = GOLD["boards"], GOLD["ranks"]
    w = (np.arange(len(boards)) % 16 + 8.0) / 64.0
    spec = BoardSpec(boards, w, np.ones(len(boards)), None, "golden boards")
    eq = AllinEquity(rules, spec, chunk=64, keep_ec=True)
    E64 = o2.allin_equity_matrix(ranks, w, hc, 52)
    inc = np.zeros((1326, 52))
    inc[np.arange(1326), hc[:, 0]] = 1
    inc[np.arange(1326), hc[:, 1]] = 1
    compat = (inc @ inc.T) == 0
    assert np.array_equal(eq.ec.cpu().numpy() * compat, E64)
    x = make_reach(11, np.repeat(boards[:1], 20, axis=0), hc).astype(np.float32)  # 20 skewed rows (some sparse, some tiny)
    x[3] *= 1e-4
    x[7] = 0.0
    x[7, 100] = 1.0  # a unit vector reads one column of E
    scale = np.linspace(0.5, 40.0, 20).astype(np.float32)
    xt = torch.zeros(20, 1328, dtype=torch.float32, device="cuda")
    xt[:, :1326] = torch.from_numpy(x).cuda()
    y = eq.values(xt, scale).cpu().numpy()[:, :1326]
    want = (x.astype(np.float64) @ E64.T) * scale[:, None].astype(np.float64)
    errs = [_rel(y[c], want[c]) for c in range(20)]
    print("dense all-in rows: relative errors (max over 20 rows) %.2e, unit-vector row %.2e" % (max(errs), errs[7]))
    assert max(errs) <= TOL, errs
    assert np.all(y[:, np.isin(hc, boards[0]).any(axis=1)] == y[:, np.isin(hc, boards[0]).any(axis=1)])  # finite


@pytest.mark.parametrize("n_cols", [1, 16, 17, 33])
@pytest.mark.parametrize("y2", ["none", "some"])
def test_value_columns_in_chunks_of_16(n_cols, y2):
    """prl_allin_values computes 16 columns per launch, all launches sharing one `partial` buffer: 1, 16, 17 and 33 columns
    (an incomplete launch, one full launch, a last launch of one column, three launches) against float64 x E^T * scale at
    1e-6.  The optional second output of a column (y2_rows, NULL as a whole or for some columns) is bit for bit y."""
    import ctypes as C
    import torch
    from pokerrl_b200 import _native as nat
    eq, E64, boards, hc = _golden_equity()
    rng = np.random.default_rng(n_cols)
    x = make_reach(100 + n_cols, np.repeat(boards[:1], n_cols, axis=0), hc).astype(np.float32)
    x[rng.random(n_cols) < 0.2] *= 1e-4
    scale = rng.uniform(0.5, 40.0, n_cols).astype(np.float32)
    xt = torch.zeros(n_cols, 1328, dtype=torch.float32, device="cuda")
    xt[:, :1326] = torch.from_numpy(x).cuda()
    yt = torch.full((n_cols, 1328), float("nan"), dtype=torch.float32, device="cuda")
    y2t = torch.full((n_cols, 1328), float("nan"), dtype=torch.float32, device="cuda")
    given = [y2 == "some" and c % 3 != 1 for c in range(n_cols)]  # column 0 always has one when any are given
    ptrs = C.c_void_p * n_cols
    y2_rows = ptrs(*[y2t[c].data_ptr() if given[c] else None for c in range(n_cols)]) if y2 == "some" else None
    nat.call("prl_allin_values", C.c_void_p(eq.tiles.data_ptr()), eq.R, ptrs(*[xt[c].data_ptr() for c in range(n_cols)]),
             ptrs(*[yt[c].data_ptr() for c in range(n_cols)]), y2_rows, scale.ctypes.data_as(C.c_void_p), n_cols,
             C.c_void_p(eq.partial.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    y, y2v = yt.cpu().numpy()[:, :1326], y2t.cpu().numpy()[:, :1326]
    want = (x.astype(np.float64) @ E64.T) * scale[:, None].astype(np.float64)
    errs = [_rel(y[c], want[c]) for c in range(n_cols)]
    print("all-in columns %d (y2 %s): worst relative error %.2e" % (n_cols, y2, max(errs)))
    assert max(errs) <= TOL, errs
    for c in range(n_cols):
        if given[c]:
            assert np.array_equal(y2v[c].view(np.int32), y[c].view(np.int32)), c
        else:
            assert np.isnan(y2v[c]).all(), c


_EQ = []


def _golden_equity():
    """(AllinEquity, float64 E, boards, hand cards) of the golden boards with weights (b % 16 + 8) / 64, built once"""
    if not _EQ:
        from pokerrl_b200.allin import AllinEquity
        rules = _rules()
        hc = np.asarray(rules.get_lut_holder().LUT_IDX_2_HOLE_CARDS).astype(np.int64)
        boards, ranks = GOLD["boards"], GOLD["ranks"]
        w = (np.arange(len(boards)) % 16 + 8.0) / 64.0
        eq = AllinEquity(rules, BoardSpec(boards, w, np.ones(len(boards)), None, "golden boards"))
        _EQ.append((eq, o2.allin_equity_matrix(ranks, w, hc, 52), boards, hc))
    return _EQ[0]


def test_suit_symmetrised_matrix_equals_full_enumeration():
    """isomorphism classes + the 24 hand permutations give the matrix of the explicit board set (a deck subset keeps it small)"""
    import torch
    from pokerrl_b200.allin import AllinEquity
    rules = _rules()
    sub = list(range(0, 28))  # 7 ranks x 4 suits: closed under suit permutations
    iso = BoardSpec.full_game(rules, isomorphic=True, deck_subset=sub)
    full = BoardSpec.full_game(rules, isomorphic=False, deck_subset=sub)
    a, b = AllinEquity(rules, iso), AllinEquity(rules, full)
    hc = np.asarray(rules.get_lut_holder().LUT_IDX_2_HOLE_CARDS).astype(np.int64)
    x = torch.zeros(4, 1328, dtype=torch.float32, device="cuda")
    x[:, :1326] = torch.from_numpy(make_reach(5, np.zeros((4, 0), np.int8), hc)).cuda()  # NOT suit-symmetric: E must be the
    ya, yb = a.values(x).cpu().numpy(), b.values(x).cpu().numpy()                        # matrix of all boards of the orbits
    err = _rel(ya, yb.astype(np.float64))
    print("iso (%d classes) vs full (%d boards): %.2e" % (len(iso.boards), len(full.boards), err))
    assert err <= TOL


def test_push_fold_cfr_plus_against_the_oracle():
    """Flop5Holdem with 3 big blinds: raise = all-in, no post-deal play.  Values of the uniform profile, the first regret
    update of each seat from identical tables and the exploitabilities against the float64 oracle."""
    from pokerrl_b200.solver import CFRSolver
    ft = fhp_tree(random_board_spec(48, 9), stack=300)
    assert int((ft.kind == o2.KIND_SHOWDOWN_ALLIN).sum()) == 1
    s = CFRSolver(ft, "CFRPlus")
    orc = oracle_tree(ft)
    c = o2.Oracle2CFR(orc, "CFRPlus", ev_normalizer=ft.game_cls.EV_NORMALIZER)
    a, b = s.exploitability_current(), c.exploitability_current()
    ev = s.bufs.ev.cpu().numpy()[:, :, :ft.R].transpose(1, 0, 2).astype(np.float64)
    errs = [_rel(ev, orc.ev), abs(a - b) / abs(b)]
    for t in range(3):
        s.iteration(1)
        c.iteration()
        reg = s.bufs.regret.cpu().numpy()[:, :ft.R].astype(np.float64)
        ref = np.zeros_like(reg)
        for n in c.t.decision_nodes():
            ref[ft.first_slot[n]:ft.first_slot[n] + ft.n_children[n]] = c.regret[n].T
        a, b = s.exploitability_current(), c.exploitability_current()
        a2, b2 = s.exploitability_average(), c.exploitability_average()
        errs += [_rel(reg, ref), abs(a - b) / abs(b), abs(a2 - b2) / abs(b2)]
    print("push/fold: ev %.2e expl %.2e | per iteration (regret, current, average): %s"
          % (errs[0], errs[1], " ".join("%.1e" % e for e in errs[2:])))
    assert errs[0] <= TOL and errs[1] <= TOL and errs[2] <= TOL  # identical inputs: uniform profile, first update
    assert max(errs) <= 1e-4  # free-running three iterations (SURVEY headline 5: round-off decides ties)


def _brute_force_equity(h1, h2):
    """(wins - losses) / C(48, 5) of hand h1 against h2 over every board, by the C evaluator pinned to lib_hand_eval.so"""
    import ctypes as C
    import itertools
    from twocard_common import ROOT, oracle_ranks
    oracle_ranks(np.zeros((1, 5), np.int8) + np.arange(5, dtype=np.int8))  # builds the oracle library
    orc = C.CDLL(os.path.join(ROOT, "oracle", "_build", "libhand_eval_oracle.so"))
    orc.orc_rank7_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
    rest = [c for c in range(52) if c not in tuple(h1) + tuple(h2)]
    boards = np.array(list(itertools.combinations(rest, 5)), dtype=np.int8)
    n = len(boards)

    def ranks(h):
        cards = np.ascontiguousarray(np.concatenate([np.tile(np.array(h, np.int8), (n, 1)), boards], axis=1))
        out = np.zeros(n, np.int32)
        orc.orc_rank7_batch(out.ctypes.data, cards.ctypes.data, n)
        return out
    a, b = ranks(h1), ranks(h2)
    return (int((a > b).sum()) - int((a < b).sum())) / n


def test_full_game_preflop_equities_against_brute_force():
    """134 459 isomorphism classes x 24 permutations = all 2 598 960 boards: two matrix entries against the enumeration of
    the C(48, 5) = 1 712 304 boards (pocket aces against pocket kings, no shared suit: 0.81052 - 0.18554), antisymmetry, and
    CFR+ on the push / fold game they define converges"""
    import torch
    from pokerrl_b200.allin import AllinEquity
    from pokerrl_b200.solver import CFRSolver
    rules = _rules()
    spec = BoardSpec.full_game(rules)
    eq = AllinEquity(rules, spec)
    lut = rules.get_lut_holder()
    hc = np.asarray(lut.LUT_IDX_2_HOLE_CARDS).astype(np.int64)
    idx = {tuple(c): i for i, c in enumerate(hc.tolist())}

    def card(rank, suit):
        return rank * 4 + suit

    AA, KK = (card(12, 0), card(12, 1)), (card(11, 2), card(11, 3))
    AKs, QQ = (card(11, 0), card(12, 0)), (card(10, 1), card(10, 2))
    x = torch.zeros(3, 1328, dtype=torch.float32, device="cuda")
    x[0, idx[KK]] = 1.0
    x[1, idx[QQ]] = 1.0
    x[2, idx[AA]] = 1.0
    y = eq.values(x).cpu().numpy().astype(np.float64)
    want = [_brute_force_equity(AA, KK), _brute_force_equity(AKs, QQ)]
    print("AA vs KK %.7f (brute force %.7f)  AKs vs QQ %.7f (%.7f)" % (y[0, idx[AA]], want[0], y[1, idx[AKs]], want[1]))
    assert abs(y[0, idx[AA]] - want[0]) < 1e-6 and abs(y[1, idx[AKs]] - want[1]) < 1e-6
    assert abs(y[2, idx[KK]] + y[0, idx[AA]]) < 1e-6
    s = CFRSolver(fhp_tree(spec, stack=300), "CFRPlus")
    e0 = s.exploitability_current()
    s.iteration(200)
    e1 = s.exploitability_average()
    print("push/fold Flop5Holdem, 3 bb: exploitability %.3f -> %.4f mbb/g after 200 CFR+ iterations" % (e0, e1))
    assert 0 <= e1 < 0.02 * e0


def test_push_fold_game_through_the_cfr_facade():
    """CFRPlus(game_cls=Flop5Holdem, starting_stack_sizes=[300]) - the reference's constructor - picks the level engine
    with the dense all-in terminal and logs the reference's experiment names; series against the float64 oracle"""
    from pokerrl_b200.cfr.CFRPlus import CFRPlus
    from pokerrl_b200.game.games import Flop5Holdem
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    spec = random_board_spec(40, 4)
    chief = ChiefBase(t_prof=None)
    cfr = CFRPlus(name="pf", chief_handle=chief, game_cls=Flop5Holdem, agent_bet_set=[1.0], starting_stack_sizes=[300], delay=0,
                  board_spec=spec)
    c = o2.Oracle2CFR(oracle_tree(fhp_tree(spec, stack=300)), "CFRPlus", ev_normalizer=Flop5Holdem.EV_NORMALIZER)
    ref = [c.exploitability_current()]
    for _ in range(2):
        cfr.iteration()
        c.iteration()
        ref.append(c.exploitability_current())
    got = [v for _, v in chief.get_experiments()["pf_Curr_S300_total_CFRp_delay0"]["Evaluation/MBB_per_G"]]
    errs = [abs(a - b) / abs(b) for a, b in zip(got, ref)]
    print("push/fold through the facade: current-strategy exploitability", got, "relative errors", ["%.1e" % e for e in errs])
    assert len(got) == 3 and max(errs[:2]) <= TOL and errs[2] <= 1e-4


def test_nl_subgame_with_all_ins_on_two_streets_against_the_oracle():
    """DiscretizedNLHoldem flop sub-game, 6 big blinds: all-in showdowns on the flop (one matrix over turn x river) and on
    every turn board (one matrix each over the river) - level engine vs float64 oracle: values of the uniform profile and
    two CFR+ iterations"""
    from pokerrl_b200.solver import CFRSolver
    ft = nl_flop_subgame()
    s = CFRSolver(ft, "CFRPlus")
    assert len(s.dtree.allin) == 4
    orc = oracle_tree(ft)
    c = o2.Oracle2CFR(orc, "CFRPlus", ev_normalizer=ft.game_cls.EV_NORMALIZER)
    a, b = s.exploitability_current(), c.exploitability_current()
    ev = s.bufs.ev.cpu().numpy()[:, :, :ft.R].transpose(1, 0, 2).astype(np.float64)
    br = s.bufs.ev_br.cpu().numpy()[:, :, :ft.R].transpose(1, 0, 2).astype(np.float64)
    errs = [_rel(ev, orc.ev), _rel(br, orc.ev_br), abs(a - b) / abs(b)]
    for t in range(2):
        s.iteration(1)
        c.iteration()
        reg = s.bufs.regret.cpu().numpy()[:, :ft.R].astype(np.float64)
        ref = np.zeros_like(reg)
        for n in c.t.decision_nodes():
            ref[ft.first_slot[n]:ft.first_slot[n] + ft.n_children[n]] = c.regret[n].T
        a, b = s.exploitability_current(), c.exploitability_current()
        errs += [_rel(reg, ref), abs(a - b) / abs(b)]
    print("NL flop sub-game with all-ins: ev %.1e ev_br %.1e expl %.1e | per iteration (regret, current): %s"
          % (errs[0], errs[1], errs[2], " ".join("%.1e" % e for e in errs[3:])))
    assert max(errs[:5]) <= 2e-6 and max(errs) <= 1e-4
