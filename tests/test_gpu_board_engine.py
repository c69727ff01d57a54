"""GPU parity of the board-resident CFR+ engine (csrc/cfr_board.cu, pokerrl_b200/board_engine.py), through the C ABI.

Oracles: tests/golden/twocard_rows.npz (brute-force float64 terminal rows on hand strengths from the REFERENCE's
lib_hand_eval.so) and oracle/cfr2_oracle.c (float64; pinned on those rows and on the numpy oracle).
Tolerance (BASELINE.json north_star): 1e-6 relative on counterfactual values and exploitability for every single step from
identical inputs (values under a given profile, one iteration from given tables); free-running trajectories are compared
at the level the reference's own float32/float64 runs agree (SURVEY.md headline 5) and the achieved error is printed."""
import ctypes as C
import os

import numpy as np
import pytest

import cfr2_c
from gen_golden_twocard_common import make_reach
from pokerrl_b200.game.holdem_boards import BoardSpec
from twocard_common import fhp_tree, oracle_ranks, random_board_spec

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "twocard_rows.npz"))
TOL = 1e-6


def _engine(spec, **kw):
    from pokerrl_b200.board_engine import BoardCFRSolver
    from pokerrl_b200.game import games
    g = games.Flop5Holdem
    args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[20000, 20000], bet_sizes_list_as_frac_of_pot=[1.0])
    return BoardCFRSolver(g, args, spec, **kw)


def _rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-300))


def test_board_tables_decode_to_the_strength_order():
    """packed records / hand ids / card rows of prl_board_build_tables against a host computation from the ranks"""
    from pokerrl_b200.board_engine import board_layout
    boards = GOLD["boards"][[0, 5, 121, 150, 199]]
    s = _engine(BoardSpec(boards, np.ones(len(boards)), np.ones(len(boards)), None, "tables"))
    L = board_layout()
    blob = s.t_blob.cpu().numpy()
    ranks = oracle_ranks(boards)
    hc = np.asarray(s.game_cls.RULES.get_lut_holder().LUT_IDX_2_HOLE_CARDS).astype(np.int64)
    for b in range(len(boards)):
        rec = blob[b, :L["sh_off"]].view(np.uint64)
        sh = blob[b, L["sh_off"]:L["rows_off"]].view(np.int16)
        rows = blob[b, L["rows_off"]:].view(np.int16).reshape(L["live_cards"], L["row_pad"])
        rk = ranks[b]
        live = np.nonzero(rk >= 0)[0]
        order = live[np.lexsort((live, rk[live]))]
        assert np.array_equal(sh[:L["n_live"]], order)
        srk = rk[order]
        gs = np.searchsorted(srk, srk, side="left")
        ge = np.searchsorted(srk, srk, side="right")
        assert np.array_equal(rec[:L["n_live"]] & 0x7ff, gs) and np.array_equal((rec[:L["n_live"]] >> 11) & 0x7ff, ge)
        live_cards = [c for c in range(52) if c not in boards[b]]
        lc_of = {c: i for i, c in enumerate(live_cards)}
        pos_of = {int(h): i for i, h in enumerate(order)}
        for c in live_cards:
            in_row = sorted(pos_of[int(h)] for h in order if c in hc[h])
            assert list(rows[lc_of[c], :46]) == in_row and list(rows[lc_of[c], 46:]) == [L["n_live"] + 1] * 2
        for i in (0, 17, 500, 1080):
            h = order[i]
            for k, (sl, st, sd) in enumerate(((22, 34, 40), (28, 46, 52))):
                c = int(hc[h, k])
                assert int((rec[i] >> np.uint64(sl)) & np.uint64(0x3f)) == lc_of[c]
                row_ranks = np.array([rk[x] for x in live if c in hc[x]])
                lt, le = int((row_ranks < rk[h]).sum()), int((row_ranks <= rk[h]).sum())
                assert int((rec[i] >> np.uint64(st)) & np.uint64(0x3f)) == lt
                assert int((rec[i] >> np.uint64(sd)) & np.uint64(0x3f)) == le - lt


def test_root_rows_against_reference_anchored_golden_rows():
    """One evaluation sweep per board with the golden opponent reach row as the trunk's reach and all regrets zero (uniform
    strategies): the board's root value row is a fixed linear combination of the golden showdown and fold rows."""
    import torch
    from pokerrl_b200 import _native as nat
    boards, K = GOLD["boards"], float(GOLD["eq_const"])
    n = len(boards)
    s = _engine(BoardSpec(boards, np.ones(n), np.ones(n), None, "golden rows"))
    hc = np.asarray(s.game_cls.RULES.get_lut_holder().LUT_IDX_2_HOLE_CARDS).astype(np.int64)
    # scaled by 2^-10 (exact): the fixed-point sums are sized for reach rows of total mass <= 1, as in a game
    reach = make_reach(int(GOLD["seed"]), boards, hc) * np.float32(2.0 ** -10)
    st = s.st
    worst = {0: 0.0, 1: 0.0}
    row = torch.zeros(s.ld, dtype=torch.float32, device=s.device)
    for p in (0, 1):
        # coefficients: every action has probability 1/A under zero regrets; own probabilities weight the value, opponent
        # probabilities weight the reach (ValueFiller.py:64-93, StrategyFiller.py:118-146)
        coef_sd, coef_fold = 0.0, 0.0
        for t in range(st["n_local"]):
            if st["kind"][t] < 3:
                continue
            w, i = 1.0, t
            while st["parent"][i] >= 0:
                w /= st["n_children"][st["parent"][i]]
                i = st["parent"][i]
            w *= st["pot"][t] / 2
            if st["kind"][t] == 4:
                coef_sd += w
            else:
                coef_fold += -w if st["acted_last"][t] == p else w
        for b in range(n):
            row[:1326] = torch.from_numpy(reach[b]).to(s.device)
            s.t_mult.zero_()
            s.t_mult[b] = 1.0
            nat.call("prl_board_sweep", C.byref(s.g), p, 1, 0, 0, C.c_void_p(row.data_ptr()), 0, 0, nat.ALGO_CFR_PLUS, 0.0, 0,
                     C.c_void_p(torch.cuda.current_stream().cuda_stream))
            got = s.w_total[2 * p].cpu().numpy().astype(np.float64) / 2.0 ** s.g.frac_bits  # evaluation of seat p: arrays 2p, 2p + 1
            ref = (coef_sd * GOLD["showdown"][b] + coef_fold * GOLD["fold"][b]) * 2.0 ** -10
            err = _rel(got, ref)
            worst[p] = max(worst[p], err)
            assert err <= TOL, (p, b, err)
    print("board sweep root rows vs brute-force golden rows: worst relative error seat0 %.2e seat1 %.2e" % (worst[0], worst[1]))


def _oracle(ft, algo="CFRPlus", **kw):
    from twocard_common import oracle_tree
    return cfr2_c.Oracle2CSolver(ft, oracle_tree(ft).board_ranks, algo, n_threads=8, **kw)


def _natural(s, ft):
    reg, avg = s.natural_tables(ft)
    return reg.cpu().numpy()[:, :ft.R].astype(np.float64), avg.cpu().numpy()[:, :ft.R].astype(np.float64)


def _live_mask(ft, spec_boards):
    """[n_slots, R] True where the row's board does not collide with the hand (trunk rows: all True)"""
    hc = np.asarray(ft.rules.get_lut_holder().LUT_IDX_2_HOLE_CARDS)
    blocked = np.zeros((len(spec_boards) + 1, ft.R), bool)
    for b, bd in enumerate(spec_boards):
        blocked[b + 1] = np.isin(hc, bd).any(axis=1)
    node_of_slot = np.nonzero(ft.slot >= 0)[0]
    return ~blocked[np.maximum(ft.board[node_of_slot], 0)]


def _with_grids(values, grids=(1, 7)):
    """parameter sets (value, grid): the default grid (2 CTAs per SM: one board or none per CTA at these sizes) under the
    value's own id, then one CTA and 7 CTAs, which loop over several boards each (7 divides none of the board counts here)"""
    return ([pytest.param(v, 0, id=str(v)) for v in values]
            + [pytest.param(v, g, id="%s-grid%d" % (v, g)) for g in grids for v in values])


def _skewed(spec, seed=0):
    """the boards of `spec` with unequal deal probabilities and multiplicities (sum of prob * mult = 1), so that a sweep that
    weighted a board with another board's numbers could not pass"""
    rng = np.random.default_rng(seed)
    n = len(spec.boards)
    mult = rng.uniform(0.5, 1.5, n)
    prob = rng.uniform(0.5, 1.5, n)
    prob /= (prob * mult).sum()
    return BoardSpec(spec.boards, prob, mult, None, spec.note + ", skewed weights")


def _teacher_forced(spec, algo="CFRPlus", grid=0, delay=0, warm=0, counters=range(4)):
    """Along an oracle run (`warm` oracle iterations first), every HALF-iteration at the iteration counters `counters` starts
    from the oracle's tables: exploitability of the current / average strategy under given tables, and the regrets / average
    after one seat's update from given tables, at 1e-6.  Returns the errors per half-iteration.
    Why per seat and why masks: where all actions of a hand are worth exactly the same, the float64 oracle's regrets are
    +-1e-15 round-off and regret matching turns them into a pure strategy (SURVEY.md headline 5) - the next seat's values
    then depend on noise.  Regrets are continuous in the inputs; the average strategy is compared with the conditioning of
    regret matching taken out (the engine stores nothing for hands that hold a board card)."""
    from pokerrl_b200 import _native as nat
    ft = fhp_tree(spec)
    orc = _oracle(ft, algo, lean=True, delay=delay)
    s = _engine(spec, algo=algo, grid=grid, delay=delay)
    assert s.g.grid == (grid or nat.lib().prl_board_grid()) and s.delay == orc.delay == delay
    orc.iteration(warm)
    live = _live_mask(ft, spec.boards)
    dec = np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]
    errs = []
    for t in counters:
        orc.iter_counter = t
        for p in (0, 1):
            s.load_natural_tables(ft, orc.regret, orc.avg)
            s.set_trunk_strategy_from_regrets()
            s.iter_counter = t
            e1 = e2 = 0.0
            if p == 0:
                a, b = s.exploitability_current(), orc.exploitability_current()
                e1 = abs(a - b) / abs(b)
                if t > delay:  # t == delay + 1: the average is the copy of the current strategy
                    a, b = s.exploitability_average(), orc.exploitability_average()
                    e2 = abs(a - b) / abs(b)
            s._update_begin(p)
            s._update_end(p)
            orc.half_iteration(p)
            reg, avg = _natural(s, ft)  # flushes seat p's pending average step / contribution
            e3 = _rel(reg * live, orc.regret * live)
            cond = np.zeros(orc.regret.shape)
            if algo == "CFRPlus":
                # average strategy of seat p's rows: sigma = r / sum(r) amplifies a regret error by max|r| / sum(r), so the
                # difference is weighted by that condition number (rows whose regret sum reaches max|r| are held to 1e-6 as is)
                for n in dec[ft.kind[dec] == p]:
                    fs, A = ft.first_slot[n], ft.n_children[n]
                    cond[fs:fs + A] = np.minimum(orc.regret[fs:fs + A].sum(axis=0) / np.abs(orc.regret).max(), 1.0)
                scale = 1.0
            else:
                # the sums take in sigma = r+ / sum(r+) of the UPDATED regrets, which amplifies a regret error by
                # max|r| / sum(r+) (a hand whose actions tie has regrets of round-off size and a strategy decided by it):
                # weighted by that condition number like the CFR+ average; the unweighted difference is returned as well
                # ... and the seat's reach at a node is the product of its strategies above it (trunk included), so a node's
                # weight is the product of the condition numbers along its path
                rp = np.maximum(orc.regret, 0.0)
                node_cond = {}
                for n in dec[ft.kind[dec] == p]:  # ascending ids: ancestors first
                    fs, A = ft.first_slot[n], ft.n_children[n]
                    c = np.minimum(rp[fs:fs + A].sum(axis=0) / np.abs(orc.regret).max(), 1.0)
                    a = ft.parent[n]
                    while a >= 0 and a not in node_cond:
                        a = ft.parent[a]
                    node_cond[n] = c * (node_cond[a] if a >= 0 else 1.0)
                    cond[fs:fs + A] = node_cond[n]
                scale = max(np.abs(orc.avg).max(), 1e-300)
            e4 = float((np.abs(avg - orc.avg) * cond * live).max() / scale)
            e5 = _rel(avg * live, orc.avg * live)
            errs.append((e1, e2, e3, e4, e5))
            assert max(e1, e2, e3, e4) <= TOL, (algo, grid, t, p, e1, e2, e3, e4, e5)
    return errs


def _print_errs(what, errs):
    print(what, "teacher-forced relative errors (expl current, expl average, regrets, average conditioned / raw) per "
          "half-iteration:", ["%.1e %.1e %.1e %.1e %.1e" % e for e in errs])


def _iso_spec():
    from pokerrl_b200.game.games import FlopHoldemRules
    return BoardSpec.full_game(FlopHoldemRules, isomorphic=True, deck_subset=[0, 1, 2, 3, 4, 5, 6, 7, 48, 49, 50, 51])


@pytest.mark.parametrize("iso, grid", _with_grids([False, True]))
def test_teacher_forced_steps_match_float64_oracle(iso, grid):
    """CFR+ along an oracle run from the start (iterations 0 .. 3), 48 random boards or the 57 suit classes of a 12-card deck"""
    spec = _iso_spec() if iso else _skewed(random_board_spec(48, 21))
    _print_errs("CFRPlus grid %d" % grid, _teacher_forced(spec, grid=grid))


@pytest.mark.parametrize("algo, grid", _with_grids(["LinearCFR", "VanillaCFR"]))
def test_linear_and_vanilla_cfr_teacher_forced(algo, grid):
    """Vanilla / Linear CFR on the board engine (unclipped weighted regrets; the reach-weighted average sums of a seat are added
    by the NEXT sweep over its rows or by flush_average): every half-iteration from the oracle's tables, regrets, average sums
    and the exploitability of the current / the normalised average strategy at 1e-6."""
    _print_errs("%s grid %d" % (algo, grid), _teacher_forced(_skewed(random_board_spec(40, 17)), algo, grid=grid))


@pytest.mark.parametrize("grid", [0, 7])
def test_cfr_plus_delay_teacher_forced(grid):
    """CFR+ with delay 2 at iteration counters 1 (no averaging step), 2 (the step copies the strategy), 3 (the first mixed
    step; the average's exploitability is that of the current strategy) and 4: the `iter >= delay` gates and the weights
    m_old / m_new with their delay offset, against the float64 oracle run with the same delay"""
    _print_errs("CFRPlus delay 2 grid %d" % grid, _teacher_forced(_skewed(random_board_spec(37, 5)), grid=grid, delay=2, warm=1,
                                                                  counters=range(1, 5)))


@pytest.mark.parametrize("algo", ["CFRPlus", "LinearCFR", "VanillaCFR"])
def test_teacher_forced_steps_late_in_a_run(algo):
    """tables of 3 oracle iterations, then half-iterations at iteration counters 997 and 998: CFR+'s m_old / m_new close to 1
    and Linear CFR's weight iter + 1 in the sweep, the trunk and the pending average contribution, far from 0"""
    _print_errs("%s at iteration 997" % algo, _teacher_forced(_skewed(random_board_spec(37, 5)), algo, grid=7, warm=3,
                                                              counters=(997, 998)))


@pytest.mark.parametrize("algo", ["LinearCFR", "VanillaCFR"])
def test_linear_and_vanilla_free_running_against_level_engine(algo):
    """the deferred average of the board engine against the level engine's in-sweep average: 5 free-running iterations"""
    from pokerrl_b200.solver import CFRSolver
    spec = random_board_spec(32, 6)
    ft = fhp_tree(spec)
    s, lv = _engine(spec, algo=algo), CFRSolver(ft, algo)
    out = []
    for t in range(5):
        s.iteration(1)
        lv.iteration(1)
        a, c = s.exploitability_current(), lv.exploitability_current()
        x, z = s.exploitability_average(), lv.exploitability_average()
        out.append((abs(a - c) / abs(c), abs(x - z) / abs(z)))
        assert max(out[-1]) <= 5e-2, (algo, t, out[-1])
    print(algo, "board engine vs level engine (current, average):", ["%.1e %.1e" % e for e in out])
    assert out[0][0] <= 1e-5 and out[0][1] <= 1e-5  # the first iteration has no ties to amplify


def test_free_running_trajectory_and_level_engine():
    """6 free-running iterations: board engine, float64 oracle and level engine (three codes, same game).  Trajectories are
    NOT expected to agree to round-off (regret matching amplifies it, see above): sanity bounds, achieved numbers printed."""
    from pokerrl_b200.solver import CFRSolver
    spec = random_board_spec(40, 5)
    ft = fhp_tree(spec)
    orc = _oracle(ft, lean=True)
    s = _engine(spec)
    lv = CFRSolver(ft, "CFRPlus")
    a0, b0 = s.exploitability_current(), orc.exploitability_current()
    assert abs(a0 - b0) <= TOL * abs(b0), (a0, b0)
    out = []
    for t in range(6):
        s.iteration(1)
        orc.iteration(1)
        lv.iteration(1)
        a, b, c = s.exploitability_current(), orc.exploitability_current(), lv.exploitability_current()
        x, y, z = s.exploitability_average(), orc.exploitability_average(), lv.exploitability_average()
        out.append((abs(a - b) / abs(b), abs(x - y) / abs(y), abs(c - b) / abs(b), abs(z - y) / abs(y)))
        assert max(out[-1]) <= 5e-2, (t, out[-1])
    print("free-running relative differences to the float64 oracle (board engine current / average, level engine current / "
          "average) per iteration:", ["%.1e %.1e %.1e %.1e" % e for e in out])


def test_fixed_point_sums_do_not_depend_on_the_grid():
    """the chance-node sums are integers: any number of CTAs (and, by the same argument, of GPUs) gives the same bits - for
    every algorithm, and for the average after a flush (Vanilla / Linear CFR: the P1-only flush sweep, then the evaluation
    of the normalised sums)"""
    import torch
    spec = _skewed(random_board_spec(64, 33))
    for algo in ("CFRPlus", "LinearCFR", "VanillaCFR"):
        runs = []
        for grid in (0, 1, 7, 64):
            s = _engine(spec, algo=algo, grid=grid)
            s.iteration(3)
            cur = s.exploitability_current()
            s.flush_average()
            runs.append((s.regret.clone(), s.bufs.regret.clone(), s.avg.clone(), s.bufs.avg.clone(), cur,
                         s.exploitability_average()))
        assert np.count_nonzero(runs[0][2].cpu().numpy()) > 0
        for grid, r in zip((1, 7, 64), runs[1:]):
            assert all(torch.equal(x, y) for x, y in zip(r[:4], runs[0][:4])) and r[4:] == runs[0][4:], (algo, grid)


def _per_board(e, tab):
    """[n_boards, rows_per_board, ldb] view of a post-deal table (a rank without boards keeps one placeholder row)"""
    return tab[:e.n_rows].view(e.n_boards, e.rows_per_board, tab.shape[1])


def test_shards_reproduce_the_single_device_run_bit_for_bit():
    """two 'ranks' on one device (boards round-robin), driven in lockstep with their integer sums added by hand in place of
    the all-reduce, against one rank holding every board: identical tables, identical exploitability.  3 boards give one
    rank a single board, 1 board leaves one rank without any."""
    import torch
    for n_boards in (30, 3, 1):
        spec = random_board_spec(n_boards, 8)
        one = _engine(spec)
        parts = [_engine(spec, rank=r, world=2, reduce_fn=lambda t: None) for r in range(2)]
        assert [e.n_boards for e in parts] == [(n_boards + 1) // 2, n_boards // 2]
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
        for r, e in enumerate(parts):  # rank r holds boards r, r + 2, ...
            e.flush_average()
            assert torch.equal(_per_board(e, e.regret), _per_board(one, one.regret)[r::2])
            assert torch.equal(_per_board(e, e.avg), _per_board(one, one.avg)[r::2])
        for e in parts:
            assert torch.equal(e.bufs.regret, one.bufs.regret) and torch.equal(e.bufs.avg, one.bufs.avg)


def test_single_launch_trunk_equals_the_level_kernel_trunk(monkeypatch):
    """prl_board_trunk (one launch for the pre-deal trunk) against the level kernels driving the same trunk: same regrets
    and exploitability up to the summation order of the fold terminals' card sums"""
    spec = random_board_spec(24, 12)
    a = _engine(spec)
    monkeypatch.setenv("PRL_TRUNK", "levels")
    b = _engine(spec)
    monkeypatch.delenv("PRL_TRUNK")
    assert a.fused_trunk and not b.fused_trunk
    for t in range(3):
        x, y = a.exploitability_current(), b.exploitability_current()
        assert abs(x - y) <= 2e-6 * abs(y), (t, x, y)
        a.iteration(1)
        b.iteration(1)
        ra, rb = a.bufs.regret.cpu().numpy().astype(np.float64), b.bufs.regret.cpu().numpy().astype(np.float64)
        assert _rel(ra[:4], rb[:4]) <= 2e-6, t
        x, y = a.exploitability_average(), b.exploitability_average()
        assert abs(x - y) <= 1e-4 * abs(y), (t, x, y)
