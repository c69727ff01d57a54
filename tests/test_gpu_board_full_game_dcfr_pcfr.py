"""Discounted CFR and Predictive CFR+ on the board engine over the full Flop5Holdem game - all 134 459 suit classes with the
24 suit permutations, at the default grid, at stack 20 000 (the 15-node post-deal shape) and 600 (the 9-node shape) -
against the chunked float64 oracle (oracle/cfr2_chunked.py), as test_gpu_board_full_game.py checks CFR+ and Linear CFR.

Only the full game builds the tables in more than one chunk, addresses rows past 2^31 bytes, walks ~500 boards per CTA and
sums the chance node over the game's whole dynamic range; here that covers DCFR's discount in the deferred update form,
PCFR+'s own sweep instantiation (PRED) with its third board table `pred`, the prediction-swapped evaluation and average
flush of PCFR+, and both algorithms' trunk branches.  Inputs: the synthetic profile (PCFR+: clipped regrets and prediction
rows), loaded into both sides at iteration counter t.  Checked:
  - PCFR+ evaluation at t = 5: the chance node's ev / ev_br rows of both seats and the exploitability, of the current
    strategy (matching of the predictions) and of the average (the normalised sums);
  - one half-iteration of each seat, DCFR (1.5, 0, 2) and PCFR+ (gamma 2) at t = 5 (a_t 0.92, b_t 0.5, w_t 36) and 997
    (a_t near 1, w_t about 1e6; stack 20 000 only): every board's regrets (PCFR+: and predictions) on live hands, its
    average sums after the flush conditioned by the strategies that weigh them (test_gpu_board_full_game), and the
    trunk's regrets, conditioned average and reach (PCFR+: its stored strategy weighted by the prediction mass).  Seat 0's
    own contribution is applied by the flush (the P1-only sweep); seat 1's update sweep first adds seat 0's contribution
    of the same iteration (the deferred form), which the oracle adds under the loaded profile.
Tolerances and allowances are test_gpu_board_full_game's; the share of the allowance used is printed."""
import functools
import time

import numpy as np
import pytest

from cfr2_chunked import ChunkedOracle, SyntheticProfile, board_slots
from pokerrl_b200.game.games import FlopHoldemRules
from pokerrl_b200.game.holdem_boards import BoardSpec
from test_gpu_board_full_game import (CHUNK, TOL, _chance_bound, _close, _expl_bound, _full_ranks, _Moves, _trunk_cond)
from twocard_common import fhp_tree

pytestmark = pytest.mark.gpu
GAMMA = 2.0
STACKS = (20000, 600)
COUNTERS = {20000: (5, 997), 600: (5,)}
REGRET_EXP = (6, -12)  # as test_gpu_board_full_game: one iteration's increment ~2^-12 on a board, ~2^6 in the trunk
# sums: one contribution is ~2^-31 times w_t on a board and ~2^-11 times w_t in the trunk (w_5 = 36 ~ 2^5.2, w_997 ~ 2^19.9)
AVG_EXP = {5: (-5, -27), 997: (9, -13)}
ALGOS = ("DCFR", "PCFRPlus")


def _engine(spec, stack, algo):
    from pokerrl_b200.board_engine import BoardCFRSolver
    from pokerrl_b200.game import games
    g = games.Flop5Holdem
    args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[stack, stack], bet_sizes_list_as_frac_of_pot=[1.0])
    return BoardCFRSolver(g, args, spec, algo=algo, pcfr_gamma=GAMMA)


def _key(algo, t):
    return "%s@%d" % (algo, t)


def _load(e, moves, prof, t, pending=False):
    """the synthetic profile into the engine at iteration counter t; the trunk's strategy from its regrets (PCFR+: its
    predictions); pending: seat 0's average contribution of iteration t is still to be added to the post-deal rows"""
    import torch
    from pokerrl_b200 import _native as nat
    e.reset()
    nb = e.n_boards
    for lo in range(0, nb, CHUNK):
        hi = min(lo + CHUNK, nb)
        rows = prof.board_rows(np.arange(lo, hi), e.device)
        for tab, r in zip((e.regret, e.avg, e.pred), rows):
            moves.load(tab, lo, r)
    tr = prof.trunk_rows(e.device)
    nts = prof.n_trunk_slots
    e.bufs.regret[:nts].zero_()
    e.bufs.avg[:nts].zero_()
    e.bufs.regret[:nts, :e.R], e.bufs.avg[:nts, :e.R] = tr[0], tr[1]
    if e.pred is None:
        e.set_trunk_strategy_from_regrets()
    else:
        q = torch.zeros((nts, e.ld), dtype=torch.float32, device=e.device)
        q[:, :e.R] = tr[2]
        e._set_trunk_strategy(q)
    e.iter_counter = t
    e._clear_pending()
    if pending:
        e._pending[0] = e.alg.sum_weight(t)
    assert e.modes == [nat.STRAT_F32, nat.STRAT_F32]
    torch.cuda.synchronize()


def _free():
    """return the engines' memory (the caller dropped its references) before the next pass allocates"""
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _peak(what):
    import torch
    print("full game %s: peak device memory %.1f GB" % (what, torch.cuda.max_memory_allocated() / 2 ** 30))


@pytest.fixture(scope="module")
def full_ranks():
    """the game's spec and hand ranks (they do not depend on the stack), computed once"""
    t0 = time.time()
    spec = BoardSpec.full_game(FlopHoldemRules)
    assert spec.boards.shape[0] == 134459 and spec.sym_perm.shape[0] == 24
    ranks = _full_ranks(spec.boards)
    return dict(spec=spec, ranks=ranks, t_ranks=time.time() - t0, t0=t0)


@pytest.fixture(scope="module", params=STACKS, ids=["stack%d" % s for s in STACKS])
def game(request, full_ranks):
    """per stack: the synthetic profiles of every (algorithm, counter), the chunked oracle and PCFR+'s evaluation"""
    t0 = time.time()
    stack = request.param
    spec, ranks = full_ranks["spec"], full_ranks["ranks"]
    tree_fn = functools.partial(fhp_tree, stack=stack)
    prof = {}

    def tables(f, lo, key):
        return prof[key].tables(f, lo, "cuda")

    co = ChunkedOracle(tree_fn, spec, ranks, tables, chunk=CHUNK, pcfr_gamma=GAMMA)
    for t in COUNTERS[stack]:
        # the same seed and regret units for every counter: the runs of one algorithm share one value sweep
        prof[_key("DCFR", t)] = SyntheticProfile(co.trunk_ft, seed=11, regret_exp=REGRET_EXP, avg_exp=AVG_EXP[t])
        prof[_key("PCFRPlus", t)] = SyntheticProfile(co.trunk_ft, seed=13, regret_exp=REGRET_EXP, avg_exp=AVG_EXP[t],
                                                     pcfr=True)
    ref = co.evaluate(_key("PCFRPlus", 5), "PCFRPlus")
    print("full game stack %d: %d oracle threads; ranks %.0f s (once per module), PCFR+ oracle evaluation %.0f s"
          % (stack, co.L.orc2_set_threads(0), full_ranks["t_ranks"], time.time() - t0))
    yield dict(stack=stack, spec=spec, ranks=ranks, prof=prof, co=co, ref=ref, rows=prof[_key("DCFR", 5)].rows, t0=t0)
    print("full game stack %d: %.0f s (module so far %.0f s)" % (stack, time.time() - t0, time.time() - full_ranks["t0"]))


def test_full_game_pcfr_evaluation(game):
    """current strategy (matching of the predictions, the prediction-swapped EVAL form) and average (the normalised sums,
    the P1-only flush and STRAT_AVG_SUM): chance-node rows of both seats and the exploitability"""
    import torch
    t0 = time.time()
    stack, ref, co = game["stack"], game["ref"], game["co"]
    e = _engine(game["spec"], stack, "PCFRPlus")
    assert e.n_boards == 134459 and e.g.grid == 2 * torch.cuda.get_device_properties(0).multi_processor_count
    R, ch = e.R, e.chance_node
    _load(e, _Moves(e, game["rows"]), game["prof"][_key("PCFRPlus", 5)], 5)
    for form in ("current", "average"):
        x = e.exploitability_current() if form == "current" else e.exploitability_average()
        r = ref[form]
        for k, a in (("ev", "abs_ev"), ("ev_br", "abs_br")):
            got = (e.bufs.ev if k == "ev" else e.bufs.ev_br)[:, ch, :R].cpu().numpy()
            for p in (0, 1):
                _close("stack %d PCFR+ %s chance %s seat %d" % (stack, form, k, p), got[p], r[k][p],
                       _chance_bound(e, r[a][p]))
        _close("stack %d PCFR+ %s exploitability" % (stack, form), np.array([x]), np.array([r["expl"]]),
               np.array([_expl_bound(e, co, r)]))
    _peak("stack %d PCFR+ evaluation" % stack)
    del e
    _free()
    print("full game stack %d PCFR+ evaluation: %.0f s" % (stack, time.time() - t0))


def _seat_conds(st, rows, x, xmax, q, top):
    """[n, rows, R] condition numbers of seat q's post-deal rows (zero elsewhere): the strategy of a node is matched from
    the rows x (regrets or predictions), min(sum x+ / xmax, 1), times those of its seat-q ancestors on the board and top
    (the trunk's, [R]) above them: the reach that weighs the node's average contribution"""
    import torch
    cond = torch.zeros_like(x)
    node_cond = {}
    for d in range(st["n_local"]):  # ascending local ids: ancestors first
        if st["kind"][d] != q or st["n_children"][d] == 0:
            continue
        ks = [rows.index(c) for c in range(st["first_child"][d], st["first_child"][d] + st["n_children"][d])]
        c = torch.clamp(x[:, ks].clamp(min=0).sum(dim=1) / xmax[:, None], max=1.0)
        a = st["parent"][d]
        while a >= 0 and a not in node_cond:
            a = st["parent"][a]
        node_cond[d] = c * (node_cond[a] if a >= 0 else top)
        cond[:, ks] = node_cond[d][:, None, :]
    return cond


def _top_cond(ft, chance_node, trunk_x, q):
    """[R]: product over seat q's trunk decision nodes above the chance node of min(sum x+ / max |x|, 1)"""
    xmax = np.abs(trunk_x).max()
    c = np.ones(trunk_x.shape[1])
    a = int(ft.parent[chance_node])
    while a >= 0:
        if ft.kind[a] == q:
            fs, A = int(ft.first_slot[a]), int(ft.n_children[a])
            c *= np.minimum(np.maximum(trunk_x[fs:fs + A], 0).sum(axis=0) / xmax, 1.0)
        a = int(ft.parent[a])
    return c


@pytest.mark.parametrize("p", [0, 1])
@pytest.mark.parametrize("algo", ALGOS)
def test_full_game_half_iteration(game, algo, p):
    """seat p's half-iteration at every counter of the stack from the synthetic tables, every board against the oracle;
    seat 0 flushes its own contribution, seat 1's update adds seat 0's pending one first"""
    import torch
    t0 = time.time()
    stack, prof, co, rows, ranks = game["stack"], game["prof"], game["co"], game["rows"], game["ranks"]
    counters = COUNTERS[stack]
    pending = p == 1
    pc = algo == "PCFRPlus"
    eng, moves = {}, {}
    for t in counters:  # only the engines of this oracle pass are resident
        e = eng[t] = _engine(game["spec"], stack, algo)
        moves[t] = _Moves(e, rows)
        _load(e, moves[t], prof[_key(algo, t)], t, pending)
        e._update_begin(p)
        e._update_end(p)
        e.flush_average()
    torch.cuda.synchronize()
    t_gpu = time.time() - t0
    runs = [(_key(algo, t), algo, t, 0) for t in counters]
    whats = ("regret",) + (("pred",) if pc else ()) + ("avg",)  # the average's conditioning reads the regrets / predictions
    worst = {(t, w): (0.0, -1) for t in counters for w in whats}
    ratio = []
    seats = (0, 1) if pending else (p,)
    top = {}

    def on_chunk(lo, hi, f, k, regret, avg, pred=None):
        t = runs[k][2]
        e = eng[t]
        st = f.board_subtree()
        sl = board_slots(f, rows)
        dev = e.device
        live = torch.from_numpy(ranks[lo:hi] >= 0).to(dev)[:, None, :]
        z = torch.zeros((), dtype=torch.float64, device=dev)
        ref = {"regret": regret, "avg": avg, "pred": pred}
        tab = {"regret": e.regret, "avg": e.avg, "pred": e.pred}
        err, refs = {}, {}
        for w in whats:
            r = refs[w] = torch.from_numpy(ref[w][sl]).to(dev)  # [n, rows, R]
            g = moves[t].fetch(tab[w], lo, hi).double()
            d = torch.where(live, (g - r).abs(), z)
            scale = torch.where(live, r.abs(), z).amax(dim=(1, 2))  # per board
            if w == "avg":  # the sums, weighted by the conditioning of the strategies that weigh each contribution
                x = refs["pred" if pc else "regret"]
                xmax = torch.where(live, x.abs(), z).amax(dim=(1, 2))
                if k not in top:  # the game's trunk rows after the update: the strategies above the boards
                    tx = (pred if pc else regret)[:co.nts]
                    top[k] = {q: torch.from_numpy(_top_cond(f, co.chance_node, tx, q)).to(dev) for q in seats}
                cond = sum(_seat_conds(st, rows, x, xmax, q, top[k][q]) for q in seats)
                d = d * cond
            err[w] = d.amax(dim=(1, 2)) / scale
        if k == 0:
            inp = prof[runs[0][0]].board_rows(np.arange(lo, hi), e.device)[0].double()
            ratio.append((torch.where(live, (refs["regret"] - inp).abs(), z).amax(dim=(1, 2)) /
                          torch.where(live, inp.abs(), z).amax(dim=(1, 2))).cpu().numpy())
        for w, v in err.items():
            i = int(torch.argmax(v))
            if float(v[i]) > worst[(t, w)][0]:
                worst[(t, w)] = (float(v[i]), lo + i)
        assert max(float(v.max()) for v in err.values()) <= TOL, (algo, t, p, lo, {w: float(v.max()) for w, v in err.items()})

    chance_ev = game["ref"]["current"]["ev"][p] if pc else None  # DCFR: a pass of its own
    trunk = co.half_iterations(p, runs, on_chunk, chance_ev=chance_ev, pending=pending)
    r = np.concatenate(ratio)
    print("full game stack %d %s seat %d: max |update| / max |input regret| per board: median %.2f, min %.2f, max %.2f"
          % (stack, algo, p, np.median(r), r.min(), r.max()))
    for (t, w), (v, b) in sorted(worst.items()):
        print("full game stack %d %s counter %d seat %d %-6s worst board %6d: relative error %.2e" % (stack, algo, t, p, w, b, v))
    nts, nt = co.nts, co.n_trunk_nodes
    for k, (key, _, t, _) in enumerate(runs):
        e = eng[t]
        R, ft = e.R, e.ft1
        name = "stack %d %s t %d seat %d trunk" % (stack, algo, t, p)
        _close(name + " regrets", e.bufs.regret[:nts, :R].cpu().numpy(), trunk[k]["regret"])
        # the trunk's average and reach carry seat p's new strategy: weighted by the conditioning of its matching
        x = trunk[k]["pred" if pc else "regret"]
        cond, reach_cond = _trunk_cond(ft, nt, nts, x, p, algo)
        for w, got, ref, c in (("average", e.bufs.avg[:nts, :R], trunk[k]["avg"], cond / np.abs(trunk[k]["avg"]).max()),
                               ("reach", e.bufs.reach[p, :nt, :R], trunk[k]["reach"][:, p],
                                reach_cond / np.abs(trunk[k]["reach"][:, p]).max())):
            d = np.abs(got.cpu().numpy().astype(np.float64) - ref)
            err = float((d * c).max())
            print("full game %s %-7s conditioned relative error %.2e (raw %.2e)" % (name, w, err, d.max() / np.abs(ref).max()))
            assert err <= TOL, (name, w, err)
        if pc:  # stored strategy against matching of the oracle's Q, weighted by the prediction mass (test_gpu_pcfr e6)
            want = trunk[k]["strat"]
            wt = np.zeros_like(want)
            for n in range(co.chance_node + 1):
                if ft.kind[n] <= 1 and ft.first_child[n] >= 0:
                    fs, A = int(ft.first_slot[n]), int(ft.n_children[n])
                    wt[fs:fs + A] = np.minimum(x[fs:fs + A].sum(axis=0) / x.max(), 1.0)
            err = float((np.abs(e.bufs.strat[:nts, :R].cpu().numpy() - want) * wt).max())
            print("full game %s strategy weighted error %.2e" % (name, err))
            assert err <= TOL, (name, "strategy", err)
    _peak("stack %d %s seat %d" % (stack, algo, p))
    del e
    eng.clear()
    moves.clear()
    _free()
    print("full game stack %d %s seat %d: %.0f s (engines and updates %.0f s; module so far %.0f s)"
          % (stack, algo, p, time.time() - t0, t_gpu, time.time() - game["t0"]))
