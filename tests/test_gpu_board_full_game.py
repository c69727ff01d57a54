"""The board engine (csrc/cfr_board.cu, pokerrl_b200/board_engine.py) on the full Flop5Holdem game - all 134 459 suit classes
with the 24 suit permutations, at the default grid - against the chunked float64 oracle (oracle/cfr2_chunked.py).

This is the instance bench.py times, and the only one where the engine builds its tables in more than one chunk, addresses
rows and blobs past 2^31 bytes, walks ~500 boards per CTA and sums the chance node over the game's full dynamic range.  Its
inputs are the synthetic profile of oracle/cfr2_chunked.py (mixed, pure, uniform-fallback and zero entries; regrets of the
size of one iteration's increment), loaded into both sides.  Checked, per board where rows are per board:
  - evaluation: the chance node's ev / ev_br rows of both seats and the exploitability, of the current and the average
    strategy, and the uniform profile's exploitability (the first value bench.py logs);
  - one half-iteration of each seat from the synthetic tables at iteration 5 (delay 0), CFR+ and Linear CFR: every board's
    regrets on live hands and its average after the flush (the conditioned comparison of test_gpu_board_engine
    ._teacher_forced), and the trunk's regrets, average and reach.  CFR+ seat 0 runs the deferred averaging form (its step
    is applied by prl_board_avg_flush), seat 1 the paired form (a pending step of iteration 4 is applied with its own).
Tolerance: 1e-6 of the board's own max |ref|.  At and above the chance node: 1e-6 of max |ref| plus the error that the
fixed-point sum inherits from its terms (each held to 1e-6 of itself, like each board) and its quantisation; the share of
that allowance used is printed."""
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from cfr2_chunked import ChunkedOracle, SyntheticProfile
from pokerrl_b200.game.games import FlopHoldemRules
from pokerrl_b200.game.holdem_boards import BoardSpec
from twocard_common import fhp_tree, oracle_ranks

pytestmark = pytest.mark.gpu
TOL = 1e-6
CHUNK = 2048
ITER = 5
# regret units: one iteration's increment is ~2^-12 on a board and ~2^6 in the trunk (printed below); Linear CFR's sums:
# one contribution is ~2^-29 on a board (reach ~2^-31 times weight 6) and ~2^-8 in the trunk
REGRET_EXP = (6, -12)
LINEAR_AVG_EXP = (-8, -30)


def _engine(spec, algo):
    from pokerrl_b200.board_engine import BoardCFRSolver
    from pokerrl_b200.game import games
    g = games.Flop5Holdem
    args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[20000, 20000], bet_sizes_list_as_frac_of_pot=[1.0])
    return BoardCFRSolver(g, args, spec, algo=algo)


class _Moves:
    """chunk-wise moves of post-deal rows between the engine's strength-ordered tables and [n, rows, R] natural tensors"""

    def __init__(self, e, rows):
        assert [c for c, _ in sorted(e.local_rows.items())] == rows  # the row order of board_engine.row_map without a tree
        self.e, self.n_rows = e, len(rows)

    def load(self, tab, lo, rows):
        import torch
        n = rows.shape[0]
        t = torch.zeros((n * self.n_rows, self.e.ld), dtype=torch.float32, device=self.e.device)
        t[:, :rows.shape[2]] = rows.reshape(n * self.n_rows, -1)
        self.e._board_permute(tab, t, 0, lo=lo, hi=lo + n)

    def fetch(self, tab, lo, hi):
        import torch
        t = torch.empty(((hi - lo) * self.n_rows, self.e.ld), dtype=torch.float32, device=self.e.device)
        self.e._board_permute(tab, t, 1, lo=lo, hi=hi)
        return t.view(hi - lo, self.n_rows, self.e.ld)[..., :self.e.R]


def _load(e, moves, prof, seat=0, due=-1):
    """the synthetic profile into the engine at iteration ITER; due >= 0: a CFR+ averaging step of that iteration pending for
    the post-deal rows of `seat`"""
    import torch
    from pokerrl_b200 import _native as nat
    e.reset()
    nb = e.n_boards
    for lo in range(0, nb, CHUNK):
        hi = min(lo + CHUNK, nb)
        reg, avg = prof.board_rows(np.arange(lo, hi), e.device)
        moves.load(e.regret, lo, reg)
        moves.load(e.avg, lo, avg)
    tr, ta = prof.trunk_rows(e.device)
    nts = prof.n_trunk_slots
    e.bufs.regret[:nts].zero_()
    e.bufs.avg[:nts].zero_()
    e.bufs.regret[:nts, :e.R], e.bufs.avg[:nts, :e.R] = tr, ta
    e.set_trunk_strategy_from_regrets()
    e.iter_counter = ITER
    e._clear_pending()
    if due >= 0:
        e._avg_due[seat] = due
    assert e.modes == [nat.STRAT_F32, nat.STRAT_F32]
    torch.cuda.synchronize()


def _full_ranks(boards):
    n = boards.shape[0]
    with ThreadPoolExecutor(max_workers=os.cpu_count()) as ex:
        parts = list(ex.map(lambda lo: oracle_ranks(boards[lo:lo + CHUNK]), range(0, n, CHUNK)))
    return np.concatenate(parts)


def _trunk_bound(ft, chance_node, rows):
    """[nt, 2, R]: the chance node's bound rows carried up the trunk (a decision node weights its children by <= 1 or takes
    their max: its bound is the sum of theirs; fold terminals are computed from the reach alone)"""
    b = np.zeros((chance_node + 1,) + rows.shape)
    b[chance_node] = rows
    for n in range(chance_node, -1, -1):
        if n != chance_node and ft.kind[n] <= 1 and ft.n_children[n] > 0:
            b[n] = b[ft.first_child[n]:ft.first_child[n] + ft.n_children[n]].sum(axis=0)
    return b


@pytest.fixture(scope="module")
def game():
    import torch
    t0 = time.time()
    spec = BoardSpec.full_game(FlopHoldemRules)
    assert spec.boards.shape[0] == 134459 and spec.sym_perm.shape[0] == 24
    ranks = _full_ranks(spec.boards)
    t_ranks = time.time() - t0
    eng = {"CFRPlus": _engine(spec, "CFRPlus"), "LinearCFR": _engine(spec, "LinearCFR")}
    e = eng["CFRPlus"]
    assert e.n_boards == 134459 and e.g.grid == 2 * torch.cuda.get_device_properties(0).multi_processor_count
    ft1 = e.ft1
    prof = {"CFRPlus": SyntheticProfile(ft1, seed=11, regret_exp=REGRET_EXP),
            "LinearCFR": SyntheticProfile(ft1, seed=11, regret_exp=REGRET_EXP, avg_exp=LINEAR_AVG_EXP)}
    rows = prof["CFRPlus"].rows
    dev = e.device

    def tables(f, lo, key):
        if key == "uniform":
            return np.zeros((f.n_slots, f.R)), np.zeros((f.n_slots, f.R))
        return prof[key].tables(f, lo, dev)

    co = ChunkedOracle(fhp_tree, spec, ranks, tables, chunk=CHUNK)
    moves = {k: _Moves(v, rows) for k, v in eng.items()}
    t1 = time.time()
    ref = co.evaluate("CFRPlus")
    ref_uniform = co.evaluate("uniform", forms=("current",))["current"]
    print("full game: %d boards, grid %d, %d oracle threads; ranks %.0f s, engines %.0f s, oracle evaluations %.0f s"
          % (e.n_boards, e.g.grid, co.L.orc2_set_threads(0), t_ranks, t1 - t0 - t_ranks, time.time() - t1))
    return dict(spec=spec, ranks=ranks, eng=eng, prof=prof, rows=rows, co=co, moves=moves, ref=ref, ref_uniform=ref_uniform,
                t0=t0)


def _close(name, got, ref, bound=None):
    """|got - ref| <= TOL max|ref| (+ bound, per entry); prints the error and the share of the allowance used"""
    scale = float(np.abs(ref).max())
    err = np.abs(np.asarray(got, np.float64) - ref)
    allow = TOL * scale + (0.0 if bound is None else bound)
    used = float((err / allow).max())
    print("full game %-34s relative error %.2e, %3.0f%% of the allowance" % (name, err.max() / scale, 100 * used))
    assert used <= 1.0, (name, float(err.max() / scale), used)


def _chance_bound(e, abs_rows):
    """error of the fixed-point chance sum: each term mult_b v_b[perm_s(h)] carries its board's error (held to TOL of itself),
    each of the n_boards * n_sym terms is rounded to 2^-frac_bits, the sum itself is exact"""
    return TOL * abs_rows + e.n_boards_total * max(e.n_sym, 1) * 2.0 ** -e.g.frac_bits


def test_full_game_evaluation(game):
    e, ref, co = game["eng"]["CFRPlus"], game["ref"], game["co"]
    R, ch = e.R, e.chance_node
    # the uniform profile at iteration 0
    e.reset()
    u = e.exploitability_current()
    ru = game["ref_uniform"]
    bu = _expl_bound(e, co, ru)
    _close("uniform exploitability", np.array([u]), np.array([ru["expl"]]), np.array([bu]))
    _load(e, game["moves"]["CFRPlus"], game["prof"]["CFRPlus"])
    for form in ("current", "average"):
        x = e.exploitability_current() if form == "current" else e.exploitability_average()
        r = ref[form]
        for k, a in (("ev", "abs_ev"), ("ev_br", "abs_br")):
            got = (e.bufs.ev if k == "ev" else e.bufs.ev_br)[:, ch, :R].cpu().numpy()
            for p in (0, 1):
                _close("%s chance %s seat %d" % (form, k, p), got[p], r[k][p], _chance_bound(e, r[a][p]))
        _close("%s exploitability" % form, np.array([x]), np.array([r["expl"]]), np.array([_expl_bound(e, co, r)]))


def _expl_bound(e, co, r):
    """the chance rows' bounds carried to the root and weighted by the root reach, in the metric's units"""
    s = 0.0
    for k, a in (("ev", "abs_ev"), ("ev_br", "abs_br")):
        b = _trunk_bound(e.ft1, e.chance_node, _chance_bound(e, r[a]))
        s += float((r["reach"][0] * b[0]).sum())
    return s * e.ev_normalizer / 2


def _trunk_cond(ft, nt, nts, regret, p, algo):
    """condition numbers of seat p's new trunk strategies (see _teacher_forced): min(sum r+ / max|r|, 1) of the node, per
    table slot (Linear CFR: times those of its seat-p ancestors, whose strategies weight its reach), and per node the product
    along its path (its reach)"""
    rmax = np.abs(regret).max()
    cond, node_cond = np.zeros((nts, regret.shape[1])), np.ones((nt, regret.shape[1]))
    for n in range(1, nt):  # parents first
        a = int(ft.parent[n])
        node_cond[n] = node_cond[a]
        if ft.kind[a] == p:
            fs, A = int(ft.first_slot[a]), int(ft.n_children[a])
            c = np.minimum(np.maximum(regret[fs:fs + A], 0).sum(axis=0) / rmax, 1.0)
            node_cond[n] = node_cond[a] * c
            cond[ft.slot[n]] = c if algo == "CFRPlus" else node_cond[n]
    return cond, node_cond


def _paired_pre_step(ft, prof, lo, p, due, regret, avg):
    """the CFR+ averaging step of iteration `due` that the engine holds pending for seat p's post-deal rows, applied to the
    oracle's input: avg = m_old * avg + m_new * (regret matching of the regrets), CFRPlus.py:65-87"""
    cw = 0.5 * due * (due + 1)
    m_old, m_new = cw / (cw + due + 1), (due + 1) / (cw + due + 1)
    st = ft.board_subtree()
    from cfr2_chunked import board_slots
    for d in range(st["n_local"]):
        if st["kind"][d] != p or st["n_children"][d] == 0:
            continue
        kids = list(range(st["first_child"][d], st["first_child"][d] + st["n_children"][d]))
        sl = board_slots(ft, kids)  # [nb, A]
        r = np.maximum(regret[sl], 0.0)  # [nb, A, R]
        s = r.sum(axis=1, keepdims=True)
        strat = np.where(s > 0, r / np.where(s > 0, s, 1.0), 1.0 / len(kids))
        avg[sl] = m_old * avg[sl] + m_new * strat
    return regret, avg


@pytest.mark.parametrize("p", [0, 1])
def test_full_game_half_iteration(game, p):
    """seat p's half-iteration of CFR+ and of Linear CFR from the synthetic tables, every board against the oracle"""
    import torch
    t0 = time.time()
    eng, prof, co, rows, moves = game["eng"], game["prof"], game["co"], game["rows"], game["moves"]
    due = ITER - 1 if p == 1 else -1  # seat 1: the paired CFR+ form
    for algo, e in eng.items():
        _load(e, moves[algo], prof[algo], seat=p, due=due if algo == "CFRPlus" else -1)
        e._update_begin(p)
        e._update_end(p)
        e.flush_average()
    torch.cuda.synchronize()
    base_tables = co.tables
    if due >= 0:
        def tables(f, lo, key):
            reg, avg = base_tables(f, lo, key)
            return _paired_pre_step(f, prof[key], lo, p, due, reg, avg) if key == "CFRPlus" else (reg, avg)
        co.tables = tables
    runs = [("CFRPlus", "CFRPlus", ITER, 0), ("LinearCFR", "LinearCFR", ITER, 0)]
    worst = {(a, w): (0.0, -1) for a, _, _, _ in runs for w in ("regret", "avg", "avg raw")}
    ratio = []
    ranks = game["ranks"]
    from cfr2_chunked import board_slots
    # Linear CFR: a board node's reach carries seat p's trunk strategy, so its weight includes the trunk's condition numbers
    e_lin, ft1 = eng["LinearCFR"], eng["LinearCFR"].ft1
    trunk_cond = torch.ones(e_lin.R, dtype=torch.float64, device=e_lin.device)
    tr = e_lin.bufs.regret[:co.nts, :e_lin.R].double()
    a = int(ft1.parent[e_lin.chance_node])
    while a >= 0:
        if ft1.kind[a] == p:
            fs, A = int(ft1.first_slot[a]), int(ft1.n_children[a])
            trunk_cond *= torch.clamp(tr[fs:fs + A].clamp(min=0).sum(dim=0) / tr.abs().max(), max=1.0)
        a = int(ft1.parent[a])

    def on_chunk(lo, hi, f, k, regret, avg):
        algo = runs[k][1]
        e = eng[algo]
        sl = board_slots(f, rows)
        ref_r = torch.from_numpy(regret[sl]).to(e.device)  # [n, rows, R]
        ref_a = torch.from_numpy(avg[sl]).to(e.device)
        got_r = moves[algo].fetch(e.regret, lo, hi).double()
        got_a = moves[algo].fetch(e.avg, lo, hi).double()
        live = torch.from_numpy(ranks[lo:hi] >= 0).to(e.device)[:, None, :]
        z = torch.zeros((), dtype=torch.float64, device=e.device)
        rmax = torch.where(live, ref_r.abs(), z).amax(dim=(1, 2))  # per board
        er = torch.where(live, (got_r - ref_r).abs(), z).amax(dim=(1, 2)) / rmax
        if k == 0:
            inp = prof["CFRPlus"].board_rows(np.arange(lo, hi), e.device)[0].double()
            ratio.append(((torch.where(live, (ref_r - inp).abs(), z).amax(dim=(1, 2)) /
                           torch.where(live, inp.abs(), z).amax(dim=(1, 2))).cpu().numpy()))
        # average: seat p's rows, weighted by the condition number of regret matching (see _teacher_forced)
        st = f.board_subtree()
        cond = torch.zeros_like(ref_a)
        node_cond = {}
        for d in range(st["n_local"]):  # ascending local ids: ancestors first
            if st["kind"][d] != p or st["n_children"][d] == 0:
                continue
            ks = [rows.index(c) for c in range(st["first_child"][d], st["first_child"][d] + st["n_children"][d])]
            rr = ref_r[:, ks] if algo == "CFRPlus" else ref_r[:, ks].clamp(min=0)
            c = torch.clamp(rr.sum(dim=1) / rmax[:, None], max=1.0)
            a = st["parent"][d]
            while a >= 0 and a not in node_cond:
                a = st["parent"][a]
            if algo != "CFRPlus":
                c = c * (node_cond[a] if a >= 0 else trunk_cond)
                node_cond[d] = c
            cond[:, ks] = c[:, None, :]
        scale = 1.0 if algo == "CFRPlus" else torch.where(live, ref_a.abs(), z).amax(dim=(1, 2))[:, None, None]
        ea = (torch.where(live, (got_a - ref_a).abs(), z) * cond / scale).amax(dim=(1, 2))
        amax = torch.where(live, ref_a.abs(), z).amax(dim=(1, 2))
        ea_raw = torch.where(live, (got_a - ref_a).abs(), z).amax(dim=(1, 2)) / amax
        for w, v in (("regret", er), ("avg", ea), ("avg raw", ea_raw)):
            i = int(torch.argmax(v))
            if float(v[i]) > worst[(algo, w)][0]:
                worst[(algo, w)] = (float(v[i]), lo + i)
        assert float(er.max()) <= TOL and float(ea.max()) <= TOL, (algo, p, lo, float(er.max()), float(ea.max()))

    try:
        trunk = co.half_iterations(p, runs, on_chunk, chance_ev=game["ref"]["current"]["ev"][p])
    finally:
        co.tables = base_tables
    r = np.concatenate(ratio)
    print("full game seat %d: max |update| / max |input regret| per board: median %.2f, min %.2f, max %.2f"
          % (p, np.median(r), r.min(), r.max()))
    for (algo, w), (v, b) in sorted(worst.items()):
        print("full game seat %d %-9s %-7s worst board %6d: relative error %.2e" % (p, algo, w, b, v))
    nts, nt = co.nts, co.n_trunk_nodes
    for k, (key, algo, it, delay) in enumerate(runs):
        e = eng[algo]
        R = e.R
        _close("seat %d %s trunk regrets" % (p, algo), e.bufs.regret[:nts, :R].cpu().numpy(), trunk[k]["regret"])
        # the trunk's average and reach carry seat p's new strategy: weighted by the condition numbers of its matching
        cond, reach_cond = _trunk_cond(e.ft1, nt, nts, trunk[k]["regret"], p, algo)
        scale = 1.0 if algo == "CFRPlus" else float(np.abs(trunk[k]["avg"]).max())
        for w, got, ref, c in (("average", e.bufs.avg[:nts, :R], trunk[k]["avg"], cond / scale),
                               ("reach", e.bufs.reach[p, :nt, :R], trunk[k]["reach"][:, p], reach_cond / np.abs(trunk[k]["reach"][:, p]).max())):
            d = np.abs(got.cpu().numpy().astype(np.float64) - ref)
            err = float((d * c).max())
            print("full game seat %d %-9s trunk %-7s conditioned relative error %.2e (raw %.2e)"
                  % (p, algo, w, err, d.max() / np.abs(ref).max()))
            assert err <= TOL, (p, algo, w, err)
    print("full game seat %d half-iterations: %.0f s (module so far %.0f s)" % (p, time.time() - t0, time.time() - game["t0"]))
