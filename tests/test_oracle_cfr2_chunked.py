"""The chunked float64 oracle (oracle/cfr2_chunked.py) against the monolithic C oracle (oracle/cfr2_c.Oracle2CSolver) on
games small enough for both: chance-node rows, exploitability of the current and the average strategy, and every table
slot after each seat's half-iteration (CFR+ and Linear CFR) from the synthetic profile, to 1e-12.  This pins the machinery
behind the full-game GPU test (tests/test_gpu_board_full_game.py) on a CPU."""
import ctypes as C

import numpy as np
import pytest

import cfr2_c
from cfr2_chunked import ChunkedOracle, SyntheticProfile, board_slots, decision_rows
from pokerrl_b200.game.games import FlopHoldemRules
from pokerrl_b200.game.holdem_boards import BoardSpec
from twocard_common import fhp_tree, oracle_ranks, random_board_spec

TOL = 1e-12
# spec, chunk size: neither divides the number of boards (272 = 2 x 100 + 72, 48 = 2 x 17 + 14)
SPECS = {
    "iso272": (lambda: BoardSpec.full_game(FlopHoldemRules, isomorphic=True, deck_subset=list(range(16))), 100),
    "random48": (lambda: random_board_spec(48, 21), 17),
}
ITER = 5


def _profiles(ft):
    return {"CFRPlus": SyntheticProfile(ft, seed=3, regret_exp=(-4, -12)),
            "LinearCFR": SyntheticProfile(ft, seed=3, regret_exp=(-4, -12), avg_exp=(-6, -16))}


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def _mono(ft, ranks, algo, regret, avg):
    rk = np.full((ranks.shape[0] + 1, ft.R), -1, np.int32)
    rk[1:] = ranks
    o = cfr2_c.Oracle2CSolver(ft, rk, algo, lean=True, n_threads=4)
    o.regret[:], o.avg[:] = regret, avg
    o.L.orc2_regret_match(C.byref(o.t))
    o.L.orc2_reach(C.byref(o.t), o.strat.ctypes.data)
    return o


def test_synthetic_profile_has_the_features_of_a_late_run():
    """mixed and pure strategies, uniform fallbacks, exact zeros; the same bits for the same keys, whatever the chunking"""
    spec = random_board_spec(12, 4)
    ft = fhp_tree(spec)
    prof = SyntheticProfile(ft, seed=3, regret_exp=(-4, -12))
    reg, avg = prof.board_rows(np.arange(12))
    r2, a2 = prof.board_rows(np.arange(5, 9))
    assert np.array_equal(reg[5:9].numpy(), r2.numpy()) and np.array_equal(avg[5:9].numpy(), a2.numpy())
    r = reg.numpy().astype(np.float64)
    assert np.all(r * 2.0 ** 32 == np.round(r * 2.0 ** 32))  # multiples of 2^-32: exact in float32 and float64
    st = ft.board_subtree()
    rows = decision_rows(st)
    d = st["parent"][rows[0]]
    grp = [k for k, c in enumerate(rows) if st["parent"][c] == d]
    pos = (r[:, grp] > 0).sum(axis=1)  # [boards, hands]: positive regrets of the hand at node d
    n = pos.size
    for what, share in (("all <= 0", (pos == 0).mean()), ("pure", (pos == 1).mean()), ("mixed", (pos >= 2).mean()),
                        ("zero entries", (r == 0).mean())):
        print("synthetic profile: %-12s %.3f" % (what, share))
        assert 0.05 < share < 0.9, what
    a = avg.numpy().astype(np.float64)[:, grp].sum(axis=1)
    assert np.abs(a - 1).max() < 1e-6 and n > 0


@pytest.mark.parametrize("name", sorted(SPECS))
def test_chunked_oracle_reproduces_the_monolithic_oracle(name):
    spec, chunk = SPECS[name][0](), SPECS[name][1]
    nb = spec.boards.shape[0]
    assert nb % chunk != 0 and nb > 2 * chunk
    ft = fhp_tree(spec)
    ranks = oracle_ranks(spec.boards)
    profs = _profiles(ft)
    co = ChunkedOracle(fhp_tree, spec, ranks, lambda f, lo, key: profs[key].tables(f, lo), chunk=chunk, n_threads=4)
    ch = co.chance_node
    rows = profs["CFRPlus"].rows
    assert co.nts + nb * len(rows) == ft.n_slots
    mono_slots = board_slots(ft, rows)

    # evaluation: chance-node rows and exploitability, current and average strategy
    got = co.evaluate("CFRPlus")
    o = _mono(ft, ranks, "CFRPlus", *profs["CFRPlus"].tables(ft, 0))
    errs = {}
    for form in ("current", "average"):
        expl = o.exploitability_current() if form == "current" else o.exploitability_average()
        errs[form + " expl"] = abs(got[form]["expl"] - expl) / abs(expl)
        for k, ref in (("ev", o.ev[ch]), ("ev_br", o.ev_br[ch])):
            errs["%s %s" % (form, k)] = _rel(got[form][k], ref)
        # the bound rows: sum over permutations and boards of |mult * child|
        kids = np.arange(ft.first_child[ch], ft.first_child[ch] + ft.n_children[ch])
        mult = np.asarray(ft.board_mult, np.float64)[ft.board[kids]][:, None, None]
        ref_abs = (mult * np.abs(o.ev[kids])).sum(axis=0)[:, co.perms].sum(axis=1)
        errs[form + " abs_ev"] = _rel(got[form]["abs_ev"], ref_abs)
    print(name, "chunked vs monolithic oracle, evaluation:", {k: "%.1e" % v for k, v in errs.items()})
    assert max(errs.values()) <= TOL, errs

    # seat p's half-iteration of CFR+ and Linear CFR from the synthetic tables, every slot
    runs = [("CFRPlus", "CFRPlus", ITER, 0), ("LinearCFR", "LinearCFR", ITER, 0)]
    for p in (0, 1):
        out = [[np.full((ft.n_slots, ft.R), np.nan) for _ in range(2)] for _ in runs]

        def on_chunk(lo, hi, f, k, regret, avg):
            src = board_slots(f, rows).ravel()
            dst = mono_slots[lo:hi].ravel()
            out[k][0][dst], out[k][1][dst] = regret[src], avg[src]

        # seat 1 computes its chance-node row in a pass of its own; seat 0 reuses the evaluation's
        trunk = co.half_iterations(p, runs, on_chunk, chance_ev=got["current"]["ev"][p] if p == 0 else None)
        for k, (key, algo, it, delay) in enumerate(runs):
            out[k][0][:co.nts], out[k][1][:co.nts] = trunk[k]["regret"], trunk[k]["avg"]
            m = _mono(ft, ranks, algo, *profs[key].tables(ft, 0))
            m.iter_counter = it
            m.half_iteration(p)
            e = (_rel(out[k][0], m.regret), _rel(out[k][1], m.avg), _rel(trunk[k]["reach"], m.reach[:co.n_trunk_nodes]),
                 _rel(trunk[k]["strat"], m.strat[:co.nts]))
            print(name, algo, "seat", p, "chunked vs monolithic (regret, avg, trunk reach, trunk strategy): %.1e %.1e %.1e %.1e" % e)
            assert max(e) <= TOL, (algo, p, e)
            # the update changed the seat's rows: the comparison is not of the inputs with themselves
            assert _rel(m.regret, profs[key].tables(ft, 0)[0]) > 1e-3
