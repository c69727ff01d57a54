"""The chunked float64 oracle (oracle/cfr2_chunked.py) against the monolithic C oracle (oracle/cfr2_c.Oracle2CSolver) on
games small enough for both: chance-node rows, exploitability of the current and the average strategy (CFR+, PCFR+), and
every table slot after each seat's half-iteration (CFR+, Linear CFR, DCFR and PCFR+ at iterations 5 and 997; seat 1's DCFR
and PCFR+ also with seat 0's average contribution pending) from the synthetic profile, to 1e-12.  This pins the machinery
behind the full-game GPU tests (tests/test_gpu_board_full_game.py, tests/test_gpu_board_full_game_dcfr_pcfr.py) on a CPU."""
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
    """CFR+, Linear CFR and DCFR share the regrets (one value sweep); PCFR+ has its own regrets and predictions"""
    return {"CFRPlus": SyntheticProfile(ft, seed=3, regret_exp=(-4, -12)),
            "LinearCFR": SyntheticProfile(ft, seed=3, regret_exp=(-4, -12), avg_exp=(-6, -16)),
            "PCFRPlus": SyntheticProfile(ft, seed=3, regret_exp=(-4, -12), avg_exp=(-6, -16), pcfr=True)}


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def _mono(ft, ranks, algo, regret, avg, pred=None):
    rk = np.full((ranks.shape[0] + 1, ft.R), -1, np.int32)
    rk[1:] = ranks
    o = cfr2_c.Oracle2CSolver(ft, rk, algo, lean=True, n_threads=4)
    o.regret[:], o.avg[:] = regret, avg
    if pred is not None:
        o.pred[:] = pred
    o.match()
    return o


def test_synthetic_profile_has_the_features_of_a_late_run():
    """mixed and pure strategies, uniform fallbacks, exact zeros; the same bits for the same keys, whatever the chunking"""
    spec = random_board_spec(12, 4)
    ft = fhp_tree(spec)
    prof = SyntheticProfile(ft, seed=3, regret_exp=(-4, -12))
    pcfr = SyntheticProfile(ft, seed=3, regret_exp=(-4, -12), pcfr=True)
    reg, avg = prof.board_rows(np.arange(12))
    r2, a2 = prof.board_rows(np.arange(5, 9))
    assert np.array_equal(reg[5:9].numpy(), r2.numpy()) and np.array_equal(avg[5:9].numpy(), a2.numpy())
    preg, pavg, pred = pcfr.board_rows(np.arange(12))
    q2 = pcfr.board_rows(np.arange(5, 9))[2]
    assert np.array_equal(pred[5:9].numpy(), q2.numpy())
    # PCFR+'s regrets are the clipped regrets of the same keys, its average rows the same
    assert np.array_equal(preg.numpy(), np.maximum(reg.numpy(), 0)) and np.array_equal(pavg.numpy(), avg.numpy())
    st = ft.board_subtree()
    rows = decision_rows(st)
    d = st["parent"][rows[0]]
    grp = [k for k, c in enumerate(rows) if st["parent"][c] == d]
    for name, r in (("regret", reg.numpy().astype(np.float64)), ("pred", pred.numpy().astype(np.float64))):
        assert np.all(r * 2.0 ** 32 == np.round(r * 2.0 ** 32))  # multiples of 2^-32: exact in float32 and float64
        pos = (r[:, grp] > 0).sum(axis=1)  # [boards, hands]: positive entries of the hand at node d
        for what, share in (("all <= 0", (pos == 0).mean()), ("pure", (pos == 1).mean()), ("mixed", (pos >= 2).mean()),
                            ("zero entries", (r == 0).mean())):
            print("synthetic profile %-6s: %-12s %.3f" % (name, what, share))
            assert 0.05 < share < 0.9, (name, what)
    assert (pred.numpy() >= 0).all() and not np.array_equal(pred.numpy() > 0, preg.numpy() > 0)  # a hash of its own
    tr = pcfr.trunk_rows()
    assert len(tr) == 3 and (tr[2].numpy() >= 0).all() and (tr[2].numpy() > 0).any()
    a = avg.numpy().astype(np.float64)[:, grp].sum(axis=1)
    assert np.abs(a - 1).max() < 1e-6


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

    # evaluation: chance-node rows and exploitability, current and average strategy (PCFR+: matching of the predictions
    # and the normalised sums)
    got = {}
    for key in ("CFRPlus", "PCFRPlus"):
        got[key] = co.evaluate(key, key)
        o = _mono(ft, ranks, key, *profs[key].tables(ft, 0))
        errs = {}
        for form in ("current", "average"):
            expl = o.exploitability_current() if form == "current" else o.exploitability_average()
            errs[form + " expl"] = abs(got[key][form]["expl"] - expl) / abs(expl)
            for k, ref in (("ev", o.ev[ch]), ("ev_br", o.ev_br[ch])):
                errs["%s %s" % (form, k)] = _rel(got[key][form][k], ref)
            # the bound rows: sum over permutations and boards of |mult * child|
            kids = np.arange(ft.first_child[ch], ft.first_child[ch] + ft.n_children[ch])
            mult = np.asarray(ft.board_mult, np.float64)[ft.board[kids]][:, None, None]
            ref_abs = (mult * np.abs(o.ev[kids])).sum(axis=0)[:, co.perms].sum(axis=1)
            errs[form + " abs_ev"] = _rel(got[key][form]["abs_ev"], ref_abs)
        print(name, key, "chunked vs monolithic oracle, evaluation:", {k: "%.1e" % v for k, v in errs.items()})
        assert max(errs.values()) <= TOL, (key, errs)

    # seat p's half-iteration from the synthetic tables, every slot.  One pass per strategy: CFR+, Linear CFR and DCFR
    # share the regrets (seat 1's DCFR also with seat 0's contribution pending: its own pass), PCFR+ its predictions.
    base = [("CFRPlus", "CFRPlus", ITER, 0), ("LinearCFR", "LinearCFR", ITER, 0)]
    dcfr = [("LinearCFR", "DCFR", ITER, 0), ("LinearCFR", "DCFR", 997, 0)]
    pcfr = [("PCFRPlus", "PCFRPlus", ITER, 0), ("PCFRPlus", "PCFRPlus", 997, 0)]
    nts = co.nts
    for p in (0, 1):
        for runs, pending in ([(base + dcfr, False), (pcfr, False)] if p == 0 else
                              [(base, False), (dcfr, True), (pcfr, True)]):
            pc = runs[0][1] == "PCFRPlus"
            out = [[np.full((ft.n_slots, ft.R), np.nan) for _ in range(3 if pc else 2)] for _ in runs]

            def on_chunk(lo, hi, f, k, *tabs):
                src = board_slots(f, rows).ravel()
                dst = mono_slots[lo:hi].ravel()
                for o_, t_ in zip(out[k], tabs):
                    o_[dst] = t_[src]

            # seat 1 computes its chance-node row in a pass of its own; seat 0 reuses the evaluation's
            ev0 = got["PCFRPlus" if pc else "CFRPlus"]["current"]["ev"][p] if p == 0 else None
            trunk = co.half_iterations(p, runs, on_chunk, chance_ev=ev0, pending=pending)
            for k, (key, algo, it, delay) in enumerate(runs):
                out[k][0][:nts], out[k][1][:nts] = trunk[k]["regret"], trunk[k]["avg"]
                if pc:
                    out[k][2][:nts] = trunk[k]["pred"]
                tabs = profs[key].tables(ft, 0)
                m = _mono(ft, ranks, algo, *tabs)
                if pending:  # seat 0's contribution of the same iteration on the post-deal rows only
                    keep = m.avg[:nts].copy()
                    cfr2_c.set_factors(m.t, algo, it)
                    m.L.orc2_avg_update(C.byref(m.t), 0, cfr2_c.ALGOS[algo], it, 0)
                    m.avg[:nts] = keep
                m.iter_counter = it
                m.half_iteration(p)
                e = [_rel(out[k][0], m.regret), _rel(out[k][1], m.avg), _rel(trunk[k]["reach"], m.reach[:co.n_trunk_nodes]),
                     _rel(trunk[k]["strat"], m.strat[:nts])]
                if pc:
                    e.append(_rel(out[k][2], m.pred))
                print(name, algo, it, "seat", p, "pending" if pending else "",
                      "chunked vs monolithic (regret, avg, trunk reach, trunk strategy[, pred]):", " ".join("%.1e" % x for x in e))
                assert max(e) <= TOL, (algo, it, p, pending, e)
                # the update changed the seat's rows: the comparison is not of the inputs with themselves
                for got_t, inp in zip((m.regret, m.avg) + ((m.pred,) if pc else ()), tabs):
                    assert _rel(got_t, inp) > 1e-3, (algo, it, p)
                if pending:  # seat 0's post-deal sums moved too
                    st = ft.board_subtree()
                    s0 = mono_slots[:, [i for i, c in enumerate(rows) if st["kind"][st["parent"][c]] == 0]].ravel()
                    assert _rel(m.avg[s0], tabs[1][s0]) > 1e-3, (algo, it)
