"""Pin the CPU oracle (oracle/cfr_numpy.py) against fixtures produced by the reference itself."""
import numpy as np
import pytest

import cfr_numpy as oc
from common import formula_profile_table, golden, make_flat_tree
from fixture_digest import array_digest


def _dfs(ft, arr_flat):
    return arr_flat[ft.dfs_permutation()]


@pytest.mark.parametrize("name", ["StandardLeduc", "NLLeduc_POT", "NLLeduc_B2"])
def test_uniform_and_random_profile_values_bit_exact(name):
    ft = make_flat_tree(name)
    g = golden("values_%s.npz" % name)
    t = oc.OracleTree(ft)
    t.fill_uniform()
    expl = t.compute_ev()
    for k, mine in (("reach", t.reach), ("ev", t.ev), ("ev_br", t.ev_br)):
        assert np.array_equal(_dfs(ft, mine), g["uniform_" + k]), k
    assert np.array_equal(expl, g["uniform_root_exploitability"])
    # seeded random profile: load the reference's float64 strategies
    strat = g["random_strat"]  # [N, R] in DFS order, column of the parent's strategy
    perm = ft.dfs_permutation()
    inv = ft.dfs
    for n in t.decision_nodes():
        fc, A = ft.first_child[n], ft.n_children[n]
        t.strategy[n] = np.stack([strat[inv[fc + a]] for a in range(A)], axis=1)
    t.update_reach()
    expl = t.compute_ev()
    for k, mine in (("reach", t.reach), ("ev", t.ev), ("ev_br", t.ev_br)):
        assert np.array_equal(_dfs(ft, mine), g["random_" + k]), k
    assert np.array_equal(expl, g["random_root_exploitability"])


def test_b3_uniform_root():
    ft = make_flat_tree("NLLeduc_B3")
    g = golden("values_NLLeduc_B3.npz")
    t = oc.OracleTree(ft)
    t.fill_uniform()
    expl = t.compute_ev()
    assert np.array_equal(t.ev[0], g["uniform_root_ev"])
    assert np.array_equal(t.ev_br[0], g["uniform_root_ev_br"])
    assert np.array_equal(expl, g["uniform_root_exploitability"])


@pytest.mark.parametrize("algo,name,n_iters", [
    ("CFRPlus", "NLLeduc_POT", 31), ("CFRPlus", "StandardLeduc", 31),
    ("LinearCFR", "NLLeduc_POT", 31), ("LinearCFR", "StandardLeduc", 11),
    ("VanillaCFR", "NLLeduc_POT", 11), ("VanillaCFR", "StandardLeduc", 31),
])
def test_cfr_trajectory_bit_exact(algo, name, n_iters):
    ft = make_flat_tree(name)
    g = golden("cfr_%s_%s.npz" % (algo, name))
    cfr = oc.OracleCFR(ft, algo=algo)
    snaps = [t for t in (0, 1, 2, 3, 4, 5, 10, 11, 30, 31) if t <= n_iters]

    def check(t):
        if t > 0:
            assert np.array_equal(_dfs(ft, cfr.table(cfr.regret)), g["it%d_regret" % t], equal_nan=True), t
            assert np.array_equal(_dfs(ft, cfr.table(cfr.avg_strat)), g["it%d_avg" % t], equal_nan=True), t
        assert np.array_equal(_dfs(ft, cfr.table(cfr.tree.strategy)), g["it%d_strat" % t], equal_nan=True), t
        assert np.array_equal(_dfs(ft, cfr.tree.ev), g["it%d_ev" % t]), t
        assert np.array_equal(_dfs(ft, cfr.tree.ev_br), g["it%d_ev_br" % t]), t

    check(0)
    for t in range(1, n_iters + 1):
        cfr.iteration()
        if t in snaps:
            check(t)
    curr = np.array(cfr.curr_series)
    avg = np.array(cfr.avg_series)
    assert np.array_equal(curr, g["curr_series"][:len(curr)])
    assert np.array_equal(avg, g["avg_series"][:len(avg)])


# ---------------------------------------------------------------------------------------------------- BigLeduc
# 24 hands: the reference's np.sum over hands runs in numpy's pairwise order.  Its fixtures hold SHA-256 digests of
# the DFS-ordered per-node arrays (oracle/fixture_digest.py) and the root rows in full.

def _digests_equal(g, prefix, arrays):
    for k, a in arrays.items():
        assert array_digest(a) == str(g["%s_%s_sha256" % (prefix, k)]), (prefix, k)


def test_bigleduc_uniform_and_formula_profile_values_bit_exact():
    ft = make_flat_tree("BigLeduc")
    g = golden("values_BigLeduc.npz")
    t = oc.OracleTree(ft)
    t.fill_uniform()
    expl = t.compute_ev()
    assert np.array_equal(t.ev[0], g["uniform_root_ev"]) and np.array_equal(t.ev_br[0], g["uniform_root_ev_br"])
    assert np.array_equal(expl, g["uniform_root_exploitability"])
    _digests_equal(g, "uniform", {k: _dfs(ft, a) for k, a in (("reach", t.reach), ("ev", t.ev), ("ev_br", t.ev_br))})
    tab = formula_profile_table(ft)
    for n in t.decision_nodes():
        fc, A = ft.first_child[n], ft.n_children[n]
        t.strategy[n] = tab[ft.slot[fc]:ft.slot[fc] + A].T.copy()
    t.update_reach()
    expl = t.compute_ev()
    assert np.array_equal(t.ev[0], g["formula_root_ev"]) and np.array_equal(t.ev_br[0], g["formula_root_ev_br"])
    assert np.array_equal(expl, g["formula_root_exploitability"])
    _digests_equal(g, "formula", {k: _dfs(ft, a) for k, a in (("reach", t.reach), ("ev", t.ev), ("ev_br", t.ev_br))})
    _digests_equal(g, "formula", {"strat": _dfs(ft, cfr_strategy_column(ft, t))})


def cfr_strategy_column(ft, t):
    """[N, R] float64: the parent's strategy column of every child of a decision node, NaN elsewhere (flat order)."""
    out = np.full((ft.n_nodes, ft.R), np.nan)
    for n in t.decision_nodes():
        fc, A = ft.first_child[n], int(ft.n_children[n])
        out[fc:fc + A] = np.asarray(t.strategy[n], np.float64).T
    return out


def test_bigleduc_cfr_plus_three_iterations_bit_exact():
    ft = make_flat_tree("BigLeduc")
    g = golden("cfr_CFRPlus_BigLeduc.npz")
    cfr = oc.OracleCFR(ft, algo="CFRPlus")

    def check(t):
        arrs = {"strat": cfr.table(cfr.tree.strategy), "reach": cfr.tree.reach, "ev": cfr.tree.ev, "ev_br": cfr.tree.ev_br}
        if t > 0:
            arrs.update(regret=cfr.table(cfr.regret), avg=cfr.table(cfr.avg_strat))
        _digests_equal(g, "it%d" % t, {k: _dfs(ft, a) for k, a in arrs.items()})
        assert np.array_equal(cfr.tree.ev[0], g["it%d_root_ev" % t]), t

    check(0)
    for t in range(1, 4):
        cfr.iteration()
        check(t)
    assert np.array_equal(np.array(cfr.curr_series), g["curr_series"][:4])
    assert np.array_equal(np.array(cfr.avg_series), g["avg_series"][:3])
