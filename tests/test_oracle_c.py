"""Pin the C oracle (oracle/cfr_oracle.c) against the reference's golden fixtures, bit for bit."""
import ctypes as C

import numpy as np
import pytest

import cfr_c
from common import formula_profile_table, golden, make_flat_tree
from fixture_digest import array_digest


def _node_vec(ft, a):
    return a.transpose(1, 0, 2)[ft.dfs_permutation()]


def _table(ft, a):
    out = np.full((ft.n_nodes, ft.R), np.nan)
    m = ft.slot >= 0
    out[m] = a[ft.slot[m]].astype(np.float64)
    return out[ft.dfs_permutation()]


@pytest.mark.parametrize("algo,name", [
    ("CFRPlus", "NLLeduc_POT"), ("CFRPlus", "StandardLeduc"), ("LinearCFR", "NLLeduc_POT"),
    ("LinearCFR", "StandardLeduc"), ("VanillaCFR", "NLLeduc_POT"), ("VanillaCFR", "StandardLeduc"),
])
def test_c_oracle_trajectory_bit_exact(algo, name):
    ft = make_flat_tree(name)
    g = golden("cfr_%s_%s.npz" % (algo, name))
    s = cfr_c.OracleCSolver(ft, algo, avg_f64=True)
    n_iters = len(g["curr_series"]) - 1
    curr, avg = [(0, s.exploitability_current())], []
    assert np.array_equal(_node_vec(ft, s.ev), g["it0_ev"])
    assert np.array_equal(_node_vec(ft, s.ev_br), g["it0_ev_br"])
    for t in range(1, n_iters + 1):
        s.iteration()
        curr.append((t, s.exploitability_current()))
        if t in (1, 2, 3, 10, 31):
            assert np.array_equal(_table(ft, s.regret), g["it%d_regret" % t], equal_nan=True), t
            assert np.array_equal(_table(ft, s.strat), g["it%d_strat" % t], equal_nan=True), t
            assert np.array_equal(_node_vec(ft, s.reach), g["it%d_reach" % t]), t
            key = "it%d_avg" % t if algo == "CFRPlus" else "it%d_avg_sum" % t
            assert np.array_equal(_table(ft, s.avg), g[key], equal_nan=True), t
        avg.append((t, s.exploitability_average()))
    assert np.array_equal(np.array(curr), g["curr_series"])
    assert np.array_equal(np.array(avg), g["avg_series"])


def test_c_oracle_b3_uniform_root():
    ft = make_flat_tree("NLLeduc_B3")
    g = golden("values_NLLeduc_B3.npz")
    s = cfr_c.OracleCSolver(ft, "CFRPlus")
    s.exploitability_current()
    assert np.array_equal(s.ev[:, 0], g["uniform_root_ev"])
    assert np.array_equal(s.ev_br[:, 0], g["uniform_root_ev_br"])


# ---------------------------------------------------------------------------------------------------- BigLeduc
# 24 hands: np.sum over hands in numpy's pairwise order (fold equity, root exploitability).  Fixtures hold SHA-256
# digests of the DFS-ordered per-node arrays (oracle/fixture_digest.py).

def _digests_equal(g, prefix, arrays):
    for k, a in arrays.items():
        assert array_digest(a) == str(g["%s_%s_sha256" % (prefix, k)]), (prefix, k)


def _root_expl(s, bufs):
    out = np.zeros(2, np.float32)
    s.L.orc_root_exploitability(C.byref(s.tree), C.byref(bufs), out.ctypes.data)
    return out


def test_c_oracle_bigleduc_uniform_and_formula_profile_values():
    from pokerrl_b200 import _native as nat
    ft = make_flat_tree("BigLeduc")
    g = golden("values_BigLeduc.npz")
    s = cfr_c.OracleCSolver(ft, "CFRPlus", avg_f64=True)
    s.exploitability_current()
    assert np.array_equal(_root_expl(s, s.bufs), g["uniform_root_exploitability"])
    _digests_equal(g, "uniform", {k: _node_vec(ft, a) for k, a in (("reach", s.reach), ("ev", s.ev), ("ev_br", s.ev_br))})
    s.avg[:] = formula_profile_table(ft)
    m = nat.modes(nat.STRAT_AVG_F64, nat.STRAT_AVG_F64)
    s.L.orc_reach_pass(C.byref(s.tree), C.byref(s.bufs), 3, m)
    s.L.orc_value_pass(C.byref(s.tree), C.byref(s.bufs), 3, 1, m)
    assert np.array_equal(s.ev[:, 0], g["formula_root_ev"]) and np.array_equal(s.ev_br[:, 0], g["formula_root_ev_br"])
    assert np.array_equal(_root_expl(s, s.bufs), g["formula_root_exploitability"])
    _digests_equal(g, "formula", {k: _node_vec(ft, a) for k, a in (("reach", s.reach), ("ev", s.ev), ("ev_br", s.ev_br))})


@pytest.mark.parametrize("algo", ["CFRPlus", "LinearCFR", "VanillaCFR"])
def test_c_oracle_bigleduc_trajectory_bit_exact(algo):
    ft = make_flat_tree("BigLeduc")
    g = golden("cfr_%s_BigLeduc.npz" % algo)
    s = cfr_c.OracleCSolver(ft, algo, avg_f64=True)
    n_iters = len(g["curr_series"]) - 1
    curr, avg = [(0, s.exploitability_current())], []
    _digests_equal(g, "it0", {"ev": _node_vec(ft, s.ev), "ev_br": _node_vec(ft, s.ev_br)})
    for t in range(1, n_iters + 1):
        s.iteration()
        curr.append((t, s.exploitability_current()))
        if t in (1, 2, 3, 10, 31):
            _digests_equal(g, "it%d" % t, {
                "regret": _table(ft, s.regret), "strat": _table(ft, s.strat), "reach": _node_vec(ft, s.reach),
                "ev": _node_vec(ft, s.ev), "ev_br": _node_vec(ft, s.ev_br),
                "avg" if algo == "CFRPlus" else "avg_sum": _table(ft, s.avg)})
        avg.append((t, s.exploitability_average()))
    assert np.array_equal(np.array(curr), g["curr_series"])
    assert np.array_equal(np.array(avg), g["avg_series"])
