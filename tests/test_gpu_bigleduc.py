"""BigLeduc (12 ranks x 2 suits, 6 raises per round, stack 100) on the one-card CUDA kernels, against the reference.

BigLeduc runs the R = 24 instantiations of csrc/cfr_levels.cu: one node per warp, lanes 24-31 idle, a 24-lane shuffle
group.  Its rows of 24 hands are long enough for np.sum to use numpy's pairwise order, which the kernels follow in the
fold equity and the root exploitability.  Every float32 quantity is compared bit for bit, like the Leduc tests in
test_gpu_cfr.py.  The fixtures (oracle/gen_golden_cfr.py) hold SHA-256 digests of the DFS-ordered per-node arrays
(oracle/fixture_digest.py), the root rows and the logged series in full.
"""
import numpy as np
import pytest
import torch

from common import formula_profile_table, golden, make_flat_tree
from fixture_digest import array_digest

pytestmark = pytest.mark.gpu


def _node_vec(ft, t):  # torch [2, N, ld] -> numpy [N, 2, R] in DFS order
    a = t.cpu().numpy()[:, :, :ft.R].transpose(1, 0, 2)
    return a[ft.dfs_permutation()]


def _table(ft, t):  # torch [n_slots, ld] -> numpy [N, R] (NaN where the node has no slot) in DFS order
    a = t.cpu().numpy()[:, :ft.R].astype(np.float64)
    out = np.full((ft.n_nodes, ft.R), np.nan)
    m = ft.slot >= 0
    out[m] = a[ft.slot[m]]
    return out[ft.dfs_permutation()]


def _digests_equal(g, prefix, arrays):
    for k, a in arrays.items():
        assert array_digest(a) == str(g["%s_%s_sha256" % (prefix, k)]), (prefix, k)


def _values(ft, s):
    return {"reach": _node_vec(ft, s.bufs.reach), "ev": _node_vec(ft, s.bufs.ev), "ev_br": _node_vec(ft, s.bufs.ev_br)}


def test_uniform_and_formula_profile_bit_exact():
    from pokerrl_b200 import _native as nat
    from pokerrl_b200.solver import CFRSolver
    ft = make_flat_tree("BigLeduc")
    g = golden("values_BigLeduc.npz")
    s = CFRSolver(ft, "CFRPlus", avg_f64=True)
    s.exploitability_current()
    assert np.array_equal(s.bufs.ev[:, 0, :ft.R].cpu().numpy(), g["uniform_root_ev"])
    assert np.array_equal(s.ops.root_exploitability(), g["uniform_root_exploitability"])
    _digests_equal(g, "uniform", _values(ft, s))
    # the formula profile as a float64 table, evaluated like an average strategy
    s.bufs.avg.copy_(torch.from_numpy(formula_profile_table(ft)))
    modes = [nat.STRAT_AVG_F64, nat.STRAT_AVG_F64]
    s.ops.reach_pass(modes)
    s.ops.value_pass(modes, 3, True)
    assert np.array_equal(s.bufs.ev[:, 0, :ft.R].cpu().numpy(), g["formula_root_ev"])
    assert np.array_equal(s.bufs.ev_br[:, 0, :ft.R].cpu().numpy(), g["formula_root_ev_br"])
    assert np.array_equal(s.ops.root_exploitability(), g["formula_root_exploitability"])
    _digests_equal(g, "formula", _values(ft, s))


@pytest.mark.parametrize("algo", ["CFRPlus", "LinearCFR", "VanillaCFR"])
@pytest.mark.parametrize("persistent", [True, False])
def test_cfr_trajectory_bit_exact(algo, persistent):
    from pokerrl_b200.solver import CFRSolver
    ft = make_flat_tree("BigLeduc")
    g = golden("cfr_%s_BigLeduc.npz" % algo)
    s = CFRSolver(ft, algo, avg_f64=True, persistent=persistent)
    n_iters = len(g["curr_series"]) - 1
    curr, avg = [(0, s.exploitability_current())], []
    for t in range(1, n_iters + 1):
        s.iteration()
        curr.append((t, s.exploitability_current()))
        if t in (1, 2, 3, 10, 31):
            arrs = dict(_values(ft, s), regret=_table(ft, s.bufs.regret), strat=_table(ft, s.bufs.strat))
            arrs["avg" if algo == "CFRPlus" else "avg_sum"] = _table(ft, s.bufs.avg)
            _digests_equal(g, "it%d" % t, arrs)
        avg.append((t, s.exploitability_average()))
    assert np.array_equal(np.array(curr), g["curr_series"]), "current-strategy exploitability series"
    assert np.array_equal(np.array(avg), g["avg_series"]), "average-strategy exploitability series"


def test_persistent_multi_iteration_launch_matches_golden():
    """20 iterations inside one cooperative launch land on the reference's iteration-20/40/60 numbers."""
    from pokerrl_b200.solver import CFRSolver
    ft = make_flat_tree("BigLeduc")
    g = golden("cfr_CFRPlus_BigLeduc.npz")
    s = CFRSolver(ft, "CFRPlus", avg_f64=True)
    for t in (20, 40, 60):
        s.iteration(20)
        assert s.exploitability_current() == g["curr_series"][t, 1]
        assert s.exploitability_average() == g["avg_series"][t - 1, 1]


def test_cfr_plus_float32_average_within_tolerance():
    """The float32 average table stays within 1e-6 relative of the float64-average reference run."""
    from pokerrl_b200.solver import CFRSolver
    ft = make_flat_tree("BigLeduc")
    g = golden("cfr_CFRPlus_BigLeduc.npz")
    s = CFRSolver(ft, "CFRPlus", avg_f64=False)
    for t in range(1, len(g["avg_series"]) + 1):
        s.iteration()
        a = s.exploitability_average()
        ref = g["avg_series"][t - 1, 1]
        assert abs(a - ref) <= 1e-6 * abs(ref), (t, a, ref)


def _series(chief, tag, metric):
    exps = chief.get_experiments()
    return np.array([e for k, e in exps.items() if tag in k][0][metric], dtype=np.float64)


def test_facade_logs_the_reference_series():
    """CFRPlus(game_cls=BigLeduc) through the PokerRL-style facade logs the reference's MA_per_G series."""
    from pokerrl_b200.cfr.CFRPlus import CFRPlus
    from pokerrl_b200.game import bet_sets
    from pokerrl_b200.game.games import BigLeduc
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    g = golden("cfr_CFRPlus_BigLeduc.npz")
    chief = ChiefBase(t_prof=None)
    cfr = CFRPlus(name="big", chief_handle=chief, game_cls=BigLeduc, agent_bet_set=bet_sets.POT_ONLY, delay=0,
                  avg_f64=True)
    for _ in range(len(g["avg_series"])):
        cfr.iteration()
    metric = "Evaluation/" + BigLeduc.WIN_METRIC
    assert metric == "Evaluation/MA_per_G"
    assert np.array_equal(_series(chief, "_Curr_S", metric), g["curr_series"])
    assert np.array_equal(_series(chief, "_Avg_total_S", metric), g["avg_series"])


def test_local_br_master_with_tabular_agent_matches_internal_average_evaluation():
    """LocalBRMaster on the tabular agent == the solver's own average-strategy exploitability, on BigLeduc."""
    from pokerrl_b200.cfr.CFRPlus import CFRPlus
    from pokerrl_b200.cfr.TabularCFREvalAgent import TabularCFREvalAgent, average_strategy_table
    from pokerrl_b200.eval.br.LocalBRMaster import LocalBRMaster
    from pokerrl_b200.game import bet_sets
    from pokerrl_b200.game.games import BigLeduc
    from pokerrl_b200.rl.base_cls.TrainingProfileBase import TrainingProfileBase
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    chief = ChiefBase(t_prof=None)
    cfr = CFRPlus(name="k", chief_handle=chief, game_cls=BigLeduc, agent_bet_set=bet_sets.POT_ONLY, delay=0)
    for _ in range(12):
        cfr.iteration()
    metric = "Evaluation/" + BigLeduc.WIN_METRIC
    ref = _series(chief, "_Avg_total_S", metric)[-1]
    t_prof = TrainingProfileBase("k", BigLeduc, bet_sets.POT_ONLY)
    br = LocalBRMaster(t_prof=t_prof, chief_handle=chief, eval_agent_cls=TabularCFREvalAgent)
    br.eval_agent.update_weights(average_strategy_table(cfr.solvers[0]))
    br.evaluate(iter_nr=12)
    got = _series(chief, ": BR Total", metric)[-1]
    assert got[0] == 12 and got[1] == ref[1]
