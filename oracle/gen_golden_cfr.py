"""Generate golden CFR / PublicTree fixtures by RUNNING THE REFERENCE ITSELF (TEST INFRASTRUCTURE).

Run in the build container only (needs a PokerRL checkout in POKERRL_REFERENCE):

    python oracle/gen_golden_cfr.py            # writes tests/golden/*.npz

What is pinned (all arrays DFS pre-order, see oracle/ref_harness.py):
  tree_<game>.npz      structure produced by PublicTree.build_tree (PublicTree.py:111-293)
  values_<game>.npz    reach/ev/ev_br of every node under the uniform profile and under a seeded random
                       profile (StrategyFiller.py:48-86, 118-146; ValueFiller.py:21-175)
  cfr_<algo>_<game>.npz  exploitability series logged by _CFRBase.py:198-262 and full regret / strategy /
                       average-strategy snapshots at selected iterations (CFRPlus.py, LinearCFR.py, VanillaCFR.py)
"""
import hashlib
import os
import sys
import time
from multiprocessing import Pool

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ref_harness as rh  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

GAMES = {
    # name: (game class name, bet set name)
    "StandardLeduc": ("StandardLeduc", "POT_ONLY"),
    "NLLeduc_POT": ("DiscretizedNLLeduc", "POT_ONLY"),
    "NLLeduc_B2": ("DiscretizedNLLeduc", "B_2"),
    "NLLeduc_B3": ("DiscretizedNLLeduc", "B_3"),
}


def _make_tree(game):
    rh.import_reference()
    from PokerRL.game import bet_sets, games
    from PokerRL.game._.tree.PublicTree import PublicTree
    from PokerRL.game.wrappers import HistoryEnvBuilder
    cls_name, bs = GAMES[game]
    game_cls = getattr(games, cls_name)
    args = game_cls.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[game_cls.DEFAULT_STACK_SIZE] * 2,
                             bet_sizes_list_as_frac_of_pot=list(getattr(bet_sets, bs)))
    bldr = HistoryEnvBuilder(env_cls=game_cls, env_args=args)
    tree = PublicTree(env_bldr=bldr, stack_size=args.starting_stack_sizes_list, stop_at_street=None)
    tree.build_tree()
    return tree, bldr


def structure_hash(s):
    h = hashlib.sha256()
    for k in ("parent", "kind", "action", "main_pot", "board", "n_children"):
        h.update(np.ascontiguousarray(s[k]).astype(np.int64).tobytes())
    return h.hexdigest()


def gen_tree(game):
    t0 = time.time()
    tree, bldr = _make_tree(game)
    s = rh.flatten_structure(tree)
    s["hash"] = np.array(structure_hash(s))
    s["n_nodes_reported"] = np.array(tree.n_nodes)
    s["n_nonterm_reported"] = np.array(tree.n_nonterm)
    np.savez_compressed(os.path.join(OUT, "tree_%s.npz" % game), **s)
    R = bldr.rules.RANGE_SIZE
    out = {}
    tree.fill_uniform_random()
    tree.compute_ev()
    if len(s["parent"]) < 5000:
        for k, v in rh.flatten_values(tree, R).items():
            out["uniform_" + k] = v
    out["uniform_root_ev"] = tree.root.ev
    out["uniform_root_ev_br"] = tree.root.ev_br
    out["uniform_root_exploitability"] = tree.root.exploitability
    if len(s["parent"]) < 5000:
        np.random.seed(1234)
        tree.fill_random_random()
        tree.compute_ev()
        for k, v in rh.flatten_values(tree, R).items():
            out["random_" + k] = v
        out["random_root_exploitability"] = tree.root.exploitability
    np.savez_compressed(os.path.join(OUT, "values_%s.npz" % game), **out)
    return game, len(s["parent"]), time.time() - t0


def gen_cfr(job):
    algo, game, n_iters, snaps = job
    rh.import_reference()
    from PokerRL.cfr.CFRPlus import CFRPlus
    from PokerRL.cfr.LinearCFR import LinearCFR
    from PokerRL.cfr.VanillaCFR import VanillaCFR
    from PokerRL.game import bet_sets, games
    from PokerRL.rl.base_cls.workers.ChiefBase import ChiefBase
    cls_name, bs = GAMES[game]
    game_cls = getattr(games, cls_name)
    chief = ChiefBase(t_prof=None)
    kw = dict(name="g", chief_handle=chief, game_cls=game_cls, agent_bet_set=list(getattr(bet_sets, bs)))
    t0 = time.time()
    if algo == "CFRPlus":
        cfr = CFRPlus(delay=0, **kw)
    elif algo == "LinearCFR":
        cfr = LinearCFR(**kw)
    else:
        cfr = VanillaCFR(**kw)
    tree = cfr._trees[0]
    R = cfr._env_bldrs[0].rules.RANGE_SIZE
    out = {}

    def snap(t):
        v = rh.flatten_values(tree, R)
        reg = rh.flatten_node_table(tree, "regret", R)
        out["it%d_regret" % t] = reg
        out["it%d_strat" % t] = v["strat"]
        out["it%d_avg" % t] = rh.flatten_node_table(tree, "avg_strat", R)
        if algo != "CFRPlus":
            out["it%d_avg_sum" % t] = rh.flatten_node_table(tree, "avg_strat_sum", R)
        out["it%d_reach" % t] = v["reach"]
        out["it%d_ev" % t] = v["ev"]
        out["it%d_ev_br" % t] = v["ev_br"]

    if 0 in snaps:
        snap(0)
    t_iter = []
    for t in range(1, n_iters + 1):
        t1 = time.perf_counter()
        cfr.iteration()
        t_iter.append(time.perf_counter() - t1)
        if t in snaps:
            snap(t)
    exps = chief._log_buf._experiments
    metric = "Evaluation/" + game_cls.WIN_METRIC
    curr = [e for e in exps if "_Curr_S" in e][0]
    avg = [e for e in exps if "_Avg_total_S" in e][0]
    out["curr_series"] = np.array(exps[curr][metric], dtype=np.float64)  # [[step, value], ...]
    out["avg_series"] = np.array(exps[avg][metric], dtype=np.float64)
    out["ref_seconds_per_iter"] = np.array(t_iter)
    out["numpy_version"] = np.array(np.__version__)
    np.savez_compressed(os.path.join(OUT, "cfr_%s_%s.npz" % (algo, game)), **out)
    return algo, game, n_iters, time.time() - t0


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    snaps = (0, 1, 2, 3, 4, 5, 10, 11, 30, 31)
    cfr_jobs = [
        ("CFRPlus", "NLLeduc_POT", 150, snaps + (150,)),
        ("CFRPlus", "StandardLeduc", 60, snaps),
        ("LinearCFR", "NLLeduc_POT", 40, snaps),
        ("LinearCFR", "StandardLeduc", 40, snaps),
        ("VanillaCFR", "NLLeduc_POT", 40, snaps),
        ("VanillaCFR", "StandardLeduc", 40, snaps),
    ]
    with Pool(8) as pool:
        r1 = pool.map_async(gen_cfr, cfr_jobs)
        r2 = pool.map_async(gen_tree, list(GAMES))
        for r in r2.get():
            print("tree", r)
        for r in r1.get():
            print("cfr", r)
