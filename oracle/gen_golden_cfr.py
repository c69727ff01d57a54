"""Generate golden CFR / PublicTree fixtures by RUNNING THE REFERENCE ITSELF (TEST INFRASTRUCTURE).

Run in the build container only (needs a PokerRL checkout in POKERRL_REFERENCE):

    python oracle/gen_golden_cfr.py            # writes tests/golden/*.npz

What is pinned (all arrays DFS pre-order, see oracle/ref_harness.py):
  tree_<game>.npz      structure produced by PublicTree.build_tree (PublicTree.py:111-293)
  values_<game>.npz    reach/ev/ev_br of every node under the uniform profile and under a seeded random
                       profile (StrategyFiller.py:48-86, 118-146; ValueFiller.py:21-175)
  cfr_<algo>_<game>.npz  exploitability series logged by _CFRBase.py:198-262 and full regret / strategy /
                       average-strategy snapshots at selected iterations (CFRPlus.py, LinearCFR.py, VanillaCFR.py)

BigLeduc (12 207 nodes, 24 hands) stores SHA-256 digests of its per-node arrays instead (oracle/fixture_digest.py,
keys ending in "_sha256"), plus the root rows and the series in full.  Its second value profile is not the seeded
random one but `fixture_digest.formula_strategy`, which the tests rebuild.  The reference's BigLeduc hand rank is run
with the one NumPy 2 fix of ref_harness._patch_big_leduc_hand_rank.

    python oracle/gen_golden_cfr.py BigLeduc   # only the fixtures of the named games
"""
import hashlib
import os
import sys
import time
from multiprocessing import Pool

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ref_harness as rh  # noqa: E402
from fixture_digest import array_digest, formula_strategy  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

GAMES = {
    # name: (game class name, bet set name)
    "StandardLeduc": ("StandardLeduc", "POT_ONLY"),
    "NLLeduc_POT": ("DiscretizedNLLeduc", "POT_ONLY"),
    "NLLeduc_B2": ("DiscretizedNLLeduc", "B_2"),
    "NLLeduc_B3": ("DiscretizedNLLeduc", "B_3"),
    "BigLeduc": ("BigLeduc", "POT_ONLY"),
}
DIGEST_GAMES = ("BigLeduc",)  # per-node arrays stored as digests


def fill_formula_profile(tree):
    """Decision-node strategies of fixture_digest.formula_strategy (chance nodes keep the uniform fill's), reach."""
    tree.fill_uniform_random()
    for i, n in enumerate(rh.dfs_nodes(tree)):
        if not n.is_terminal and n.p_id_acting_next in (0, 1):
            n.strategy = formula_strategy(i, len(n.children), tree.env_bldr.rules.RANGE_SIZE)
    tree.update_reach_probs()


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
    out["uniform_root_reach"] = tree.root.reach_probs
    out["numpy_version"] = np.array(np.__version__)
    if game in DIGEST_GAMES:
        for k, v in rh.flatten_values(tree, R).items():
            if k != "strat":
                out["uniform_%s_sha256" % k] = np.array(array_digest(v))
        fill_formula_profile(tree)
        tree.compute_ev()
        for k, v in rh.flatten_values(tree, R).items():
            out["formula_%s_sha256" % k] = np.array(array_digest(v))
        out["formula_root_reach"] = tree.root.reach_probs
        out["formula_root_ev"] = tree.root.ev
        out["formula_root_ev_br"] = tree.root.ev_br
        out["formula_root_exploitability"] = tree.root.exploitability
    elif len(s["parent"]) < 5000:
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

    def snap_digests(t):
        v = rh.flatten_values(tree, R)
        arrs = dict(regret=rh.flatten_node_table(tree, "regret", R), strat=v["strat"],
                    avg=rh.flatten_node_table(tree, "avg_strat", R), reach=v["reach"], ev=v["ev"], ev_br=v["ev_br"])
        if algo != "CFRPlus":
            arrs["avg_sum"] = rh.flatten_node_table(tree, "avg_strat_sum", R)
        for k, a in arrs.items():
            out["it%d_%s_sha256" % (t, k)] = np.array(array_digest(a))
        out["it%d_root_ev" % t] = tree.root.ev
        out["it%d_root_ev_br" % t] = tree.root.ev_br

    def snap(t):
        if game in DIGEST_GAMES:
            return snap_digests(t)
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
    only = sys.argv[1:] or list(GAMES)
    snaps = (0, 1, 2, 3, 4, 5, 10, 11, 30, 31)
    big_snaps = (0, 1, 2, 3, 10, 31)
    cfr_jobs = [
        ("CFRPlus", "NLLeduc_POT", 150, snaps + (150,)),
        ("CFRPlus", "StandardLeduc", 60, snaps),
        ("LinearCFR", "NLLeduc_POT", 40, snaps),
        ("LinearCFR", "StandardLeduc", 40, snaps),
        ("VanillaCFR", "NLLeduc_POT", 40, snaps),
        ("VanillaCFR", "StandardLeduc", 40, snaps),
        ("CFRPlus", "BigLeduc", 60, big_snaps),
        ("LinearCFR", "BigLeduc", 40, big_snaps),
        ("VanillaCFR", "BigLeduc", 40, big_snaps),
    ]
    cfr_jobs = [j for j in cfr_jobs if j[1] in only]
    with Pool(8) as pool:
        r1 = pool.map_async(gen_cfr, cfr_jobs)
        r2 = pool.map_async(gen_tree, [g for g in GAMES if g in only])
        for r in r2.get():
            print("tree", r)
        for r in r1.get():
            print("cfr", r)
