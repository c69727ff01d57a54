"""Best response on the board engine (board_engine.BoardPolicyEvaluator, the board-table agent of TabularCFREvalAgent and
prl_board_policy_query) against the float64 C oracle, the level-engine PublicTree and the solver's own evaluation."""
import ctypes as C
import time

import numpy as np
import pytest
import torch

import cfr2_c
from pokerrl_b200.board_engine import BoardPolicyEvaluator, board_keys
from pokerrl_b200.game import games
from pokerrl_b200.game.PublicTree import PublicTree
from pokerrl_b200.game.holdem_boards import BoardSpec, canonical_keys, suit_permutation_hand_tables
from pokerrl_b200.game.wrappers import HistoryEnvBuilder
from twocard_common import oracle_tree, random_board_spec

pytestmark = pytest.mark.gpu
G = games.Flop5Holdem
STACK = [20000, 20000]
TOL = 1e-6


def _bldr():
    return HistoryEnvBuilder(env_cls=G, env_args=G.ARGS_CLS(n_seats=2, starting_stack_sizes_list=list(STACK),
                                                            bet_sizes_list_as_frac_of_pot=[1.0]))


def _mix(x):  # splitmix64 finaliser on uint64 arrays
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


class HashAgent:
    """suit-asymmetric, hand-dependent policy: the probabilities are a hash of (board, abstract node, hand); about a fifth of
    the (node, hand) pairs are pure, another fifth put zero on one action"""

    def __init__(self, n_actions):
        self.n_actions = n_actions

    def probs(self, ft, nodes):
        R = ft.R
        keys = np.concatenate([[0], board_keys(ft.board_spec.boards)]).astype(np.uint64)
        out = np.zeros((len(nodes), R, self.n_actions), np.float32)
        h = np.arange(R, dtype=np.uint64)
        with np.errstate(over="ignore"):
            for d, n in enumerate(nodes):
                fc, A = int(ft.first_child[n]), int(ft.n_children[n])
                acts = ft.action[fc:fc + A]
                base = _mix(keys[max(int(ft.board[n]), 0)] * np.uint64(1000003) + np.uint64(int(ft.abs_id[n]) * 7919)) + h
                x = _mix(base)
                w = np.stack([(_mix(x + np.uint64(a + 1)) >> np.uint64(11)).astype(np.float64) / 2.0 ** 53 + 0.01
                              for a in range(A)], axis=1)
                kind = (x % np.uint64(5)).astype(np.int64)
                pick = ((x >> np.uint64(8)) % np.uint64(A)).astype(np.int64)
                onehot = np.eye(A)[pick]
                w = np.where((kind == 0)[:, None], onehot, np.where((kind == 1)[:, None], w * (1 - onehot), w))
                out[d][:, acts] = (w / w.sum(axis=1, keepdims=True)).astype(np.float32)
        return out

    def get_a_probs_for_public_tree(self, tree):
        return torch.from_numpy(self.probs(tree.flat, tree.decision_nodes())).to(tree.dtree.device)

    def set_to_public_tree_node_state(self, node):
        self._node = node

    def get_a_probs_for_each_hand(self):
        return self.probs(self._node.tree.flat, [self._node.idx])[0]


class PerNodeHashAgent(HashAgent):
    def get_a_probs_for_public_tree(self, tree):
        return None


def _oracle_expl(spec, agent):
    from twocard_common import fhp_tree
    ft = fhp_tree(spec)
    orc = cfr2_c.Oracle2CSolver(ft, oracle_tree(ft).board_ranks, "CFRPlus", n_threads=8)
    dec = np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]
    pr = agent.probs(ft, dec)
    for d, n in enumerate(dec):
        fs, fc, A = int(ft.first_slot[n]), int(ft.first_child[n]), int(ft.n_children[n])
        orc.strat[fs:fs + A] = pr[d][:, ft.action[fc:fc + A]].T.astype(np.float64)
    orc.L.orc2_reach(C.byref(orc.t), orc.strat.ctypes.data)
    return orc.compute_ev()


def _level_expl(spec, agent):
    pt = PublicTree(_bldr(), STACK, None, put_out_new_round_after_limit=True, board_spec=spec)
    pt.build_tree()
    pt.fill_with_agent_policy(agent)
    pt.compute_ev()
    return np.asarray(pt.root.exploitability, np.float64)


SPECS = {"random300": lambda: random_board_spec(300, 17),
         "deck16_iso": lambda: BoardSpec.full_game(G.RULES, isomorphic=True, deck_subset=list(range(36, 52)))}


@pytest.mark.parametrize("name", sorted(SPECS))
def test_hash_agent_against_the_float64_oracle_and_the_level_engine(name):
    spec = SPECS[name]()
    agent = HashAgent(_bldr().N_ACTIONS)
    got = BoardPolicyEvaluator(_bldr(), STACK, spec).evaluate(agent)
    ref = _oracle_expl(spec, agent)
    lvl = _level_expl(spec, agent)
    for what, r in (("oracle", ref), ("level engine", lvl)):
        err = np.abs(got - r) / np.abs(r)
        print("%s: board evaluator vs %s per-seat relative error %.2e %.2e" % (name, what, err[0], err[1]))
        assert np.all(err <= TOL), (name, what, got, r)


def test_chunking_and_per_node_agents_give_the_same_bits():
    spec = random_board_spec(300, 17)
    agent = HashAgent(_bldr().N_ACTIONS)
    res = {c: BoardPolicyEvaluator(_bldr(), STACK, spec, chunk=c).evaluate(agent) for c in (1, 7, 64, None)}
    for c, e in res.items():
        assert np.array_equal(e, res[None]), (c, e, res[None])
    per_node = BoardPolicyEvaluator(_bldr(), STACK, spec).evaluate(PerNodeHashAgent(_bldr().N_ACTIONS))
    assert np.array_equal(per_node, res[None])


def _train(algo_cls, spec, iters, name):
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    chief = ChiefBase(t_prof=None)
    cfr = algo_cls(name=name, chief_handle=chief, game_cls=G, agent_bet_set=[1.0], starting_stack_sizes=[STACK[0]],
                   eval_every=iters, board_spec=spec)
    for _ in range(iters):
        cfr.iteration()
    avg = [v for k, v in chief.get_experiments().items() if k.startswith(name + "_Avg_total_S")][0]
    return cfr, chief, avg["Evaluation/" + G.WIN_METRIC][-1][1]


def _br(cfr, chief, spec, name):
    from pokerrl_b200.cfr.TabularCFREvalAgent import TabularCFREvalAgent
    from pokerrl_b200.eval.br.LocalBRMaster import LocalBRMaster
    from pokerrl_b200.rl.base_cls.TrainingProfileBase import TrainingProfileBase
    t_prof = TrainingProfileBase(name, G, [1.0], eval_stack_sizes=[list(STACK)])
    br = LocalBRMaster(t_prof=t_prof, chief_handle=chief, eval_agent_cls=TabularCFREvalAgent, board_spec=spec)
    br._eval_agent = TabularCFREvalAgent.from_cfr(t_prof, cfr)
    t0 = time.time()
    br.evaluate(iter_nr=cfr.iter_counter)
    dt = time.time() - t0
    got = [v for k, v in chief.get_experiments().items() if k.startswith(name + " ") and k.endswith(": BR Total")][0]
    return br, got["Evaluation/" + G.WIN_METRIC][-1][1], dt


@pytest.fixture(scope="module")
def full_game():
    from pokerrl_b200.cfr.CFRPlus import CFRPlus
    torch.cuda.reset_peak_memory_stats()
    cfr, chief, avg = _train(CFRPlus, None, 20, "fg")
    br, val, dt = _br(cfr, chief, None, "fg")
    print("full game CFR+ 20 iterations: _Avg_total %r, BR %r (evaluation %.1f s)" % (avg, val, dt))
    return dict(cfr=cfr, chief=chief, avg=avg, br=br, val=val, agent=br.eval_agent)


def test_full_game_cfrp_agent_br_equals_the_solvers_average_evaluation(full_game):
    """same rows, sweep kernel and integer chance sums: bit for bit"""
    assert full_game["val"] == full_game["avg"], (full_game["val"], full_game["avg"])


@pytest.mark.parametrize("algo", ["CFRPlus", "LinearCFR"])
def test_small_spec_trained_agent(algo):
    from pokerrl_b200.cfr.CFRPlus import CFRPlus
    from pokerrl_b200.cfr.LinearCFR import LinearCFR
    spec = random_board_spec(300, 3)
    cfr, chief, avg = _train({"CFRPlus": CFRPlus, "LinearCFR": LinearCFR}[algo], spec, 20, "s" + algo)
    _, val, _ = _br(cfr, chief, spec, "s" + algo)
    print("%s 300 boards: _Avg_total %r, BR %r, relative %.2e" % (algo, avg, val, abs(val - avg) / abs(avg)))
    if algo == "CFRPlus":
        assert val == avg
    else:  # normalised on the host by division, in the sweep by the kernel's normalisation
        assert abs(val - avg) <= TOL * abs(avg)


def _restated(agent, boards, ft_rows):
    """numpy restatement of prl_board_policy_query at the post-deal decision nodes: [n, 6, R, n_actions]"""
    from pokerrl_b200.board_engine import _decision_locals
    b = agent._board
    st = ft_rows.board_subtree()
    keys = b.keys.cpu().numpy()
    ck, s = canonical_keys(boards)
    cls = np.searchsorted(keys, ck)
    assert np.all(keys[cls] == ck)
    hp = suit_permutation_hand_tables()
    ph = b.pos_hand[torch.from_numpy(cls).to(b.pos_hand.device)].cpu().numpy().astype(np.int64)  # [n, 1081]
    rpb = 14
    rows = b.rows.view(-1, rpb, b.rows.shape[1])[torch.from_numpy(cls).to(b.rows.device)].cpu().numpy()
    from pokerrl_b200.board_engine import board_game
    _, _, local_rows = board_game(st, G.RULES, 1, 1328, 24, grid=1)
    locs = _decision_locals(st)
    n, R, nA = len(boards), 1326, agent._n_actions
    out = np.zeros((n, len(locs), R, nA), np.float32)
    hc = np.asarray(G.RULES.get_lut_holder().LUT_IDX_2_HOLE_CARDS).astype(np.int64)
    for q in range(n):
        pos = np.full(R, -1, np.int64)
        pos[ph[q]] = np.arange(ph.shape[1])
        blocked = np.isin(hc, boards[q]).any(axis=1)
        hh = hp[s[q]].astype(np.int64)
        p = np.where(blocked, -1, pos[hh])
        for d, i in enumerate(locs):
            for c in range(st["first_child"][i], st["first_child"][i] + st["n_children"][i]):
                a = int(ft_rows.action[st["node_base"][c] + st["node_k"][c]])
                out[q, d, :, a] = np.where(p >= 0, rows[q, local_rows[c][0], np.maximum(p, 0)], 0.0)
    return out


def test_query_kernel_against_numpy(full_game):
    from twocard_common import fhp_tree
    agent = full_game["agent"]
    rng = np.random.default_rng(5)
    rand = np.sort(np.stack([rng.choice(52, 5, replace=False) for _ in range(1700)]), axis=1)
    special = []
    while len(special) < 300:
        kind = len(special) % 4
        r = rng.choice(13, 5, replace=False)
        s = rng.integers(0, 4, 5)
        if kind == 0:  # paired
            r, s = np.array([r[0], r[0], r[1], r[2], r[3]]), np.array([0, 1, s[2], s[3], s[4]])
        elif kind == 1:  # flush (monotone)
            s = np.full(5, s[0])
        elif kind == 2:  # four to a flush
            s = np.array([s[0]] * 4 + [(s[0] + 1) % 4])
        else:  # suit-symmetric: the same ranks on two suits
            r, s = np.array([r[0], r[0], r[1], r[1], r[2]]), np.array([0, 1, 0, 1, 2])
        b = np.sort(r * 4 + s)
        if len(set(b.tolist())) == 5:
            special.append(b)
    boards = np.unique(np.concatenate([rand, np.array(special)]).astype(np.int8), axis=0)[:2000]
    spec = BoardSpec(boards, np.ones(len(boards)), np.ones(len(boards)), None, "query boards")
    ft = fhp_tree(spec)
    pt = type("T", (), {})()
    pt.flat, pt.dtree = ft, type("D", (), {"device": torch.device("cuda:0")})()
    got = agent.get_a_probs_for_public_tree(pt).cpu().numpy()
    want = _restated(agent, boards.astype(np.int64), ft)
    st = ft.board_subtree()
    from pokerrl_b200.board_engine import _decision_locals
    dec = np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]
    dec_idx = np.full(ft.n_nodes, -1, np.int64)
    dec_idx[dec] = np.arange(dec.size)
    J = np.arange(len(boards))
    for d, i in enumerate(_decision_locals(st)):
        rows = dec_idx[st["node_base"][i] + J * st["node_m"][i] + st["node_k"][i]]
        assert np.array_equal(got[rows], want[:, d]), d
    # one-node queries are slices of the batched answer
    from pokerrl_b200.game.PublicTree import NodeView
    for n in list(dec[:5]) + list(rng.choice(dec, 20, replace=False)):
        agent.set_to_public_tree_node_state(NodeView(pt, n))
        assert np.array_equal(agent.get_a_probs_for_each_hand(), got[dec_idx[n]])


def test_non_isomorphic_agent_queried_off_its_spec_raises():
    from pokerrl_b200.cfr.CFRPlus import CFRPlus
    from pokerrl_b200.cfr.TabularCFREvalAgent import TabularCFREvalAgent
    from pokerrl_b200.rl.base_cls.TrainingProfileBase import TrainingProfileBase
    spec = random_board_spec(40, 9)
    cfr, _, _ = _train(CFRPlus, spec, 2, "off")
    agent = TabularCFREvalAgent.from_cfr(TrainingProfileBase("off", G, [1.0], eval_stack_sizes=[list(STACK)]), cfr)
    pt = PublicTree(_bldr(), STACK, None, board_spec=random_board_spec(40, 10))
    pt.build_structure()
    with pytest.raises(ValueError, match="not in this agent's board spec"):
        agent.get_a_probs_for_public_tree(pt)
    same = PublicTree(_bldr(), STACK, None, board_spec=spec)
    same.build_structure()
    assert agent.get_a_probs_for_public_tree(same).shape[0] == same.decision_nodes().size


def test_all_deals_match_the_classes(full_game):
    """the full-game CFR+ agent on every one of the 2 598 960 deals: the class representatives' answers mapped onto each
    deal; differs from the class-based value only where a class's rows are suit-symmetric up to rounding"""
    agent, val = full_game["agent"], full_game["val"]
    spec = BoardSpec.full_game(G.RULES, isomorphic=False)
    assert spec.boards.shape[0] == 2598960
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    ev = BoardPolicyEvaluator(_bldr(), STACK, spec)
    e = ev.evaluate(agent, profile=True)
    dt = time.time() - t0
    peak = torch.cuda.max_memory_allocated()
    got = (float(e[0]) * G.EV_NORMALIZER + float(e[1]) * G.EV_NORMALIZER) / 2
    rel = abs(got - val) / abs(val)
    print("all deals: %.6f vs classes %.6f mbb/g, relative difference %.2e; %.1f s (%s), chunk %d, peak %.2f GB above %.2f GB"
          % (got, val, rel, dt, ", ".join("%s %.1f s" % kv for kv in ev.times.items()), ev.chunk, (peak - base) / 1e9,
             base / 1e9))
    assert rel <= TOL
    bound = ev.chunk * ev.bytes_per_board + 256 * 2 ** 20  # chunk formula + trunk, chance sums, hand-rank batch
    assert peak - base <= bound, (peak - base, bound)
