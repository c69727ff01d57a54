"""Best response as a playable agent: BoardPolicyEvaluator.best_response (the export form of the board sweep),
PublicTree.best_response_table (level engine) and LocalBRMaster.best_response_agent.

The main check does not depend on ties: an agent that plays the best response at seat s and the evaluated agent everywhere
else has an exploitability of exactly 0.0 at seat s.  Seat s's child values depend only on the opponent's reach and the
payoffs; a one-hot strategy makes ev equal the chosen child's value exactly; the opponent's nodes sum ev and ev_br over the
same children; the chance sums are integers."""
import gc

import numpy as np
import pytest
import torch

from pokerrl_b200.board_engine import BoardPolicyEvaluator
from pokerrl_b200.game import games
from pokerrl_b200.game.PublicTree import PublicTree
from pokerrl_b200.game.wrappers import HistoryEnvBuilder
from test_gpu_board_br import HashAgent, PerNodeHashAgent
from twocard_common import fhp_tree, oracle_tree, random_board_spec

pytestmark = pytest.mark.gpu
G = games.Flop5Holdem
MARGIN = 1e-5


def _bldr(stack):
    return HistoryEnvBuilder(env_cls=G, env_args=G.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[stack, stack],
                                                            bet_sizes_list_as_frac_of_pot=[1.0]))


def _t_prof(name, stack, game=G):
    from pokerrl_b200.rl.base_cls.TrainingProfileBase import TrainingProfileBase
    return TrainingProfileBase(name, game, [1.0], eval_stack_sizes=[[stack, stack]])


class _Hash(HashAgent):
    def set_stack_size(self, stack_size):  # what LocalBRMaster tells its agent
        pass


class Composite:
    """the best response `br` at seat `seat`'s decision nodes, `base` at every other node"""

    def __init__(self, br, base, seat):
        self.br, self.base, self.seat = br, base, seat

    def get_a_probs_for_public_tree(self, tree):
        pb = self.base.get_a_probs_for_public_tree(tree)
        if pb is None:
            return None
        pr = torch.as_tensor(self.br.get_a_probs_for_public_tree(tree)).to(pb.device)
        kind = torch.from_numpy(tree.flat.kind[tree.decision_nodes()].astype(np.int64)).to(pb.device)
        return torch.where((kind == self.seat)[:, None, None], pr, torch.as_tensor(pb, dtype=torch.float32))

    def set_to_public_tree_node_state(self, node):
        self._node = node
        self.br.set_to_public_tree_node_state(node)
        self.base.set_to_public_tree_node_state(node)

    def get_a_probs_for_each_hand(self):
        who = self.br if self._node.tree.flat.kind[self._node.idx] == self.seat else self.base
        return np.asarray(who.get_a_probs_for_each_hand(), np.float32)


def _cfr_agent(spec, stack, iters, name):
    from pokerrl_b200.cfr.CFRPlus import CFRPlus
    from pokerrl_b200.cfr.TabularCFREvalAgent import TabularCFREvalAgent
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    cfr = CFRPlus(name=name, chief_handle=ChiefBase(None), game_cls=G, agent_bet_set=[1.0], starting_stack_sizes=[stack],
                  eval_every=10 ** 9, board_spec=spec)
    for _ in range(iters):
        cfr.iteration()
    return TabularCFREvalAgent.from_cfr(_t_prof(name, stack), cfr)


def _br_agent(tables, stack):
    from pokerrl_b200.cfr.TabularCFREvalAgent import TabularCFREvalAgent
    return TabularCFREvalAgent.from_board_tables(_t_prof("br", stack), tables)


def _agent(kind, spec, stack):
    n_actions = _bldr(stack).N_ACTIONS
    return {"hash": lambda: HashAgent(n_actions), "per_node_hash": lambda: PerNodeHashAgent(n_actions),
            "cfrp": lambda: _cfr_agent(spec, stack, 6, "c%d" % stack)}[kind]()


@pytest.mark.parametrize("stack", [20000, 600])
@pytest.mark.parametrize("kind", ["hash", "per_node_hash", "cfrp"])
def test_composite_with_the_best_response_is_exactly_unexploitable(stack, kind):
    spec = random_board_spec(48, 100 + stack % 7)
    agent = _agent(kind, spec, stack)
    ref = BoardPolicyEvaluator(_bldr(stack), [stack, stack], spec).evaluate(agent)
    first = None
    for chunk in (1, 7, None):
        ev = BoardPolicyEvaluator(_bldr(stack), [stack, stack], spec, chunk=chunk)
        e, tables = ev.best_response(agent)
        assert np.array_equal(e, ref), (chunk, e, ref)  # bit-identical to evaluate(), any chunking
        if first is None:
            first = tables
        else:  # the exported tables do not depend on the chunking either
            assert torch.equal(tables.rows, first.rows) and torch.equal(tables.trunk, first.trunk), chunk
            assert torch.equal(tables.pos_hand, first.pos_hand) and torch.equal(tables.keys, first.keys)
        br = _br_agent(tables, stack)
        for seat in (0, 1):
            got = ev.evaluate(Composite(br, agent, seat))
            print("stack %d %s chunk %s seat %d: composite %r (agent %r)" % (stack, kind, chunk, seat, got, ref))
            assert got[seat] == 0.0, (stack, kind, chunk, seat, got)


def _oracle_ev_br(ft, agent):
    t = oracle_tree(ft)
    dec = np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]
    pr = agent.probs(ft, dec)
    for d, n in enumerate(dec):
        fc, A = int(ft.first_child[n]), int(ft.n_children[n])
        t.strategy[n] = pr[d][:, ft.action[fc:fc + A]].astype(np.float64)
    t.update_reach()
    t.compute_ev()
    return t.ev_br


def _check_actions(ft, ev_br, answers, what):
    """answers [n_dec, R, n_actions] (one-hot, zero rows for blocked hands) against the float64 ev_br: the same child
    where the top two differ by more than MARGIN of the node's max |ev_br|, elsewhere a child within that margin"""
    dec = np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]
    near = decided = 0
    for d, n in enumerate(dec):
        fc, A, k = int(ft.first_child[n]), int(ft.n_children[n]), int(ft.kind[n])
        v = ev_br[fc:fc + A, k]  # [A, R]
        a = answers[d][:, ft.action[fc:fc + A]].T  # [A, R]
        live = a.sum(axis=0) > 0
        assert np.all(a[:, live].sum(axis=0) == 1.0), (what, n)
        tol = MARGIN * max(np.abs(v).max(), 1e-300)
        srt = np.sort(v, axis=0)
        clear = live & (srt[-1] - srt[-2] > tol) if A > 1 else live
        chosen = np.argmax(a, axis=0)
        assert np.all(chosen[clear] == np.argmax(v, axis=0)[clear]), (what, n)
        vv = v[chosen, np.arange(v.shape[1])]
        assert np.all(vv[live] >= v.max(axis=0)[live] - tol), (what, n)
        near += int((live & ~clear).sum())
        decided += int(clear.sum())
    print("%s: %d (node, hand) pairs decided, %d near-ties" % (what, decided, near))


def _structure(spec, stack):
    pt = PublicTree(_bldr(stack), [stack, stack], None, put_out_new_round_after_limit=True, board_spec=spec)
    pt.build_structure()
    return pt


def test_board_and_level_engine_best_responses_against_the_float64_oracle(monkeypatch):
    from pokerrl_b200.eval.br.LocalBRMaster import LocalBRMaster
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    stack = 20000
    spec = random_board_spec(12, 41)
    ft = fhp_tree(spec, stack)
    agent = _Hash(_bldr(stack).N_ACTIONS)
    ev_br = _oracle_ev_br(ft, agent)
    res = {}
    for engine in ("board", "levels"):
        monkeypatch.setenv("PRL_ENGINE", engine)
        master = LocalBRMaster(t_prof=_t_prof("m" + engine, stack), chief_handle=ChiefBase(None),
                               eval_agent_cls=lambda t_prof: agent, board_spec=spec)
        assert isinstance(master._game_trees[0], PublicTree) == (engine == "levels")
        e0, e1, br = master.best_response_agent(0)
        res[engine] = np.array([e0, e1])
        pt = _structure(spec, stack)
        answers = torch.as_tensor(br.get_a_probs_for_public_tree(pt)).cpu().numpy()
        _check_actions(pt.flat, ev_br, answers, engine)
    rel = np.abs(res["board"] - res["levels"]) / np.abs(res["levels"])
    print("exploitability board %r levels %r, relative %r" % (res["board"], res["levels"], rel))
    assert np.all(rel <= 1e-6)


@pytest.mark.parametrize("name", ["StandardLeduc", "BigLeduc", "NLLeduc_POT"])
def test_one_card_table_equals_argmax_of_the_float32_oracle(name):
    from cfr_numpy import OracleTree
    from pokerrl_b200.cfr.CFRPlus import CFRPlus
    from pokerrl_b200.cfr.TabularCFREvalAgent import TabularCFREvalAgent
    from pokerrl_b200.eval.br.LocalBRMaster import LocalBRMaster
    from pokerrl_b200.game import bet_sets
    from pokerrl_b200.rl.base_cls.TrainingProfileBase import TrainingProfileBase
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    game = {"StandardLeduc": games.StandardLeduc, "BigLeduc": games.BigLeduc, "NLLeduc_POT": games.DiscretizedNLLeduc}[name]
    chief = ChiefBase(None)
    cfr = CFRPlus(name="o" + name, chief_handle=chief, game_cls=game, agent_bet_set=bet_sets.POT_ONLY, delay=0)
    for _ in range(7):
        cfr.iteration()
    t_prof = TrainingProfileBase("o" + name, game, bet_sets.POT_ONLY)
    master = LocalBRMaster(t_prof=t_prof, chief_handle=chief, eval_agent_cls=TabularCFREvalAgent)
    master._eval_agent = TabularCFREvalAgent.from_cfr(t_prof, cfr)
    e0, e1, br = master.best_response_agent(0)
    gt = master._game_trees[0]
    ft = gt.flat
    assert (e0, e1) == master._compute_br_heads_up(0)
    orc = OracleTree(ft)
    tab = master.eval_agent._table
    dec = orc.decision_nodes()
    for n in dec:
        fs, A = int(ft.first_slot[n]), int(ft.n_children[n])
        orc.strategy[n] = np.ascontiguousarray(tab[fs:fs + A].T)
    orc.update_reach()
    orc.compute_ev()
    want = np.zeros_like(br._table)
    for n in dec:
        fs, fc, A, k = int(ft.first_slot[n]), int(ft.first_child[n]), int(ft.n_children[n]), int(ft.kind[n])
        want[fs + np.argmax(orc.ev_br[fc:fc + A, k], axis=0), np.arange(ft.R)] = 1.0
    assert np.array_equal(br._table, want), name
    for seat in (0, 1):
        gt.fill_with_agent_policy(Composite(br, master.eval_agent, seat))
        gt.compute_ev()
        assert float(gt.root.exploitability[seat]) == 0.0, (name, seat, gt.root.exploitability)


def test_state_dict_round_trip_and_another_tree_raises(tmp_path):
    import os
    from pokerrl_b200.cfr.TabularCFREvalAgent import TabularCFREvalAgent
    stack = 20000
    spec = random_board_spec(16, 5)
    _, tables = BoardPolicyEvaluator(_bldr(stack), [stack, stack], spec).best_response(HashAgent(_bldr(stack).N_ACTIONS))
    br = _br_agent(tables, stack)
    pt = _structure(spec, stack)
    want = br.get_a_probs_for_public_tree(pt).cpu()
    again = TabularCFREvalAgent(t_prof=_t_prof("br", stack))
    again.load_state_dict(br.state_dict())
    assert torch.equal(again.get_a_probs_for_public_tree(pt).cpu(), want)
    br.store_to_disk(str(tmp_path), "br")
    disk = TabularCFREvalAgent.load_from_disk(os.path.join(str(tmp_path), "br.pkl"))
    assert torch.equal(disk.get_a_probs_for_public_tree(pt).cpu(), want)
    with pytest.raises(ValueError, match="different betting tree"):
        br.get_a_probs_for_public_tree(_structure(spec, 600))


def test_restricted_nash_response_takes_the_best_response_as_its_model():
    from pokerrl_b200.cfr.RestrictedNashResponse import RestrictedNashResponse
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    stack = 20000
    spec = random_board_spec(16, 8)
    _, tables = BoardPolicyEvaluator(_bldr(stack), [stack, stack], spec).best_response(HashAgent(_bldr(stack).N_ACTIONS))
    rnr = RestrictedNashResponse("rnr_br", ChiefBase(None), G, [1.0], _br_agent(tables, stack), 0.5,
                                 starting_stack_sizes=[stack], board_spec=spec)
    for _ in range(3):
        rnr.iteration()
    assert rnr.counter_agent().rows.shape == tables.rows.shape


def test_full_game_cfrp_agent_composite_is_exactly_unexploitable():
    stack = 20000
    torch.cuda.reset_peak_memory_stats()
    agent = _cfr_agent(None, stack, 10, "fullbr")  # the solver is freed with the CFRPlus object
    gc.collect()
    torch.cuda.empty_cache()
    ev = BoardPolicyEvaluator(_bldr(stack), [stack, stack])
    assert ev.n_boards_total == 134459
    e, tables = ev.best_response(agent)
    br = _br_agent(tables, stack)
    for seat in (0, 1):
        got = ev.evaluate(Composite(br, agent, seat))
        print("full game seat %d: composite %r, agent %r" % (seat, got, e))
        assert got[seat] == 0.0, (seat, got)
    print("peak device memory %.2f GB" % (torch.cuda.max_memory_allocated() / 1e9))
