"""Reference harness (TEST INFRASTRUCTURE ONLY — never imported by the product path).

Imports a checkout of the PokerRL reference (directory given by POKERRL_REFERENCE; only the fixture generators need it,
never the tests) with the two stub packages under oracle/ref_stubs, and
provides helpers that flatten the reference's object tree (PokerRL/game/_/tree/nodes.py:8-62)
into DFS-pre-order arrays so that golden fixtures can be committed under tests/golden/.

DFS pre-order = the order of `PublicTree._build_tree` (PublicTree.py:161-166): a node, then
each of its children in `node.children` order, recursively.
"""
import os
import sys

import numpy as np

REFERENCE_ROOT = os.environ.get("POKERRL_REFERENCE", "")
_STUBS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_stubs")


def reference_available():
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "PokerRL"))


def import_reference():
    """Put the reference and the gym/pycrayon stubs on sys.path. Returns the PokerRL module."""
    if not reference_available():
        raise RuntimeError("PokerRL reference not found at %r: set POKERRL_REFERENCE to a PokerRL checkout" % REFERENCE_ROOT)
    for p in (_STUBS, REFERENCE_ROOT):
        if p not in sys.path:
            sys.path.insert(0, p)
    import PokerRL  # noqa
    _patch_big_leduc_hand_rank()
    return PokerRL


def _patch_big_leduc_hand_rank():
    """The ONLY deviation from the reference's code: BigLeducRules.get_hand_rank (game_rules.py:133-140) computes
    `10000 + hand_2d[0, 0]` on an int8 scalar, which raises OverflowError under NumPy 2 (NEP 50).  NumPy < 2 promoted
    it to int16 and returned 10000 + rank; this evaluates the same expression on a Python int, which is that value."""
    from PokerRL.game._.rl_env.game_rules import BigLeducRules

    if getattr(BigLeducRules.get_hand_rank, "_python_int_pair_bonus", False):
        return

    def get_hand_rank(self, hand_2d, board_2d):
        if board_2d[0, 0] == hand_2d[0, 0]:
            return 10000 + int(hand_2d[0, 0])
        else:
            return hand_2d[0, 0]

    get_hand_rank._python_int_pair_bonus = True
    BigLeducRules.get_hand_rank = get_hand_rank


# node kind codes shared with pokerrl_b200.game.flat_tree
KIND_P0, KIND_P1, KIND_CHANCE, KIND_FOLD, KIND_SHOWDOWN, KIND_SHOWDOWN_ALLIN = 0, 1, 2, 3, 4, 5


def dfs_nodes(tree):
    out = []

    def rec(n):
        out.append(n)
        for c in n.children:
            rec(c)

    rec(tree.root)
    return out


def flatten_structure(tree):
    """Structure arrays of a reference PublicTree in DFS pre-order."""
    from PokerRL.game.Poker import Poker
    from PokerRL.game.PokerEnvStateDictEnums import EnvDictIdxs, PlayerDictIdxs

    nodes = dfs_nodes(tree)
    idx = {id(n): i for i, n in enumerate(nodes)}
    N = len(nodes)
    lut = tree.env_bldr.lut_holder
    n_board = tree.env_bldr.rules.N_TOTAL_BOARD_CARDS
    last_round = tree.env_bldr.rules.ALL_ROUNDS_LIST[-1]
    s = dict(
        parent=np.full(N, -1, np.int32), depth=np.zeros(N, np.int32), kind=np.zeros(N, np.int8),
        action=np.full(N, -1, np.int32), main_pot=np.zeros(N, np.int64), round=np.zeros(N, np.int8),
        board=np.full((N, n_board), -127, np.int8), n_children=np.zeros(N, np.int32),
        acted_last=np.full(N, -2, np.int8), stack=np.zeros((N, 2), np.int64), bet=np.zeros((N, 2), np.int64),
    )
    for i, n in enumerate(nodes):
        st = n.env_state
        s["parent"][i] = -1 if n.parent is None else idx[id(n.parent)]
        s["depth"][i] = n.depth
        s["main_pot"][i] = st[EnvDictIdxs.main_pot]
        s["round"][i] = st[EnvDictIdxs.current_round]
        s["board"][i] = lut.get_1d_cards(st[EnvDictIdxs.board_2d])
        s["n_children"][i] = len(n.children)
        for p in range(2):
            s["stack"][i, p] = st[EnvDictIdxs.seats][p][PlayerDictIdxs.stack]
            s["bet"][i, p] = st[EnvDictIdxs.seats][p][PlayerDictIdxs.current_bet]
        if n.p_id_acted_last == tree.CHANCE_ID:
            s["acted_last"][i] = -1
            # child of a chance node: "action" = index of this node among its siblings (1D card for Leduc)
            s["action"][i] = n.parent.children.index(n)
        elif n.p_id_acted_last is not None:
            s["acted_last"][i] = n.p_id_acted_last
            s["action"][i] = n.action
        if n.is_terminal:
            if n.action == Poker.FOLD:
                s["kind"][i] = KIND_FOLD
            elif st[EnvDictIdxs.current_round] == last_round:
                s["kind"][i] = KIND_SHOWDOWN
            else:
                s["kind"][i] = KIND_SHOWDOWN_ALLIN
        elif n.p_id_acting_next == tree.CHANCE_ID:
            s["kind"][i] = KIND_CHANCE
        else:
            s["kind"][i] = KIND_P0 if n.p_id_acting_next == 0 else KIND_P1
    return s


def flatten_values(tree, R):
    """reach / ev / ev_br [N,2,R] float32 and per-child strategy column [N,R] float64 (NaN where the
    parent is not a decision node), DFS pre-order."""
    nodes = dfs_nodes(tree)
    N = len(nodes)
    reach = np.zeros((N, 2, R), np.float32)
    ev = np.zeros((N, 2, R), np.float32)
    ev_br = np.zeros((N, 2, R), np.float32)
    strat = np.full((N, R), np.nan, np.float64)
    for i, n in enumerate(nodes):
        assert n.reach_probs.dtype == np.float32 and n.ev.dtype == np.float32 and n.ev_br.dtype == np.float32
        reach[i], ev[i], ev_br[i] = n.reach_probs, n.ev, n.ev_br
        if n.parent is not None and n.parent.p_id_acting_next in (0, 1):
            k = n.parent.children.index(n)
            strat[i] = n.parent.strategy[:, k]
    return dict(reach=reach, ev=ev, ev_br=ev_br, strat=strat)


def flatten_node_table(tree, key, R, dtype=np.float64):
    """A per-decision-node table stored in node.data[key] ([R,A]) → [N,R] indexed by child node."""
    nodes = dfs_nodes(tree)
    out = np.full((len(nodes), R), np.nan, dtype)
    for i, n in enumerate(nodes):
        if n.parent is not None and n.parent.p_id_acting_next in (0, 1):
            d = n.parent.data
            if d is not None and d.get(key) is not None:
                out[i] = d[key][:, n.parent.children.index(n)]
    return out
