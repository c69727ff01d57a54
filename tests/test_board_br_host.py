"""Host side of the board engine's policy evaluation and board-table agent (no GPU): the canonicalisation rule of
prl_board_policy_query restated in numpy, and the map from a chunk tree's slots to the strength-ordered rows."""
import os
from math import comb

import numpy as np

from pokerrl_b200.game.holdem_boards import _combos_52_5, canonical_keys, permutations
from twocard_common import fhp_tree, random_board_spec

DATA = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pokerrl_b200", "game", "data",
                    "flop5_iso_classes.npz")


def test_canonical_keys_reproduce_the_flop5_classes():
    """over all C(52, 5) boards: the distinct canonical keys are the 134 459 representatives, their counts the orbit sizes,
    and the chosen (first minimal) permutation maps each board onto its representative"""
    from pokerrl_b200.board_engine import board_keys
    z = np.load(DATA)
    reps, orbit = z["boards"], z["orbit"].astype(np.int64)
    boards = _combos_52_5()
    assert boards.shape[0] == comb(52, 5)
    perms = np.array(list(permutations(range(4))), np.int64)
    keys = np.empty(boards.shape[0], np.int64)
    for lo in range(0, boards.shape[0], 1 << 19):
        b = boards[lo:lo + (1 << 19)].astype(np.int64)
        k, s = canonical_keys(b)
        keys[lo:lo + b.shape[0]] = k
        mapped = (b // 4) * 4 + perms[s][np.arange(b.shape[0])[:, None], b % 4]
        assert np.array_equal(board_keys(mapped), k)
        if lo == 0:  # the tie rule: no earlier permutation reaches the same key
            for q in range(24):
                kq = board_keys((b // 4) * 4 + perms[q][b % 4])
                assert not np.any((q < s) & (kq == k))
    uniq, counts = np.unique(keys, return_counts=True)
    assert np.array_equal(uniq, board_keys(reps))
    assert np.array_equal(counts, orbit)


def test_row_map_agrees_with_the_board_subtree():
    """every post-deal slot of a chunk tree maps to row j * rows_per_board + row_of(local node) of its board j"""
    from pokerrl_b200.board_engine import board_game, row_map
    ft = fhp_tree(random_board_spec(23, 5))
    st = ft.board_subtree()
    _, rpb, local_rows = board_game(st, ft.rules, 23, 1328, 0, grid=1)
    src, dst = row_map(local_rows, ft)
    got = {}
    for k in range(len(src) // 2):
        for j in range(23):
            got[dst[2 * k] + j * dst[2 * k + 1]] = src[2 * k] + j * src[2 * k + 1]
    A = ft.abs_nodes
    local = sorted([i for i, n in enumerate(A) if n.cdepth == 1], key=lambda i: (A[i].depth, i))
    want = {}
    for n in np.nonzero((ft.slot >= 0) & (ft.cdepth == 1))[0]:
        j = int(ft.board[n]) - 1
        want[int(ft.slot[n])] = j * rpb + local_rows[local.index(int(ft.abs_id[n]))][0]
    assert got == want and len(want) == 23 * rpb
