"""Host-side structure of the two-card trees (no GPU): Flop5Holdem betting structure of SURVEY.md §8 and the
suit-isomorphism board classes."""
import numpy as np

from pokerrl_b200.game import games, holdem_boards as hb
from pokerrl_b200.game.flat_tree import enumerate_betting_tree
from pokerrl_b200.game.hu_engine import HUBetting
from twocard_common import fhp_tree, hulh_flop_subgame, nl_flop_subgame, random_board_spec


def test_flop5holdem_betting_structure():
    g = games.Flop5Holdem
    args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[20000, 20000], bet_sizes_list_as_frac_of_pot=[1.0])
    A = enumerate_betting_tree(HUBetting(g, args))
    post = [n for n in A if n.cdepth == 1]
    dec = [n for n in post if n.kind <= 1]
    assert len(dec) == 6 and sum(len(n.children) for n in dec) == 14          # SURVEY.md §8 header
    assert sum(n.kind == 4 for n in post) == 5 and sum(n.kind == 3 for n in post) == 4
    assert [len(n.children) for n in A if n.cdepth == 0 and n.kind <= 1] == [2, 2]  # SB {fold, raise}, BB {fold, call}


def test_limit_holdem_betting_structure():
    g = games.LimitHoldem
    args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[48, 48], bet_sizes_list_as_frac_of_pot=[1.0])
    A = enumerate_betting_tree(HUBetting(g, args))
    assert sum(n.kind == 3 for n in A) == 5103 and sum(n.kind == 4 for n in A) == 5103  # 10 206 terminal sequences
    assert sum(n.kind <= 1 and n.children != [] for n in A) == 6378


def test_suit_isomorphism_classes_small_deck():
    deck = [0, 1, 2, 3, 4, 5, 6, 7, 48, 49, 50, 51]  # ranks 2, 3, A in all four suits: closed under suit permutations
    boards = hb.all_boards(deck, 5)
    reps, orbit = hb.canonical_boards(boards)
    assert orbit.sum() == len(boards) == 792
    perms = hb.suit_permutation_hand_tables()
    assert perms.shape == (24, 1326) and np.array_equal(np.sort(perms, axis=1), np.tile(np.arange(1326), (24, 1)))
    # every board is a suit permutation of exactly one representative
    keys = {tuple(r) for r in reps.tolist()}
    assert len(keys) == len(reps)


def test_flat_tree_layout_two_card():
    ft = fhp_tree(random_board_spec(20, 0))
    nb = ft.board_spec.boards.shape[0]
    assert ft.n_nodes == 5 + 15 * nb and ft.n_slots == 4 + 14 * nb
    ch = np.nonzero(ft.kind == 2)[0]
    assert len(ch) == 1 and ft.n_children[ch[0]] == nb
    kids = np.arange(ft.first_child[ch[0]], ft.first_child[ch[0]] + nb)
    assert np.array_equal(ft.board[kids], 1 + np.arange(nb))  # global board ids, 0 = the empty board


def test_structure_records_restate_the_pointer_chains():
    """prl_tree_t.node_rec2 / work_rec2 (pokerrl_b200/solver.py:structure_records) hold exactly what the v1 kernels read
    through parent -> first_child -> slot chains"""
    from pokerrl_b200.solver import structure_records
    from twocard_common import fhp_tree, random_board_spec
    ft = fhp_tree(random_board_spec(5, 3))
    order, _ = ft.work_order()
    nrec, wrec = structure_records(ft, order)
    for n in range(ft.n_nodes):
        p = int(ft.parent[n])
        assert nrec[n, 0] == p and nrec[n, 1] == ft.slot[n]
        if p >= 0:
            assert nrec[n, 2] == ft.slot[ft.first_child[p]]
            assert nrec[n, 3] & 0xff == ft.kind[p] and nrec[n, 3] >> 8 == ft.n_children[p]
    for t in range(ft.n_nodes):
        n = int(order[t])
        assert wrec[t, 0] == n and wrec[t, 3] & 0xff == ft.kind[n]
        if ft.n_children[n] > 0:
            assert wrec[t, 3] >> 8 == ft.n_children[n]
            assert wrec[t, 1] == ft.first_child[n] and wrec[t, 2] == ft.slot[ft.first_child[n]]
        else:  # terminal entries carry what terminal2_kernel_v3 needs
            assert wrec[t, 1] == ft.board[n] and wrec[t, 3] >> 8 == (int(ft.acted_last[n]) & 0xff)
            assert wrec[t, 2:3].view(np.float32)[0] == np.float32(ft.pot[n])


def test_work_order_puts_fold_rows_first_among_terminals():
    """The value sweep launches fold2_kernel over the first level_nfold terminal entries of a level and
    terminal2_kernel_v3 over the showdown entries after them, so v3 never meets a fold row: per level the work list must
    be non-terminals, then every fold terminal, then showdowns, then all-in showdowns"""
    from pokerrl_b200 import _native as nat
    trees = [fhp_tree(random_board_spec(5, 3)), hulh_flop_subgame([[20, 21, 22], [30, 31]]), nl_flop_subgame()]
    assert (trees[2].kind == nat.KIND_SHOWDOWN_ALLIN).any()
    for ft in trees:
        order, level_nonterm = ft.work_order()
        for d in range(ft.n_levels):
            lo, hi = int(ft.level_start[d]), int(ft.level_start[d + 1])
            kinds = ft.kind[order[lo:hi]]
            n_fold = int((ft.kind[lo:hi] == nat.KIND_FOLD).sum())  # DeviceTree's level_nfold[d]
            n_show = int((kinds == nat.KIND_SHOWDOWN).sum())
            n_allin = int((kinds == nat.KIND_SHOWDOWN_ALLIN).sum())
            nt = int(level_nonterm[d])
            assert nt + n_fold + n_show + n_allin == hi - lo
            assert (kinds[:nt] <= nat.KIND_CHANCE).all()
            assert (kinds[nt:nt + n_fold] == nat.KIND_FOLD).all()
            assert (kinds[nt + n_fold:nt + n_fold + n_show] == nat.KIND_SHOWDOWN).all()
            assert (kinds[nt + n_fold + n_show:] == nat.KIND_SHOWDOWN_ALLIN).all()
