"""Shared helpers for the parity tests."""
import os

import numpy as np

from pokerrl_b200.game import bet_sets, games
from pokerrl_b200.game.flat_tree import FlatTree

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# fixture name -> (game class name, bet set name); mirrors oracle/gen_golden_cfr.py:GAMES
GAMES = {
    "StandardLeduc": ("StandardLeduc", "POT_ONLY"),
    "NLLeduc_POT": ("DiscretizedNLLeduc", "POT_ONLY"),
    "NLLeduc_B2": ("DiscretizedNLLeduc", "B_2"),
    "NLLeduc_B3": ("DiscretizedNLLeduc", "B_3"),
    "BigLeduc": ("BigLeduc", "POT_ONLY"),
}


def make_flat_tree(name):
    cn, bs = GAMES[name]
    g = getattr(games, cn)
    args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[g.DEFAULT_STACK_SIZE] * 2,
                      bet_sizes_list_as_frac_of_pot=getattr(bet_sets, bs))
    return FlatTree(g, args)


def golden(fname):
    return np.load(os.path.join(GOLDEN, fname), allow_pickle=False)


def formula_profile_table(ft):
    """oracle/fixture_digest.formula_strategy of every decision node (the second value profile of the BigLeduc
    fixtures) as a float64 [n_slots, R] strategy table: row slot[c] = probability of moving to child c, per hand."""
    from fixture_digest import formula_strategy
    tab = np.zeros((ft.n_slots, ft.R))
    for n in np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]:
        A, fs = int(ft.n_children[n]), int(ft.first_slot[n])
        tab[fs:fs + A] = formula_strategy(int(ft.dfs[n]), A, ft.R).T
    return tab
