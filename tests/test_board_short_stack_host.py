"""Short-stack Flop5Holdem on the board engine, CPU only: which post-deal shape each stack has, that the library's second
compiled shape (csrc/cfr_board.cu `ShapeFHPShort`) is that subtree, and that its fold-relation table is the derived one."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

from pokerrl_b200.game import games
from twocard_common import fhp_tree, random_board_spec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
SRC = open(os.path.join(ROOT, "pokerrl_b200", "csrc", "cfr_board.cu")).read()


def _shape_arrays(struct):
    """kind / parent / first_child / n_children of a shape struct of the kernel source"""
    body = SRC[SRC.index("struct %s :" % struct):]
    body = body[:body.index("};")]
    n = int(re.search(r"static constexpr int N = (\d+);", body).group(1))
    out = {}
    for key, name in (("kind", "kKind"), ("parent", "kParent"), ("first_child", "kFirstChild"), ("n_children", "kNChildren")):
        vals = [int(x) for x in re.search(r"%s = pack_nodes\(\{\{([^}]*)\}\}\)" % name, body).group(1).split(",")]
        assert len(vals) == n
        out[key] = vals
    return out


def _subtree(stack):
    return fhp_tree(random_board_spec(1, 0), stack).board_subtree()


def _args(stack):
    g = games.Flop5Holdem
    return g, g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[stack, stack], bet_sizes_list_as_frac_of_pot=[1.0])


def _same_shape(st, arrays):
    return st is not None and all(list(st[k]) == v for k, v in arrays.items())


@pytest.mark.parametrize("stack", [301, 600, 899, 900])
def test_short_stacks_have_the_nine_node_shape(stack):
    from pokerrl_b200.board_engine import supports
    st = _subtree(stack)
    assert _same_shape(st, _shape_arrays("ShapeFHPShort")), st
    # the two calls of the all-in bet have pot 2 x stack, every other node the 600 of the flop
    assert st["pot"] == [600.0] * 6 + [2.0 * stack, 600.0, 2.0 * stack]
    assert supports(*_args(stack), "CFRPlus")


@pytest.mark.parametrize("stack", [901, 1000, 20000])
def test_deep_stacks_have_the_fifteen_node_shape(stack):
    from pokerrl_b200.board_engine import supports
    assert _same_shape(_subtree(stack), _shape_arrays("ShapeFHP"))
    assert supports(*_args(stack), "CFRPlus")


@pytest.mark.parametrize("stack", [250, 300])
def test_push_fold_stacks_have_no_board_subtree(stack):
    from pokerrl_b200.board_engine import supports
    assert _subtree(stack) is None
    assert not supports(*_args(stack), "CFRPlus")


def test_short_fold_relation_table_of_the_kernel_is_the_derived_one():
    import fold_relations as fr
    a = _shape_arrays("ShapeFHPShort")
    m = re.search(r"constexpr int c\[2\]\[2\]\[3\] = (\{\{.*?\}\}\});", SRC, re.S)
    got = np.array(eval(m.group(1).replace("{", "[").replace("}", "]").rstrip(";")))
    for seed, trials in ((0, 40), (5, 60)):
        want = fr.derive(a["kind"], a["first_child"], a["n_children"], trials=trials, seed=seed)
        assert got.shape == (2, 2, 3) and np.array_equal(got, want), (seed, got, want)


def test_library_row_layout_of_each_shape():
    """prl_board_rows / prl_board_layout for the descriptor of each stack's subtree; a subtree that matches no compiled shape
    is refused"""
    from pokerrl_b200 import _native as nat
    from pokerrl_b200.board_engine import _fill_shape, board_layout, shape_rows
    for stack, n_local, rows in ((600, 9, 8), (20000, 15, 14)):
        st = _subtree(stack)
        g = nat.PrlBoardGame()
        _fill_shape(g, st)
        row_of, rpb = shape_rows(g)
        assert rpb == rows and board_layout(g)["n_local"] == n_local
        children = [c for c in range(1, n_local) if st["kind"][st["parent"][c]] <= 1]
        assert sorted(row_of[c] for c in children) == list(range(rows))
        assert all(row_of[c] == -1 for c in range(16) if c not in children)
        # seat 0's rows first (both shapes give each seat half of the rows)
        assert max(row_of[c] for c in children if st["kind"][st["parent"][c]] == 0) < rows // 2
    assert board_layout()["n_local"] == 0
    g = nat.PrlBoardGame()
    _fill_shape(g, _subtree(600))
    g.kind[2] = 1
    assert nat.lib().prl_board_shape_ok(C.byref(g)) == 0
    with pytest.raises(RuntimeError, match="no compiled shape"):
        shape_rows(g)
