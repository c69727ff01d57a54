"""The +-1 table `FoldLinFHP` compiled into the board sweep kernel (csrc/cfr_board.cu) equals the derivation of
tools/fold_relations.py, and the shape arrays the derivation uses are the kernel's `ShapeFHP`.  CPU only."""
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def _c_array(src, name):
    m = re.search(r"%s = pack_nodes\(\{\{([^}]*)\}\}\)" % name, src)
    return [int(x) for x in m.group(1).split(",")]


def test_fold_relation_table_of_the_kernel_is_the_derived_one():
    import fold_relations as fr
    src = open(os.path.join(ROOT, "pokerrl_b200", "csrc", "cfr_board.cu")).read()
    assert _c_array(src, "kKind") == fr.KIND and _c_array(src, "kFirstChild") == fr.FIRST and _c_array(src, "kNChildren") == fr.NCH
    m = re.search(r"constexpr int c\[2\]\[4\]\[5\] = (\{\{.*?\}\}\});", src, re.S)
    got = np.array(eval(m.group(1).replace("{", "[").replace("}", "]").rstrip(";")))
    want = fr.derive()
    assert got.shape == (2, 4, 5) and np.array_equal(got, want), (got, want)
    # each fold vector's combination reproduces the vector for fresh random strategies of BOTH seats (the sweep's own seat
    # copies the reach, so its strategy must not matter)
    assert np.array_equal(fr.derive(seed=5, trials=60), want)
