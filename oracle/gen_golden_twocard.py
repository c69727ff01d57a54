"""Golden terminal rows for TWO-HOLE-CARD games, anchored on the reference's own hand evaluator
(TEST INFRASTRUCTURE; needs a PokerRL checkout in POKERRL_REFERENCE):

    python oracle/gen_golden_twocard.py      # writes tests/golden/twocard_rows.npz

The reference cannot evaluate a Hold'em public tree (ValueFiller.py:18-19, PublicTree.py:193-203), so no reference
`node.ev` exists for these games.  What the reference DOES provide is (a) the hand strengths - its native
`lib_hand_eval.so` through CppHandeval.get_hand_rank_all_hands_on_given_boards_52_holdem (CppHandeval.py:45-65) - and
(b) the terminal-value statements for one-card games (ValueFiller.py:103-158).  This script evaluates those statements
literally, by brute force over all hand pairs in float64, generalised as SURVEY.md appendix A says:

  showdown (ValueFiller.py:127-158):  eq[h] = K * sum over opponent hands h' that share no card with h and hold no
           board card of  sign(rank[h] - rank[h']) * reach_opp[h'],  eq[h] = 0 if h holds a board card
           ("h_opp != h and h_opp != c" becomes "h' disjoint from h and from the board"; ties add 0)
  fold     (ValueFiller.py:103-125):  eq[h] = K * sum over opponent hands h' disjoint from h of reach_opp[h'],
           0 if h holds a board card; the sign flip for the folder (:112, :124) is applied by the consumer
  K = C(52,2) / C(50,2)  (eq_const N/(N-1) of ValueFiller.py:19 for two-card hands)

for 200 boards (random + quads / full houses / trips / two pairs / one-suit / straights on board: tie-heavy) and seeded
opponent reach rows.  The fixture pins BOTH oracle/cfr2_numpy.py's vectorised formulas and the CUDA terminal kernels
(tests/test_oracle_twocard_rows.py, tests/test_gpu_twocard.py) at R = 1326 with ranks that come from the reference
binary itself.  Reach rows are regenerated in the tests from the stored seed (numpy Generator streams are stable); their
float64 sums are stored as a guard.
"""
import os
import sys
from math import comb

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ref_harness as rh  # noqa: E402
from gen_golden_holdem import targeted_boards  # noqa: E402
from gen_golden_twocard_common import make_reach  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
SEED = 20260924
R = 1326


if __name__ == "__main__":
    rh.import_reference()
    from PokerRL.game._.cpp_wrappers.CppHandeval import CppHandeval
    from PokerRL.game.games import DiscretizedNLHoldem
    lut = DiscretizedNLHoldem.get_lut_holder()
    hc = np.asarray(lut.LUT_IDX_2_HOLE_CARDS).astype(np.int64)  # [R, 2]
    rng = np.random.default_rng(SEED)
    rand = np.stack([np.sort(rng.choice(52, 5, replace=False)) for _ in range(120)]).astype(np.int8)
    targ = targeted_boards(rng)
    targ = targ[rng.choice(len(targ), 80, replace=False)]
    boards = np.concatenate([rand, np.sort(targ, axis=1)]).astype(np.int8)
    ranks = CppHandeval().get_hand_rank_all_hands_on_given_boards_52_holdem(boards_1d=boards, lut_holder=lut)
    ranks = np.asarray(ranks, np.int32)
    reach = make_reach(SEED + 1, boards, hc)
    inc = np.zeros((R, 52), bool)
    inc[np.arange(R), hc[:, 0]] = True
    inc[np.arange(R), hc[:, 1]] = True
    disjoint = ~((inc.astype(np.int8) @ inc.astype(np.int8).T) > 0)  # [R, R]: h and h' share no card
    K = comb(52, 2) / comb(50, 2)
    showdown = np.zeros((len(boards), R))
    fold = np.zeros((len(boards), R))
    n_ties = 0
    for b in range(len(boards)):
        live = ranks[b] >= 0
        assert np.array_equal(live, ~np.isin(hc, boards[b]).any(axis=1))
        rk = ranks[b].astype(np.int64)
        ro = reach[b].astype(np.float64)
        ok = disjoint & live[:, None] & live[None, :]
        sgn = np.sign(rk[:, None] - rk[None, :]) * ok
        n_ties += int(((rk[:, None] == rk[None, :]) & ok).sum())
        showdown[b] = K * (sgn @ ro)
        fold[b] = K * ((disjoint & live[:, None]) @ ro)
    print("boards", len(boards), "tied compatible hand pairs", n_ties, "max |showdown|", np.abs(showdown).max())
    np.savez_compressed(os.path.join(OUT, "twocard_rows.npz"), boards=boards, ranks=ranks, seed=np.array(SEED + 1),
                        reach_sum=reach.astype(np.float64).sum(axis=1), showdown=showdown, fold=fold,
                        eq_const=np.array(K))
    print("wrote twocard_rows.npz")
