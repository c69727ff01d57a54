"""Golden traces of the REFERENCE's PokerRange (PokerRL/game/PokerRange.py:9-160) under a scripted sequence of the operations
the LBR evaluator performs (TEST INFRASTRUCTURE; needs a PokerRL checkout in POKERRL_REFERENCE):

    python oracle/gen_golden_poker_range.py      # writes tests/golden/poker_range.npz

ops: 0 reset | 1 set_cards_to_zero_prob(cards) | 2 mul_and_norm(vector seed) | 3 update_after_action(action, probs seed) |
4 update_after_new_round(round, board).  After every op the float32 range is recorded."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ref_harness as rh  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def script(rng):
    """[(op, a, b, cards[5])]: two hands' worth of operations incl. a range driven to zero (falls back to uniform)"""
    ops = []
    for hand in range(3):
        deck = rng.permutation(52).astype(np.int8)
        ops.append((0, 0, 0, np.full(5, -127, np.int8)))
        ops.append((1, 0, 0, np.concatenate([deck[:2], np.full(3, -127, np.int8)])))
        for step in range(3):
            ops.append((3, int(rng.integers(0, 3)), int(rng.integers(1, 1 << 30)), np.full(5, -127, np.int8)))
        board = deck[2:7].copy()
        ops.append((4, 1, 0, board))  # flop dealt
        ops.append((2, 0, int(rng.integers(1, 1 << 30)), np.full(5, -127, np.int8)))
        ops.append((3, 1, int(rng.integers(1, 1 << 30)), np.full(5, -127, np.int8)))
        ops.append((4, 2, 0, board))  # turn
        ops.append((4, 3, 0, board))  # river
        if hand == 1:
            ops.append((2, 1, 0, np.full(5, -127, np.int8)))  # multiply by zeros: sum 0 -> uniform again
    return ops


def vector(seed, n, cols=None):
    r = np.random.default_rng(seed)
    return (r.random(n if cols is None else (n, cols)) ** 2).astype(np.float32)


if __name__ == "__main__":
    rh.import_reference()
    from PokerRL.game.PokerRange import PokerRange
    from PokerRL.game.games import DiscretizedNLHoldem
    from PokerRL.game import bet_sets
    from PokerRL.game.wrappers import VanillaEnvBuilder
    args = DiscretizedNLHoldem.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[20000, 20000], bet_sizes_list_as_frac_of_pot=bet_sets.B_2)
    bldr = VanillaEnvBuilder(env_cls=DiscretizedNLHoldem, env_args=args)
    lut = bldr.lut_holder
    ops = script(np.random.default_rng(5))
    r = PokerRange(env_bldr=bldr)
    trace = []
    for op, a, b, cards in ops:
        if op == 0:
            r.reset()
        elif op == 1:
            r.set_cards_to_zero_prob(cards_2d=lut.get_2d_cards(cards[cards >= 0]))
        elif op == 2:
            r.mul_and_norm(np.zeros(1326, np.float32) if a == 1 else vector(b, 1326))
        elif op == 3:
            r.update_after_action(action=a, all_a_probs_for_all_hands=vector(b, 1326, 3))
        else:
            n_out = {1: 3, 2: 4, 3: 5}[a]
            bd = np.full(5, -127, np.int8)
            bd[:n_out] = cards[:n_out]
            r.update_after_new_round(new_round=a, board_now_2d=lut.get_2d_cards(bd))
        trace.append(np.copy(r.range))
    np.savez_compressed(os.path.join(OUT, "poker_range.npz"), op=np.array([o[0] for o in ops], np.int32),
                        a=np.array([o[1] for o in ops], np.int64), b=np.array([o[2] for o in ops], np.int64),
                        cards=np.array([o[3] for o in ops], np.int8), ranges=np.array(trace, np.float32))
    print("wrote poker_range.npz:", len(ops), "operations")
