"""Golden check-down equities for the LBR roll-out kernel, produced by RUNNING THE REFERENCE's _LBRRolloutManager
(PokerRL/eval/lbr/LocalLBRWorker.py:377-512) on Hold'em states (TEST INFRASTRUCTURE; needs a PokerRL checkout in POKERRL_REFERENCE):

    python oracle/gen_golden_lbr.py      # writes tests/golden/lbr_rollouts.npz

Each query = (LBR hand, dealt board cards, agent range with the LBR / board cards removed); flop, turn and river states,
dense and sparse ranges.  The reference walks every completion of the board through its native hand evaluator."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ref_harness as rh  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

if __name__ == "__main__":
    rh.import_reference()
    from PokerRL.eval.lbr.LocalLBRWorker import _LBRRolloutManager
    from PokerRL.game import bet_sets
    from PokerRL.game.PokerRange import PokerRange
    from PokerRL.game.games import DiscretizedNLHoldem
    from PokerRL.game.wrappers import VanillaEnvBuilder

    class TProf:
        DEBUGGING = False

    args = DiscretizedNLHoldem.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[20000, 20000],
                                        bet_sizes_list_as_frac_of_pot=bet_sets.B_2)
    bldr = VanillaEnvBuilder(env_cls=DiscretizedNLHoldem, env_args=args)
    env = bldr.get_new_env(is_evaluating=True)
    lut = bldr.lut_holder
    rng = np.random.default_rng(77)
    hands, boards, n_dealt, ranges, equity = [], [], [], [], []
    for k, n_q in ((3, 3), (4, 5), (5, 5)):
        for qi in range(n_q):
            cards = rng.choice(52, k + 2, replace=False).astype(np.int8)
            lbr_1d, board_1d = np.sort(cards[:2]), cards[2:]
            env.reset()
            b = np.full(5, -127, np.int8)
            b[:k] = board_1d
            env.board = lut.get_2d_cards(b)
            env.current_round = {3: 1, 4: 2, 5: 3}[k]
            lbr_2d = lut.get_2d_cards(lbr_1d)
            r = PokerRange(env_bldr=bldr)
            raw = rng.random(1326).astype(np.float32) ** (1 + qi)
            if qi % 2 == 1:
                raw[rng.random(1326) < 0.7] = 0.0
            r._range = raw / raw.sum()
            r.set_cards_to_zero_prob(cards_2d=lbr_2d)
            r.set_cards_to_zero_prob(cards_2d=lut.get_2d_cards(board_1d))
            rng_before = np.copy(r.range)
            mgr = _LBRRolloutManager(t_prof=TProf(), env_bldr=bldr, env=env, lbr_hand_2d=lbr_2d)
            eq = float(mgr.get_lbr_checkdown_equity(agent_range=r))
            assert np.array_equal(rng_before, r.range)
            hands.append(lbr_1d)
            boards.append(b)
            n_dealt.append(k)
            ranges.append(rng_before.astype(np.float32))
            equity.append(eq)
            print("dealt", k, "query", qi, "equity", eq)
    np.savez_compressed(os.path.join(OUT, "lbr_rollouts.npz"), hands=np.array(hands, np.int8), boards=np.array(boards, np.int8),
                        n_dealt=np.array(n_dealt, np.int32), ranges=np.array(ranges, np.float32), equity=np.array(equity, np.float64))
    print("wrote lbr_rollouts.npz")
