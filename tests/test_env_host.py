"""Host betting machine (pokerrl_b200/game/hu_engine.py - the transition function shared by the tree compiler and the CUDA
env) replayed against trajectories of the reference env (tests/golden/env_*.npz): legal-action sets, episode lengths and
final chip movements must agree step by step (no GPU)."""
import numpy as np
import pytest

from common import golden
from pokerrl_b200.game import bet_sets, games
from pokerrl_b200.game import hu_engine as eng

GAMES = ["DiscretizedNLHoldem_B5", "DiscretizedNLHoldem_B5_short", "DiscretizedNLLeduc_B3", "StandardLeduc", "LimitHoldem",
         "Flop5Holdem", "BigLeduc"]


@pytest.mark.parametrize("name", GAMES)
def test_host_engine_replays_reference_env(name):
    g = golden("env_%s.npz" % name)
    game = getattr(games, str(g["game"]))
    stack = int(g["stack"])
    args = game.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[stack, stack],
                         bet_sizes_list_as_frac_of_pot=list(getattr(bet_sets, str(g["bet_set"]))))
    bet = eng.HUBetting(game, args)
    norm = float(stack)  # observation normaliser = mean starting stack (PokerEnv.py:1267)
    for e in range(min(150, g["deck"].shape[0])):
        s = bet.reset()
        for t in range(int(g["n_steps"][e])):
            legal = np.zeros(int(g["n_actions"]), np.uint8)
            legal[bet.legal_actions(s)] = 1
            assert np.array_equal(legal, g["legal"][e, t]), (e, t)
            out, _ = bet.step(s, int(g["action"][e, t]))
            done = out not in (eng.CONTINUE, eng.NEXT_ROUND)
            assert done == bool(g["done"][e, t]), (e, t)
            if not done:
                o = g["obs"][e, t]
                # table-state scalars of the observation: main pot and biggest bet (PokerEnv.py:1004-1031)
                assert o[4] == np.float32(s.main_pot / norm) and o[5] == np.float32(max(s.bet) / norm), (e, t)
                k = 7 + 3 + 2
                assert o[k + s.cur] == 1.0  # next actor one-hot
