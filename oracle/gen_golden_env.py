"""Golden PokerEnv trajectories produced by RUNNING THE REFERENCE ENV (TEST INFRASTRUCTURE; needs a PokerRL checkout in POKERRL_REFERENCE):

    python oracle/gen_golden_env.py [game ...]   # writes tests/golden/env_<game>.npz (default: every game)

For each game: E episodes of uniformly random legal play in evaluation mode (PokerEnv.py:1075-1159,
DiscretizedPokerEnv.py:47-135, LimitPokerEnv.py:27-59).  Recorded per episode: the shuffled deck (1D card ids, top
first), and per step the legal-action mask before the step, the action, and the returned (obs float32, rewards float64,
done).  The batched CUDA env must reproduce obs / rewards / done / legal masks exactly when fed the same decks and actions
(RNG streams cannot match numpy's MT19937 - SURVEY.md §8d config 5)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ref_harness as rh  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

GAMES = {
    "DiscretizedNLHoldem_B5": ("DiscretizedNLHoldem", "B_5", 20000, 400),
    "DiscretizedNLHoldem_B5_short": ("DiscretizedNLHoldem", "B_5", 700, 300),  # shallow stacks: all-ins, capped raises
    "DiscretizedNLLeduc_B3": ("DiscretizedNLLeduc", "B_3", 20000, 200),
    "StandardLeduc": ("StandardLeduc", "POT_ONLY", 13, 200),
    "LimitHoldem": ("LimitHoldem", "POT_ONLY", 48, 300),
    "Flop5Holdem": ("Flop5Holdem", "POT_ONLY", 20000, 200),
    "BigLeduc": ("BigLeduc", "POT_ONLY", 100, 200),  # pair bonus 10000: runs with ref_harness's hand-rank fix
}
T_MAX = 48


def run(name):
    rh.import_reference()
    from PokerRL.game import bet_sets, games
    cls_name, bs, stack, E = GAMES[name]
    g = getattr(games, cls_name)
    args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[stack, stack],
                      bet_sizes_list_as_frac_of_pot=list(getattr(bet_sets, bs)))
    lut = g.get_lut_holder()
    env = g(env_args=args, lut_holder=lut, is_evaluating=True)
    n_act, n_deck = env.N_ACTIONS, env.N_CARDS_IN_DECK
    obs_size = env.observation_space.shape[0]
    np.random.seed(2026)
    deck = np.zeros((E, n_deck), np.int8)
    obs0 = np.zeros((E, obs_size), np.float32)
    legal = np.zeros((E, T_MAX, n_act), np.uint8)
    action = np.full((E, T_MAX), -1, np.int8)
    obs = np.zeros((E, T_MAX, obs_size), np.float32)
    rew = np.zeros((E, T_MAX, 2), np.float64)
    done = np.zeros((E, T_MAX), np.uint8)
    n_steps = np.zeros(E, np.int32)
    for e in range(E):
        o, _, _, _ = env.reset()
        # the deck as it was right after the shuffle: hole cards were drawn from the top (seat 0 first)
        drawn = [lut.get_1d_cards(env.seats[p].hand) for p in range(2)]
        rest = lut.get_1d_cards(env.deck.deck_remaining)
        deck[e] = np.concatenate(drawn + [rest])
        obs0[e] = o
        t = 0
        while True:
            la = env.get_legal_actions()
            legal[e, t, la] = 1
            a = la[np.random.randint(len(la))]
            action[e, t] = a
            o, r, d, _ = env.step(a)
            obs[e, t], rew[e, t], done[e, t] = o, np.asarray(r, np.float64), d
            t += 1
            if d:
                break
            assert t < T_MAX
        n_steps[e] = t
    np.savez_compressed(os.path.join(OUT, "env_%s.npz" % name), deck=deck, obs0=obs0, legal=legal, action=action,
                        obs=obs, rew=rew, done=done, n_steps=n_steps, stack=np.array(stack),
                        n_actions=np.array(n_act), game=np.array(cls_name), bet_set=np.array(bs))
    return name, E, float(n_steps.mean()), int(n_steps.max())


if __name__ == "__main__":
    for n in sys.argv[1:] or GAMES:
        print(run(n))
