"""Golden LBR EPISODES, produced by RUNNING THE REFERENCE's LocalLBRWorker (PokerRL/eval/lbr/LocalLBRWorker.py:12-308) against a
deterministic hand-dependent policy (TEST INFRASTRUCTURE; needs a PokerRL checkout in POKERRL_REFERENCE):

    python oracle/gen_golden_lbr_run.py      # writes tests/golden/lbr_runs.npz

Two games: Flop5Holdem (fixed limit, `_run_limit`) and DiscretizedNLHoldem with bet_sets.B_2 (`_run_no_limit`, LBR allowed
the agent's bet sizes), both with `lbr_check_to_round = FLOP` (LBR check / calls before the flop: a roll-out over all
C(48,5) boards per decision is out of reach for the reference).  Recorded per hand: the deal (hole cards + the rest of the
deck in drawing order), the uniform random numbers the agent's action sampling consumed, LBR's winnings; per LBR decision
the utility vector it maximised.  The agent's policy is a fixed function of (hand index, legal actions, street) so that
ranges, fold probabilities and roll-outs are exercised with non-trivial numbers; it is restated in tests/lbr_common.py."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ref_harness as rh  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
N_HANDS = {"Flop5Holdem": 150, "DiscretizedNLHoldem": 80}


def policy_table(range_size, n_actions, legal, street):
    """float32 [R, N_ACTIONS]: weight 1 + ((7 h + 13 a + 3 street) mod 5) on the legal actions, rows normalised"""
    h = np.arange(range_size, dtype=np.int64)[:, None]
    a = np.arange(n_actions, dtype=np.int64)[None, :]
    w = (1 + ((7 * h + 13 * a + 3 * street) % 5)).astype(np.float32)
    mask = np.zeros(n_actions, np.float32)
    mask[list(legal)] = 1.0
    w = w * mask[None, :]
    return (w / w.sum(axis=1, keepdims=True)).astype(np.float32)


def main():
    rh.import_reference()
    import importlib
    W = importlib.import_module("PokerRL.eval.lbr.LocalLBRWorker")  # the package re-exports the class under the module's name
    W = sys.modules["PokerRL.eval.lbr.LocalLBRWorker"]
    from PokerRL.eval.lbr.LBRArgs import LBRArgs
    from PokerRL.game import bet_sets
    from PokerRL.game.Poker import Poker
    from PokerRL.game.games import DiscretizedNLHoldem, Flop5Holdem
    from PokerRL.rl.base_cls.EvalAgentBase import EvalAgentBase

    rec = {"draws": [], "utils": []}

    class TableAgent(EvalAgentBase):
        ALL_MODES = ["table"]

        def can_compute_mode(self):
            return True

        def update_weights(self, w):
            pass

        def _state_dict(self):
            return {}

        def _load_state_dict(self, s):
            pass

        def get_a_probs_for_each_hand(self):
            env = self._internal_env_wrapper.env
            return policy_table(self.env_bldr.rules.RANGE_SIZE, self.env_bldr.N_ACTIONS, env.get_legal_actions(), env.current_round)

        def get_action(self, step_env=True, need_probs=False):
            env = self._internal_env_wrapper.env
            probs = self.get_a_probs_for_each_hand()
            hand = env.get_range_idx(p_id=env.current_player.seat_id)
            u = float(np.random.random())
            rec["draws"][-1].append(u)
            action = int(min(np.searchsorted(np.cumsum(probs[hand].astype(np.float64)), u, side="right"), probs.shape[1] - 1))
            while probs[hand, action] == 0:  # u beyond the last legal action through rounding
                action -= 1
            if step_env:
                self._internal_env_wrapper.step(action=action)
            return action, (probs if need_probs else None)

    out = {}
    for game, bet_set in ((Flop5Holdem, None), (DiscretizedNLHoldem, bet_sets.B_2)):
        name = game.__name__
        kw = dict(n_seats=2, starting_stack_sizes_list=[20000, 20000])
        if bet_set is not None:
            kw["bet_sizes_list_as_frac_of_pot"] = bet_set
        env_args = game.ARGS_CLS(**kw)

        class TProf:
            n_seats = 2
            DISTRIBUTED = CLUSTER = DEBUGGING = HAVE_GPU = False
            env_builder_cls_str = "VanillaEnvBuilder"
            game_cls_str = name
            device_inference = None
            module_args = {"env": env_args,
                           "lbr": LBRArgs(lbr_bet_set=bet_set if bet_set is not None else bet_sets.B_2,
                                          n_lbr_hands_per_seat=N_HANDS[name], lbr_check_to_round=Poker.FLOP,
                                          use_gpu_for_batch_eval=False)}

        worker = W.LocalLBRWorker(t_prof=TProf(), chief_handle=None, eval_agent_cls=TableAgent)
        decks = []
        orig_reset = worker._reset_episode

        def recording_reset(orig_reset=orig_reset, worker=worker, decks=decks):
            ret = orig_reset()
            csd = worker._env.cards_state_dict()
            lut = worker._eval_env_bldr.lut_holder
            hands = np.concatenate([np.asarray(lut.get_1d_cards(np.asarray(h))).reshape(-1) for h in csd["hand"]])
            rest = np.asarray(lut.get_1d_cards(np.asarray(csd["deck"]["deck_remaining"]))).reshape(-1)
            decks.append(np.concatenate([hands, rest]).astype(np.int8))
            rec["draws"].append([])
            rec["utils"].append([])
            return ret

        worker._reset_episode = recording_reset
        # LBR's utilities per decision: np.argmax is the last thing each decision does with them
        real_argmax = np.argmax

        def spy_argmax(a, *args, **kw2):
            if isinstance(a, np.ndarray) and a.dtype == np.float32 and a.ndim == 1 and rec["utils"]:
                rec["utils"][-1].append(np.array(a, np.float64))
            return real_argmax(a, *args, **kw2)

        W.np.argmax = spy_argmax
        wins = {}
        for seat in (0, 1):
            np.random.seed(1234 + seat)
            first = len(decks)
            res = worker.run(agent_seat_id=seat, n_iterations=N_HANDS[name], mode="table", stack_size=[20000, 20000])
            wins[seat] = (first, np.asarray(res, np.float64))
        W.np.argmax = real_argmax
        n = len(decks)
        assert all(d.size == 52 and len(set(d.tolist())) == 52 for d in decks)
        max_draws = max(len(d) for d in rec["draws"][-n:])
        draws = np.full((n, max_draws), -1.0)
        for i, d in enumerate(rec["draws"][-n:]):
            draws[i, :len(d)] = d
        n_act = max(len(x) for u in rec["utils"][-n:] for x in u)
        max_dec = max(len(u) for u in rec["utils"][-n:])
        utils = np.full((n, max_dec, max(len(x) for u in rec["utils"][-n:] for x in u)), np.nan)
        for i, u in enumerate(rec["utils"][-n:]):
            for k, x in enumerate(u):
                utils[i, k, :len(x)] = x
        out[name + "_decks"] = np.array(decks, np.int8)
        out[name + "_draws"] = draws
        out[name + "_utils"] = utils
        out[name + "_agent_seat"] = np.concatenate([np.full(N_HANDS[name], s, np.int8) for s in (0, 1)])
        out[name + "_winnings"] = np.concatenate([wins[0][1], wins[1][1]])
        print(name, "hands", n, "mean LBR winnings per seat", wins[0][1].mean(), wins[1][1].mean(), "decisions recorded",
              sum(len(u) for u in rec["utils"][-n:]), "n_act", n_act)
        rec["draws"].clear()
        rec["utils"].clear()
    np.savez_compressed(os.path.join(OUT, "lbr_runs.npz"), **out)
    print("wrote lbr_runs.npz")


if __name__ == "__main__":
    main()
