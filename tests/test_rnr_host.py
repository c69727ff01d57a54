"""Restricted Nash response without a GPU: the float64 restatement (tests/rnr_common.py) against the CFR+ oracle, and the
refusals of cfr.RestrictedNashResponse, which all come before anything is allocated on a device."""
import math

import numpy as np
import pytest

import cfr2_numpy as o2
from rnr_common import Oracle2RNR, random_model
from twocard_common import fhp_tree, oracle_tree, random_board_spec


def _slots(ft, per_node):
    out = np.zeros((ft.n_slots, ft.R))
    for n in np.nonzero((ft.kind <= 1) & (ft.first_child >= 0))[0]:
        if per_node[n] is not None:
            fs, A = int(ft.first_slot[n]), int(ft.n_children[n])
            out[fs:fs + A] = per_node[n].T
    return out


@pytest.mark.parametrize("seat", [0, 1])
def test_p0_is_the_cfr_plus_oracle_bit_for_bit(seat):
    ft = fhp_tree(random_board_spec(3, 2))
    cfr = o2.Oracle2CFR(oracle_tree(ft), "CFRPlus")
    rnr = Oracle2RNR(oracle_tree(ft), seat, 0.0, random_model(ft, 1))
    for _ in range(3):
        cfr.iteration()
        rnr.iteration()
        assert np.array_equal(_slots(ft, cfr.regret), rnr.regret)
        assert np.array_equal(_slots(ft, cfr.avg), rnr.avg)


def test_p1_values_are_the_values_against_the_model():
    ft = fhp_tree(random_board_spec(3, 4))
    model = random_model(ft, 2)
    rnr = Oracle2RNR(oracle_tree(ft), 1, 1.0, model)
    rnr.iteration()
    got = rnr.values(1)
    want = rnr._play("current", "model")[0][:, 1]
    assert np.array_equal(got, want)
    assert not np.array_equal(got, rnr._play("current", "current")[0][:, 1])
    assert not np.any(rnr.regret[:, :][_seat_rows(ft, 0)])  # the free copy never plays at p = 1


def _seat_rows(ft, seat):
    rows = np.zeros(ft.n_slots, bool)
    for n in np.nonzero((ft.kind == seat) & (ft.first_child >= 0))[0]:
        rows[int(ft.first_slot[n]):int(ft.first_slot[n]) + int(ft.n_children[n])] = True
    return rows


@pytest.mark.parametrize("p", [-0.1, 1.5, math.nan, math.inf, "x"])
def test_probability_outside_the_unit_interval_is_refused(p):
    from pokerrl_b200.cfr import RestrictedNashResponse
    from pokerrl_b200.game import games
    with pytest.raises((ValueError, TypeError)):
        RestrictedNashResponse("r", None, games.Flop5Holdem, [1.0], model=None, p=p)


@pytest.mark.parametrize("game, stack", [("StandardLeduc", None), ("LimitHoldem", None), ("Flop5Holdem", 300)])
def test_games_the_board_engine_does_not_run_are_refused(game, stack):
    from pokerrl_b200.cfr import RestrictedNashResponse
    from pokerrl_b200.game import bet_sets, games
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    G = getattr(games, game)
    with pytest.raises(ValueError, match="board engine"):
        RestrictedNashResponse("r", ChiefBase(t_prof=None), G, bet_sets.POT_ONLY if game != "Flop5Holdem" else [1.0], None,
                               0.5, starting_stack_sizes=None if stack is None else [stack])


def test_distributed_runs_are_refused(monkeypatch):
    import torch.distributed as dist
    from pokerrl_b200.cfr import RestrictedNashResponse
    from pokerrl_b200.game import games
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda: 2)
    with pytest.raises(ValueError, match="one GPU"):
        RestrictedNashResponse("r", None, games.Flop5Holdem, [1.0], None, 0.5)


def test_checkpoint_identity_refuses_another_p_seat_or_model():
    from pokerrl_b200 import algorithm
    from pokerrl_b200.board_engine import rnr_identity
    mine = {"engine": "board", "algo": "CFRPlus", **rnr_identity(0, 0.5, 1234)}
    algorithm.check_identity(dict(mine), mine)
    for k, v in (("rnr_p", 0.25), ("rnr_seat", 1), ("rnr_model", 99)):
        with pytest.raises(ValueError, match=k):
            algorithm.check_identity({**mine, k: v}, mine)
    with pytest.raises(ValueError, match="rnr_"):  # a checkpoint of a plain CFR+ run
        algorithm.check_identity({k: v for k, v in mine.items() if not k.startswith("rnr")}, mine)


@pytest.mark.parametrize("game", ["StandardLeduc", "LimitHoldem"])
def test_a_model_of_another_betting_tree_is_refused(game):
    from pokerrl_b200.cfr import RestrictedNashResponse
    from pokerrl_b200.game import bet_sets, games
    from pokerrl_b200.rl.base_cls.EvalAgentBase import EvalAgentBase
    from pokerrl_b200.rl.base_cls.TrainingProfileBase import TrainingProfileBase
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    agent = EvalAgentBase(TrainingProfileBase("m", getattr(games, game), bet_sets.POT_ONLY))
    with pytest.raises(ValueError, match="different betting tree|does not run"):
        RestrictedNashResponse("r", ChiefBase(t_prof=None), games.Flop5Holdem, [1.0], agent, 0.5)
    with pytest.raises(ValueError, match="EvalAgentBase or BoardPolicyTables"):
        RestrictedNashResponse("r", ChiefBase(t_prof=None), games.Flop5Holdem, [1.0], object(), 0.5)
