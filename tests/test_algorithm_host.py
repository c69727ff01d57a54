"""The host rules of the four CFR algorithms (pokerrl_b200.algorithm) without a GPU: where the average strategy is, the weight
of an iteration in the average sums, which parameters each algorithm keeps, and the checkpoint keys of both engines."""
import math
import types

import pytest
import torch

from pokerrl_b200 import _native as nat
from pokerrl_b200 import dcfr
from pokerrl_b200.algorithm import ALGOS, AVERAGE, CURRENT, SUMS, Algorithm, check_identity

NAMES = ["VanillaCFR", "CFRPlus", "LinearCFR", "DCFR"]


@pytest.mark.parametrize("delay", [0, 2])
@pytest.mark.parametrize("name", NAMES)
def test_average_source_by_counter(name, delay):
    a = Algorithm(name, delay, device="cpu")
    if name != "CFRPlus":
        assert [a.average(t) for t in range(5)] == [SUMS] * 5
        return
    for t in range(delay + 1):
        with pytest.raises(RuntimeError, match="no average strategy before iteration delay\\+1"):
            a.average(t)
    assert [a.average(t) for t in range(delay + 1, 5)] == [CURRENT] + [AVERAGE] * (3 - delay)


@pytest.mark.parametrize("params", [dcfr.DEFAULT, (1.0, 0.5, 3.0)])
def test_sum_weight(params):
    f = dcfr.factors(*params, 998)
    for t in (0, 1, 997):
        assert Algorithm("VanillaCFR").sum_weight(t) == 1.0
        assert Algorithm("LinearCFR").sum_weight(t) == float(t + 1)
        assert Algorithm("CFRPlus", delay=2).sum_weight(t) is None
        w = Algorithm("DCFR", dcfr=params, device="cpu").sum_weight(t)
        assert type(w) is float and w == float(f[t, 2]), (params, t)


def test_unknown_names_and_parameters_of_other_algorithms():
    for bad in ("CFR+", "DiscountedCFR", "cfrplus"):
        with pytest.raises(ValueError, match="unknown algorithm"):
            Algorithm(bad)
    with pytest.raises(ValueError, match="finite"):
        Algorithm("DCFR", dcfr=(math.nan, 0.0, 2.0))
    for name in NAMES:
        a = Algorithm(name, delay=3, dcfr=(1.0, 0.5, 3.0), device="cpu")
        assert a.name == name and a.code == ALGOS[name]
        assert a.delay == (3 if name == "CFRPlus" else 0)
        assert a.dcfr == ((1.0, 0.5, 3.0) if name == "DCFR" else None)
        assert (a.factor_table(4) is None) == (name != "DCFR")
        if name != "DCFR":  # parameters DCFR would refuse are not looked at
            assert Algorithm(name, dcfr=(math.nan, "x", None)).dcfr is None
    assert ALGOS == {"VanillaCFR": nat.ALGO_VANILLA, "CFRPlus": nat.ALGO_CFR_PLUS, "LinearCFR": nat.ALGO_LINEAR,
                     "DCFR": nat.ALGO_DCFR}


def _tables(*names):
    return types.SimpleNamespace(**{n: torch.zeros(2, 3) for n in names})


def _level_solver(alg, avg_f64=False, **kw):
    from pokerrl_b200.solver import CFRSolver
    s = CFRSolver.__new__(CFRSolver)
    s.alg, s.avg_f64, s.ft, s.iter_counter, s.modes = alg, avg_f64, types.SimpleNamespace(n_nodes=7), 3, [0, 0]
    s.bufs = _tables("regret", "strat", "avg")
    s.__dict__.update(kw)
    return s


def _board_solver(alg):
    from pokerrl_b200.board_engine import BoardCFRSolver
    s = BoardCFRSolver.__new__(BoardCFRSolver)
    s.alg, s.device, s.iter_counter, s.modes = alg, -1, 3, [0, 0]
    s.rank, s.world, s.n_boards, s.n_boards_total = 1, 2, 5, 9
    s.regret, s.avg, s.bufs = torch.zeros(2, 3), torch.zeros(2, 3), _tables("regret", "strat", "avg")
    s._pending, s._avg_due = [0.0, 0.0], [-1, -1]
    return s


@pytest.mark.parametrize("name", NAMES)
def test_checkpoint_headers_of_both_engines(name):
    """the header keys as both engines have written them since DCFR was added"""
    alg = Algorithm(name, delay=2, device="cpu")
    d = [1.5, 0.0, 2.0] if name == "DCFR" else None
    delay = 2 if name == "CFRPlus" else 0
    assert alg.identity() == {"algo": name, "delay": delay, "dcfr": d}
    level = _level_solver(alg, avg_f64=name == "CFRPlus").state_dict()
    assert {k: level[k] for k in ("engine", "algo", "delay", "avg_f64", "dcfr", "rank", "world", "n_nodes")} == {
        "engine": "levels", "algo": name, "delay": delay, "avg_f64": name == "CFRPlus", "dcfr": d, "rank": 0, "world": 1,
        "n_nodes": 7}
    sharded = _level_solver(alg, rank=1, world=4).state_dict()
    assert (sharded["rank"], sharded["world"]) == (1, 4)
    board = _board_solver(alg).state_dict()
    assert {k: board[k] for k in ("engine", "algo", "delay", "dcfr", "rank", "world", "n_boards", "n_boards_total")} == {
        "engine": "board", "algo": name, "delay": delay, "dcfr": d, "rank": 1, "world": 2, "n_boards": 5, "n_boards_total": 9}


def test_check_identity_names_the_key_and_refuses_a_missing_one():
    mine = {"engine": "board", **Algorithm("DCFR", device="cpu").identity(), "rank": 0}
    check_identity(dict(mine, iter_counter=3), mine)
    with pytest.raises(ValueError, match="checkpoint mismatch on 'dcfr': file has \\[1.0, 0.5, 3.0\\]"):
        check_identity(dict(mine, dcfr=[1.0, 0.5, 3.0]), mine)
    with pytest.raises(ValueError, match="checkpoint mismatch on 'rank': file has None"):
        check_identity({k: v for k, v in mine.items() if k != "rank"}, mine)
    other = {"engine": "levels", **Algorithm("CFRPlus", delay=1).identity()}
    check_identity(dict(other, dcfr=None), other)  # written by CFR+: dcfr None
    with pytest.raises(ValueError, match="'delay'"):
        check_identity(dict(other, delay=0), other)
