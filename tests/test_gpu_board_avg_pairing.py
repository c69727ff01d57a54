"""CFR+ averaging on the board engine two iterations at a time (csrc/cfr_board.cu, AVG; BoardCFRSolver._avg_due): an update
sweep with nothing pending leaves its averaging step pending and the seat's next sweep applies both.  Every result must be the
same bits as the immediate form, where each sweep writes its own step (prl_board_sweep), whatever interrupts the pairs."""
import numpy as np
import pytest

from twocard_common import random_board_spec

pytestmark = pytest.mark.gpu


def _engine(spec, immediate=False, args=None, **kw):
    """Flop5Holdem with the game arguments `args` (default: stacks of 20 000 chips, pot-size bets)"""
    from pokerrl_b200.board_engine import BoardCFRSolver
    from pokerrl_b200.game import games

    class Immediate(BoardCFRSolver):
        """every update sweep writes its own averaging step: the form before pairing, through the unchanged C entry point"""

        def _sweep_begin(self, bufs, p, evaluate, src_own, src_opp):
            self._board_sweep(bufs, p, evaluate, src_own, src_opp, self.iter_counter, self.delay, self.algo)

    g = games.Flop5Holdem
    if args is None:
        args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[20000, 20000], bet_sizes_list_as_frac_of_pot=[1.0])
    return (Immediate if immediate else BoardCFRSolver)(g, args, spec, **kw)


def _assert_same(a, b):
    """post-deal and trunk tables bit for bit (a's pending steps flushed; b's have none), exploitability exactly"""
    import torch
    a.flush_average()
    assert a._avg_due == [-1, -1] and b._avg_due == [-1, -1]
    assert a.iter_counter == b.iter_counter
    for x, y in ((a.regret, b.regret), (a.avg, b.avg), (a.bufs.regret, b.bufs.regret), (a.bufs.strat, b.bufs.strat),
                 (a.bufs.avg, b.bufs.avg)):
        assert torch.equal(x, y)
    assert a.exploitability_current() == b.exploitability_current()
    if a.iter_counter > a.delay:
        assert a.exploitability_average() == b.exploitability_average()


@pytest.mark.parametrize("delay, grid", [pytest.param(d, 0, id=str(d)) for d in (0, 2)]
                         + [pytest.param(d, 7, id="%d-grid7" % d) for d in (0, 2)])
def test_paired_averaging_equals_the_immediate_form(delay, grid):
    """grid 7: every CTA walks 3 or 4 of the 24 boards, so the defer and paired forms carry their state from board to board"""
    spec = random_board_spec(24, 41)
    a, ref = _engine(spec, delay=delay, grid=grid), _engine(spec, immediate=True, delay=delay, grid=grid)
    for n in (1, 2, 3, 7):
        a.reset()
        ref.reset()
        a.iteration(n)
        ref.iteration(n)
        assert (a._avg_due != [-1, -1]) == (n > delay and (n - delay) % 2 == 1)  # iterations delay .. n - 1 have a step
        _assert_same(a, ref)


def test_interrupted_pairs_equal_an_uninterrupted_run():
    """state_dict -> load_state_dict and an average evaluation in the middle of a pair, then more iterations"""
    spec = random_board_spec(24, 43)
    a, ref = _engine(spec), _engine(spec, immediate=True)
    ref.iteration(7)
    a.iteration(3)
    assert a._avg_due == [2, 2]
    st = a.state_dict()  # flushes
    a.reset()
    a.load_state_dict(st)
    a.iteration(4)
    _assert_same(a, ref)
    a.reset()
    a.iteration(3)
    x = a.exploitability_average()  # flushes seat 0 and 1 in the middle of their pairs
    a.iteration(4)
    _assert_same(a, ref)
    ref.reset()
    ref.iteration(3)
    assert x == ref.exploitability_average()


def test_shards_pair_like_one_device():
    """two 'ranks' on one device against one rank holding every board, odd iteration count, after a flush; 3 boards give one
    rank a single board, 1 board leaves one rank without any"""
    import torch
    for n_boards in (30, 3, 1):
        spec = random_board_spec(n_boards, 44)
        one = _engine(spec)
        parts = [_engine(spec, rank=r, world=2, reduce_fn=lambda t: None) for r in range(2)]
        for it in range(5):
            one.iteration(1)
            for p in (0, 1):
                for e in parts:
                    e._update_begin(p)
                tot = parts[0].w_total + parts[1].w_total
                for e in parts:
                    e.w_total.copy_(tot)
                    e._update_end(p)
            for e in parts:
                e.iter_counter += 1
        for e in [one] + parts:
            assert e._avg_due == [4, 4]
            e.flush_average()
        ldb, rpb = one.regret.shape[1], one.rows_per_board

        def per_board(e, tab):  # a rank without boards keeps one placeholder row
            return tab[:e.n_rows].view(e.n_boards, rpb, ldb)
        for r, e in enumerate(parts):  # rank r holds boards r, r + 2, ...
            assert torch.equal(per_board(e, e.regret), per_board(one, one.regret)[r::2])
            assert torch.equal(per_board(e, e.avg), per_board(one, one.avg)[r::2])
            assert torch.equal(e.bufs.regret, one.bufs.regret) and torch.equal(e.bufs.avg, one.bufs.avg)
        assert np.count_nonzero(one.avg.cpu().numpy()) > 0
