"""The restricted Nash response on the full Flop5Holdem game (134 459 suit classes, stack 20 000, default grid): the model
reach tables of 2.93 GB, rows and F addressed past 2^31 bytes, hundreds of boards per CTA, two solvers resident at once.

Check: when the model IS the free copy's current strategy, the mixture (1 - p) * free + p * model is the free copy's reach,
so the exploiter's update at any p must equal the plain CFR+ update from the same tables - and the plain CFR+ path is pinned
to the chunked float64 oracle on this very game by test_gpu_board_full_game.py.  What differs is only round-off: the model's
rows are the float64-normalised matching of the same regrets, and the sweep adds two weighted copies of the reach.  For each
exploiter seat, from a CFR+ solver after one iteration: the model = its current strategy (BoardPolicyTables.from_solver at
iteration delay + 1), an RNR game at p = 0.5 with the solver's tables and its board tables shared, one update of the exploiter
on both; every board's regrets (live hands) and the trunk's regrets at 1e-6 of the board's / trunk's max |ref|."""
import time

import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 1e-6


def test_full_game_exploiter_update_equals_cfr_plus_when_the_model_is_the_free_strategy():
    from pokerrl_b200.board_engine import BoardCFRSolver, BoardPolicyEvaluator, BoardPolicyTables, BoardRNRSolver
    from pokerrl_b200.cfr.RestrictedNashResponse import _TablesAgent
    from pokerrl_b200.game import games
    from pokerrl_b200.game.wrappers import HistoryEnvBuilder
    t0 = time.time()
    G = games.Flop5Holdem
    args = G.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[20000, 20000], bet_sizes_list_as_frac_of_pot=[1.0])
    bldr = HistoryEnvBuilder(env_cls=G, env_args=args)
    ref = BoardCFRSolver(G, args, None, algo="CFRPlus")
    assert ref.n_boards == 134459
    ref.iteration(1)
    nb, rpb, ldb = ref.n_boards, ref.rows_per_board, ref.L["ldb"]
    for s in (0, 1):
        model = BoardPolicyTables.from_solver(ref)  # iteration delay + 1: regret matching of the regrets (flushes ref)
        x = BoardRNRSolver(G, args, s, 0.5, None, share_boards=ref)
        ev = BoardPolicyEvaluator(bldr, stack_size=[20000, 20000], board_spec=ref.spec_full, device=ref.device)
        x.set_model(ev.model_reach(_TablesAgent(model, bldr.N_ACTIONS), {s: x.model_reach}))
        del ev, model
        torch.cuda.empty_cache()
        for a, b in ((x.regret, ref.regret), (x.avg, ref.avg), (x.bufs.regret, ref.bufs.regret),
                     (x.bufs.strat, ref.bufs.strat), (x.bufs.avg, ref.bufs.avg), (x.bufs.reach, ref.bufs.reach)):
            a.copy_(b)
        x.modes, x.iter_counter, x._avg_due = list(ref.modes), ref.iter_counter, list(ref._avg_due)
        mem = torch.cuda.max_memory_allocated() / 2 ** 30
        for e in (x, ref):
            e._update_begin(s)
            e._update_end(s)
            e.flush_average()
        torch.cuda.synchronize()
        worst = 0.0
        for lo in range(0, nb, 8192):  # per board, live hands (the padding past them is 0 in both)
            hi = min(lo + 8192, nb)
            got = x.regret[lo * rpb:hi * rpb].view(hi - lo, -1).double()
            want = ref.regret[lo * rpb:hi * rpb].view(hi - lo, -1).double()
            scale = want.abs().amax(dim=1).clamp(min=1e-300)
            worst = max(worst, float(((got - want).abs().amax(dim=1) / scale).max()))
        nts, R = ref.n_trunk_slots, ref.R
        tw = ref.bufs.regret[:nts, :R].double()
        trunk = float((x.bufs.regret[:nts, :R].double() - tw).abs().max() / tw.abs().max())
        print("full game RNR p 0.5 exploiter %d: board regrets %.2e, trunk regrets %.2e (peak memory %.1f GiB, %.0f s so far)"
              % (s, worst, trunk, mem, time.time() - t0))
        assert worst <= TOL and trunk <= TOL, (s, worst, trunk)
        del x
        torch.cuda.empty_cache()
    print("full game RNR test: %.0f s" % (time.time() - t0))
