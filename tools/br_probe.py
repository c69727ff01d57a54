"""Wall time and memory of one best-response evaluation on the board engine (board_engine.BoardPolicyEvaluator): a
full-game Flop5Holdem CFR+ agent (a few iterations, TabularCFREvalAgent.from_cfr) evaluated on the 134 459 suit classes and
on all 2 598 960 deals, split into agent query, table build and sweeps (synchronised phases), with the peak of
torch.cuda.max_memory_allocated, the card and its power limit.  --best-response: on the classes, BoardPolicyEvaluator.best_response
against evaluate (same split), then the launch time of the export form of the evaluation sweep against the plain one (CUDA
events, alternated, on the last chunk's boards).

    python tools/br_probe.py [--iters 4] [--chunk N] [--skip-deals] [--best-response]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _power_limit():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                       text=True).strip()
    except Exception as e:  # noqa: BLE001 - informative only
        return "unknown (%s)" % type(e).__name__


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=4)
    ap.add_argument("--chunk", type=int, default=None)
    ap.add_argument("--skip-deals", action="store_true")
    ap.add_argument("--best-response", action="store_true")
    a = ap.parse_args()
    import torch
    from pokerrl_b200.board_engine import BoardPolicyEvaluator
    from pokerrl_b200.cfr.CFRPlus import CFRPlus
    from pokerrl_b200.cfr.TabularCFREvalAgent import TabularCFREvalAgent
    from pokerrl_b200.game import games
    from pokerrl_b200.game.holdem_boards import BoardSpec
    from pokerrl_b200.game.wrappers import HistoryEnvBuilder
    from pokerrl_b200.rl.base_cls.TrainingProfileBase import TrainingProfileBase
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    G, stack = games.Flop5Holdem, [20000, 20000]
    print("card %s, power limit %s" % (torch.cuda.get_device_name(0), _power_limit()))
    cfr = CFRPlus(name="probe", chief_handle=ChiefBase(None), game_cls=G, agent_bet_set=[1.0], eval_every=10 ** 9)
    for _ in range(a.iters):
        cfr.iteration()
    agent = TabularCFREvalAgent.from_cfr(TrainingProfileBase("probe", G, [1.0], eval_stack_sizes=[stack]), cfr)
    bldr = HistoryEnvBuilder(env_cls=G, env_args=G.ARGS_CLS(n_seats=2, starting_stack_sizes_list=stack,
                                                            bet_sizes_list_as_frac_of_pot=[1.0]))
    if a.best_response:
        del cfr
        torch.cuda.empty_cache()
        return best_response(bldr, stack, agent, a.chunk, G)
    specs = [("classes", None)] + ([] if a.skip_deals else [("all deals", BoardSpec.full_game(G.RULES, isomorphic=False))])
    for name, spec in specs:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        ev = BoardPolicyEvaluator(bldr, stack, spec, chunk=a.chunk)
        t1 = time.perf_counter()
        e = ev.evaluate(agent, profile=True)
        t2 = time.perf_counter()
        print("%-9s %8d boards, chunk %6d: %.1f s (set-up %.1f s; %s), exploitability %.6f mbb/g, peak %.2f GB "
              "(%.2f GB held before: solver + agent)"
              % (name, ev.n_boards_total, ev.chunk, t2 - t0, t1 - t0, ", ".join("%s %.1f s" % kv for kv in ev.times.items()),
                 (e[0] + e[1]) / 2 * G.EV_NORMALIZER, torch.cuda.max_memory_allocated() / 1e9, base / 1e9))
        del ev


def best_response(bldr, stack, agent, chunk, G):
    import torch
    from pokerrl_b200 import _native as nat
    from pokerrl_b200.board_engine import SRC_AVG, BoardPolicyEvaluator
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ev = BoardPolicyEvaluator(bldr, stack, None, chunk=chunk)
    for what in ("evaluate", "best_response", "evaluate", "best_response"):
        t0 = time.perf_counter()
        out = getattr(ev, what)(agent, profile=True)
        dt = time.perf_counter() - t0
        e = out if what == "evaluate" else out[0]
        print("%-13s %d classes, chunk %d: %.1f s (%s), exploitability %r" % (what, ev.n_boards_total, ev.chunk, dt,
              ", ".join("%s %.2f s" % kv for kv in ev.times.items()), list(e)))
        del out
    print("peak %.2f GB (%.2f GB held before: the agent)" % (torch.cuda.max_memory_allocated() / 1e9, base / 1e9))
    # launch time of the export form against the plain evaluation sweep, on the boards of the last chunk
    nb = ev.g.n_boards
    scratch = torch.empty((nb * ev.rows_per_board, ev.L["ldb"]), dtype=torch.float32, device=ev.device)
    times = {0: [], 1: []}
    for rep in range(12):
        for export in (0, 1):
            ev.g.br_out = scratch.data_ptr() if export else None
            s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s0.record()
            for p in (0, 1):
                ev._board_sweep(ev.bufs, p, True, SRC_AVG, SRC_AVG, 0, 0, nat.ALGO_CFR_PLUS)
            s1.record()
            torch.cuda.synchronize()
            if rep >= 2:
                times[export].append(s0.elapsed_time(s1) / 2)
    ev.g.br_out = None
    plain, exp = float(np.median(times[0])), float(np.median(times[1]))
    print("evaluation sweep on %d boards (median of 10 alternated pairs, per seat): plain %.3f ms, export %.3f ms (%+.1f %%); "
          "export writes %.2f GB per seat" % (nb, plain, exp, 100 * (exp / plain - 1), nb * ev.rows_per_board / 2 * 4352 / 1e9))


if __name__ == "__main__":
    main()
