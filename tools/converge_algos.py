"""Exploitability against solve time of CFR+ (delay 0), Linear CFR, Discounted CFR and Predictive CFR+ on full Flop5Holdem
(board engine).

    python tools/converge_algos.py --budget 150 --eval-every 20 [--marks 15,30,60,120,150] [--dcfr 1.5,0,2] [--pcfr-gamma 2]
                                  [--algos CFRPlus,LinearCFR,DCFR,PCFRPlus] [--boards N]

Each algorithm runs alone on the GPU for the same solve-time budget (seconds of CFR iterations, evaluation excluded); every
--eval-every iterations the exact exploitability of its average strategy (mbb/g, the number the project reports) is
computed.  Prints one JSON line: the device name and power limit read in this run, each algorithm's iterations/s, and its
exploitability at each mark = the last evaluation whose solve time does not exceed the mark.  --boards N (debugging only)
takes the first N board classes instead of the full game.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def device_info():
    import torch
    info = {"device": torch.cuda.get_device_name(), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        info["power_limit_w"] = float(out.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


def run(algo, spec, budget, eval_every, dcfr, pcfr_gamma):
    import torch
    from pokerrl_b200.board_engine import BoardCFRSolver
    from pokerrl_b200.game import games
    g = games.Flop5Holdem
    args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[20000, 20000], bet_sizes_list_as_frac_of_pot=[1.0])
    s = BoardCFRSolver(g, args, spec, algo=algo, dcfr=dcfr, pcfr_gamma=pcfr_gamma)
    s.iteration(2)  # warm-up of every kernel, then a fresh start
    s.reset()
    torch.cuda.synchronize()
    curve, solve, it = [], 0.0, 0
    while solve < budget:
        t0 = time.perf_counter()
        s.iteration(eval_every)
        torch.cuda.synchronize()
        solve += time.perf_counter() - t0
        it += eval_every
        curve.append({"iteration": it, "solve_s": round(solve, 3), "mbb_per_g_average": s.exploitability_average()})
    del s
    torch.cuda.empty_cache()
    return {"iterations_per_s": it / solve, "curve": curve}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--budget", type=float, default=150.0, help="solve seconds per algorithm")
    ap.add_argument("--eval-every", type=int, default=20)
    ap.add_argument("--marks", default="15,30,60,120,150", help="solve-time marks (s) of the reported exploitability")
    ap.add_argument("--dcfr", default="1.5,0,2", help="DCFR alpha,beta,gamma")
    ap.add_argument("--pcfr-gamma", type=float, default=2.0, help="PCFR+ gamma (average weight t^gamma)")
    ap.add_argument("--algos", default="CFRPlus,LinearCFR,DCFR,PCFRPlus", help="which algorithms, in this order")
    ap.add_argument("--boards", type=int, default=0, help="debugging: the first N board classes only")
    a = ap.parse_args()
    import torch
    from pokerrl_b200.game.games import FlopHoldemRules
    from pokerrl_b200.game.holdem_boards import BoardSpec
    if not torch.cuda.is_available():
        raise SystemExit("converge_algos.py measures on a CUDA device; none is visible")
    spec = BoardSpec.full_game(FlopHoldemRules)
    if a.boards:
        n = a.boards
        spec = BoardSpec(spec.boards[:n], spec.board_prob[:n], spec.board_mult[:n], spec.sym_perm, "first %d classes" % n)
    dcfr = tuple(float(x) for x in a.dcfr.split(","))
    marks = [float(x) for x in a.marks.split(",")]
    out = dict(device_info(), workload="Flop5Holdem full game (%d board classes), stack 20000, pot-size bets" % len(spec.boards),
               budget_solve_s=a.budget, eval_every=a.eval_every, algorithms={})
    labels = {"CFRPlus": "CFR+ delay 0", "LinearCFR": "Linear CFR", "DCFR": "DCFR%r" % (dcfr,),
              "PCFRPlus": "PCFR+(gamma %g)" % a.pcfr_gamma}
    for algo in a.algos.split(","):
        label = labels[algo]
        r = run(algo, spec, a.budget, a.eval_every, dcfr, a.pcfr_gamma)
        at = {}
        for m in marks:
            done = [c for c in r["curve"] if c["solve_s"] <= m]
            at[str(m)] = done[-1]["mbb_per_g_average"] if done else None
        out["algorithms"][label] = {"iterations_per_s": r["iterations_per_s"], "mbb_per_g_average_at_solve_s": at,
                                    "curve": r["curve"]}
        print(label, "%.1f it/s" % r["iterations_per_s"], at, file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
