"""Restricted Nash response on full Flop5Holdem (stack 20 000): the exploitation / exploitability curve over p, the rate and the
memory of each run, and the per-launch time of the exploiter's update forms against the plain CFR+ forms.

    python tools/rnr_curve.py [--iters 100] [--model-iters 10] [--ps 0,0.1,0.25,0.5,0.75,1] [--launches 10] [--out FILE]

The model is an exploitable agent: the CFR+ average after --model-iters iterations (BoardPolicyTables).  Each p runs a fixed
budget of --iters iterations of both games; exploitation and exploitability (mbb/g, seat-averaged) are evaluated once at the
end, outside the timed loop.  Launch times (CUDA events, --launches launches of each form, alternated, after one warm-up
each) compare, on the same seat 0 rows, game 0's exploiter update (RNR form) with game 1's free-copy update (the plain CFR+
form), in the deferred (average left pending) and the paired (pending step applied) averaging modes.  Prints the GPU's name
and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, check=True).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % type(e).__name__


def _launch_ms(torch, fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--model-iters", type=int, default=10)
    ap.add_argument("--ps", default="0,0.1,0.25,0.5,0.75,1")
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from pokerrl_b200.board_engine import BoardCFRSolver, BoardPolicyTables
    from pokerrl_b200.cfr import RestrictedNashResponse
    from pokerrl_b200.game import games
    from pokerrl_b200.rl.base_cls.workers.ChiefBase import ChiefBase
    G, S = games.Flop5Holdem, 20000
    args = G.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[S, S], bet_sizes_list_as_frac_of_pot=[1.0])
    card = _card()
    t0 = time.time()
    s = BoardCFRSolver(G, args, None, algo="CFRPlus")
    s.iteration(a.model_iters)
    model_expl = s.exploitability_average()
    model = BoardPolicyTables.from_solver(s)
    del s
    torch.cuda.empty_cache()
    print("card: %s; model: CFR+ average after %d iterations, exploitability %.4f mbb/g (%.0f s)"
          % (card, a.model_iters, model_expl, time.time() - t0), flush=True)
    out = {"card": card, "model_iters": a.model_iters, "model_exploitability_mbb": model_expl, "iters": a.iters, "runs": [],
           "launch_ms": None}
    for p in [float(x) for x in a.ps.split(",")]:
        torch.cuda.reset_peak_memory_stats()
        t1 = time.time()
        rnr = RestrictedNashResponse("c", ChiefBase(t_prof=None), G, [1.0], model, p, starting_stack_sizes=[S],
                                     eval_every=10 ** 9)
        torch.cuda.synchronize()
        setup = time.time() - t1
        t2 = time.time()
        for _ in range(a.iters):
            rnr.iteration()
        torch.cuda.synchronize()
        rate = a.iters / (time.time() - t2)
        exploitation, exploitability = rnr.values()[0]
        run = dict(p=p, exploitation_mbb=exploitation, exploitability_mbb=exploitability, iterations_per_s=rate,
                   setup_s=setup, peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30,
                   resident_gib=torch.cuda.memory_allocated() / 2 ** 30)
        print("p %.2f: exploitation %.4f mbb/g, exploitability %.4f mbb/g, %.2f iterations/s, set-up %.0f s, memory %.1f GiB "
              "resident (peak %.1f)" % (p, exploitation, exploitability, rate, setup, run["resident_gib"], run["peak_gib"]),
              flush=True)
        out["runs"].append(run)
        if p == 0.5 and a.launches > 0:
            g0, g1 = rnr.games[0]
            t = g0.iter_counter
            forms = {"rnr deferred": lambda: g0._board_update_cfrp(0, -1, 0),
                     "cfr+ deferred": lambda: g1._board_update_cfrp(0, -1, 0),
                     "rnr paired": lambda: g0._board_update_cfrp(0, t - 1, 1),
                     "cfr+ paired": lambda: g1._board_update_cfrp(0, t - 1, 1)}
            ms = {k: [] for k in forms}
            for _ in range(3):  # alternated rounds
                for k, f in forms.items():
                    ms[k].append(_launch_ms(torch, f, a.launches))
            out["launch_ms"] = {k: min(v) for k, v in ms.items()}
            print("launch times (seat 0 update, best of 3 rounds of %d): %s" % (
                a.launches, ", ".join("%s %.3f ms" % kv for kv in out["launch_ms"].items())), flush=True)
            del forms, g0, g1  # the closures hold the games
        del rnr
        torch.cuda.empty_cache()
    print("card (read again): %s; total %.0f s" % (_card(), time.time() - t0))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
