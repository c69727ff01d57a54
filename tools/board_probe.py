"""Timing probe of the board engine on one GPU: python tools/board_probe.py [n_boards] [iterations] [grid] [stack]
(stack default 20000: the 15-node post-deal shape; 301 to 900: the 9-node one).  CUDA-event times of the iteration, of each form of the CFR+ update sweep and of the average flush (per launch, over many
launches), and of the evaluation passes, with the bytes each form moves and the card it ran on."""
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pokerrl_b200 import _native as nat  # noqa: E402
from pokerrl_b200.board_engine import BoardCFRSolver, _stream  # noqa: E402
from pokerrl_b200.game import games  # noqa: E402
from pokerrl_b200.game.holdem_boards import BoardSpec  # noqa: E402

nb = int(sys.argv[1]) if len(sys.argv) > 1 else 20000
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 10
grid = int(sys.argv[3]) if len(sys.argv) > 3 else 0
stack = int(sys.argv[4]) if len(sys.argv) > 4 else 20000
g = games.Flop5Holdem
args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[stack, stack], bet_sizes_list_as_frac_of_pot=[1.0])
t0 = time.perf_counter()
spec = BoardSpec.full_game(g.RULES)
if nb < spec.boards.shape[0]:
    spec = BoardSpec(spec.boards[:nb], spec.board_prob[:nb], spec.board_mult[:nb], spec.sym_perm, "first %d" % nb)
t_spec = time.perf_counter() - t0
t0 = time.perf_counter()
s = BoardCFRSolver(g, args, spec, grid=grid)
torch.cuda.synchronize()
t_build = time.perf_counter() - t0
s.iteration(3)
torch.cuda.synchronize()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
ev[0].record()
s.iteration(iters)
ev[1].record()
torch.cuda.synchronize()
it_ms = ev[0].elapsed_time(ev[1]) / iters
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
a = s.exploitability_current()
b = s.exploitability_average()
e1.record()
torch.cuda.synchronize()
eval_ms = e0.elapsed_time(e1)


def per_launch_ms(launch, reps=10):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        launch()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


# the forms of one seat's CFR+ update at iteration t (after this the solver's tables are no longer a CFR+ run)
t, stream = s.iter_counter, _stream(s.device)
forms = {
    "defer": lambda p: s._board_update_cfrp(p, -1, 0),
    "paired": lambda p: s._board_update_cfrp(p, t - 1, 1),
    "flush": lambda p: nat.call("prl_board_avg_flush", C.byref(s.g), p, t - 1, s.delay, stream),
}
# a seat owns half of a board's rows: defer reads the opponent's and its own regrets and writes its own (3 halves), paired also
# reads and writes its average (5 halves), flush reads its regrets and average and writes its average (3 halves)
row, half = s.L["ldb"] * 4, s.rows_per_board // 2
bytes_per_board = {"defer": 3 * half * row + s.L["blob"], "paired": 5 * half * row + s.L["blob"], "flush": 3 * half * row}
times = {k: [] for k in forms}
for rnd in range(3):
    for k, launch in forms.items():
        for p in (0, 1):
            times[k].append(per_launch_ms(lambda: launch(p)))
res = {}
for k in forms:
    ms = statistics.median(times[k])
    res[k] = {"ms": ms, "ms_all": times[k], "bytes": s.n_boards * bytes_per_board[k],
              "GBps": s.n_boards * bytes_per_board[k] / (ms * 1e-3) / 1e9}
try:
    card = subprocess.check_output(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                                    "--format=csv,noheader"], text=True).strip()
except (OSError, subprocess.CalledProcessError):
    card = torch.cuda.get_device_name() + " (power limit not readable)"
print(json.dumps({"card": card, "boards": s.n_boards, "spec_s": t_spec, "build_s": t_build, "ms_per_iteration": it_ms,
                  "iterations_per_s": 1e3 / it_ms, "update_sweep_forms": res, "eval_both_ms": eval_ms, "expl_cur": a,
                  "expl_avg": b, "mem_GB": torch.cuda.max_memory_allocated() / 2 ** 30, "grid": s.g.grid,
                  **({"stack": stack, "rows_per_board": s.rows_per_board} if stack != 20000 else {})}))
