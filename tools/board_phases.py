"""Phase stamps of the board sweep on one GPU:
    python tools/build_variants.py stamps && PRL_LIB_PATH=pokerrl_b200/lib/variants/lib_stamps.so python tools/board_phases.py [n_boards] [grid]
For each form of board_sweep_kernel (CFR+ update: defer, paired; evaluation) the SM cycles thread 0 of each CTA spends from the
unit start to B1 and between consecutive barriers B1 .. B5 (median and p90 over the sampled units of every CTA, both seats),
next to the CUDA-event time per launch of the same forms and of avg_flush_kernel, and the L2 footprint model of the row
prefetches (DESIGN.md §6.1).  Prints a table, then one JSON line."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pokerrl_b200 import _native as nat  # noqa: E402
from pokerrl_b200.board_engine import BoardCFRSolver, _stream  # noqa: E402
from pokerrl_b200.game import games  # noqa: E402
from pokerrl_b200.game.holdem_boards import BoardSpec  # noqa: E402

PHASES = ["P1 (start-B1)", "P2a+scan (B1-B2)", "totals (B2-B3)", "write-back (B3-B4)", "P3 (B4-B5)", "unit"]
# rows per board a form reads through the prefetched streams / writes (7 rows per seat and table)
ROWS = {"defer": dict(opp=7, own=7, written=7), "paired": dict(opp=7, own=14, written=14), "eval": dict(opp=7, own=7, written=0)}


def card():
    q = "--query-gpu=name,power.limit,clocks.max.sm"
    try:
        out = subprocess.check_output(["nvidia-smi", "-i", str(torch.cuda.current_device()), q, "--format=csv,noheader,nounits"],
                                      text=True).strip()
        name, plim, mhz = [x.strip() for x in out.split(",")]
        return name, float(plim), float(mhz)
    except (OSError, subprocess.CalledProcessError, ValueError):
        return torch.cuda.get_device_name(), None, None


def main():
    nb = int(sys.argv[1]) if len(sys.argv) > 1 else 134459
    grid = int(sys.argv[2]) if len(sys.argv) > 2 else 0
    L = nat.lib()
    if not hasattr(L, "prl_board_stamps"):
        raise SystemExit("%s has no phase stamps: build tools/build_variants.py stamps and point PRL_LIB_PATH at it" % nat.LIB_PATH)
    L.prl_board_stamps.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
    L.prl_board_stamps.restype = C.c_int
    shape = (C.c_int32 * 3)()
    buf = np.zeros(1 << 16, np.int64)

    def read_stamps():
        torch.cuda.synchronize()
        if L.prl_board_stamps(buf.ctypes.data, shape) != 0:
            raise RuntimeError(L.prl_last_error().decode())
        n = shape[0] * shape[1] * shape[2]
        assert n <= buf.size
        return buf[:n].reshape(shape[0], shape[1], shape[2]).copy()

    g = games.Flop5Holdem
    args = g.ARGS_CLS(n_seats=2, starting_stack_sizes_list=[20000, 20000], bet_sizes_list_as_frac_of_pot=[1.0])
    spec = BoardSpec.full_game(g.RULES)
    if nb < spec.boards.shape[0]:
        spec = BoardSpec(spec.boards[:nb], spec.board_prob[:nb], spec.board_mult[:nb], spec.sym_perm, "first %d" % nb)
    s = BoardCFRSolver(g, args, spec, grid=grid)
    s.iteration(3)
    torch.cuda.synchronize()
    t, stream = s.iter_counter, _stream(s.device)
    forms = {
        "defer": lambda p: s._board_update_cfrp(p, -1, 0),
        "paired": lambda p: s._board_update_cfrp(p, t - 1, 1),
        "eval": lambda p: s._sweep_begin(s.bufs, p, True, 0, 0),
        "flush": lambda p: nat.call("prl_board_avg_flush", C.byref(s.g), p, t - 1, s.delay, stream),
    }
    name, plim, mhz = card()
    n_grid = s.g.grid
    res = {}
    for k, launch in forms.items():
        ms, units = [], []
        for p in (0, 1):
            launch(p)  # warm
            read_stamps()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            launch(p)
            e1.record()
            st = read_stamps()  # the stamps of the timed launch (the flush kernel writes none)
            ms.append(e0.elapsed_time(e1))
            st = st[:n_grid].reshape(-1, st.shape[2])
            ok = (st[:, 7] > 0) & (st[:, 5] > st[:, 0])  # it = 0 waits for the first board's tables: left out
            units.append(st[ok])
        u = np.concatenate(units)
        r = {"ms": ms, "cycles_per_board_slot": None, "units": int(u.shape[0])}
        if mhz:
            r["cycles_per_board_slot"] = float(np.median(ms)) * 1e-3 * mhz * 1e6 * n_grid / s.n_boards
        if u.shape[0]:
            d = np.stack([u[:, 1] - u[:, 0], u[:, 2] - u[:, 1], u[:, 3] - u[:, 2], u[:, 4] - u[:, 3], u[:, 5] - u[:, 4],
                          u[:, 5] - u[:, 0]], axis=1)
            r["phases"] = {ph: {"median": float(np.median(d[:, i])), "p90": float(np.percentile(d[:, i], 90))}
                           for i, ph in enumerate(PHASES)}
            r["sms"] = int(np.unique(u[:, 6]).size)
        res[k] = r

    # L2 footprint model: rows of the prefetched streams resident per CTA at the top of a unit, plus the lines the previous
    # unit stored (not yet written back), times the grid, against the card's L2
    l2 = torch.cuda.get_device_properties(s.device).L2_cache_size
    row = s.L["ldb"] * 4
    model = {}
    for k, rw in ROWS.items():
        clean1 = (rw["opp"] + rw["own"]) * row
        model[k] = {"clean_per_cta_one_board": clean1, "dirty_per_cta": rw["written"] * row,
                    "total_two_boards_ahead": n_grid * (2 * clean1 + rw["written"] * row),
                    "total_one_phase_ahead": n_grid * (clean1 + rw["written"] * row)}

    print("%s, power limit %s W, max SM clock %s MHz, L2 %.1f MB, %d boards, grid %d (%s)"
          % (name, plim, mhz, l2 / 2 ** 20, s.n_boards, n_grid, os.path.basename(nat.LIB_PATH)))
    print("%-8s %9s %9s  " % ("form", "ms", "cyc/slot") + "  ".join("%20s" % ph for ph in PHASES))
    for k, r in res.items():
        cells = ["%20s" % ("%d / %d" % (r["phases"][ph]["median"], r["phases"][ph]["p90"])) for ph in PHASES] if "phases" in r else []
        print("%-8s %9.3f %9s  " % (k, float(np.median(r["ms"])), "%.0f" % r["cycles_per_board_slot"] if r["cycles_per_board_slot"] else "-")
              + "  ".join(cells))
    print("(phase cells: median / p90 SM cycles per unit; cyc/slot = event time x max clock x grid / boards)")
    print("L2 footprint model (MB = 2^20 B; L2 %.1f MB):" % (l2 / 2 ** 20))
    for k, m in model.items():
        print("  %-7s clean per CTA, one board %5.1f KB, dirty per CTA %5.1f KB: rows two boards ahead %5.1f MB, one phase ahead %5.1f MB"
              % (k, m["clean_per_cta_one_board"] / 1024, m["dirty_per_cta"] / 1024, m["total_two_boards_ahead"] / 2 ** 20,
                 m["total_one_phase_ahead"] / 2 ** 20))
    print(json.dumps({"card": name, "power_limit_w": plim, "max_sm_mhz": mhz, "l2_bytes": l2, "boards": s.n_boards, "grid": n_grid,
                      "lib": os.path.basename(nat.LIB_PATH), "forms": res, "l2_model": model}))


if __name__ == "__main__":
    main()
