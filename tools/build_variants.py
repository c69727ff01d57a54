"""A/B builds of the board sweep kernel: python tools/build_variants.py
Compiles csrc/cfr_board.cu with different PRL_BV_* switches into pokerrl_b200/lib/variants/lib_<name>.so (the other
translation units are taken from the regular build); run one with PRL_LIB_PATH=<that file> python tools/board_probe.py."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pokerrl_b200.csrc import build as B  # noqa: E402

# switches left in csrc/cfr_board.cu: each accepted change against its predecessor (the rejected ones were removed from the
# source)
_ON = dict(RED=1, P1PIPE=1, FOLDLIN=1, ERT=1, ROWTOTF=1, NEWTON=1, PF=1, STAMPS=0)
VARIANTS = {
    "final": dict(_ON),
    "base": dict(RED=0, P1PIPE=0, FOLDLIN=0, ERT=0, ROWTOTF=0, NEWTON=1, PF=0, STAMPS=0),
    "no_red": dict(_ON, RED=0),
    "no_p1pipe": dict(_ON, P1PIPE=0),
    "no_foldlin": dict(_ON, FOLDLIN=0),
    "no_ert": dict(_ON, ERT=0),
    "no_rowtotf": dict(_ON, ROWTOTF=0),
    "no_newton": dict(_ON, NEWTON=0),
    "pf0": dict(_ON, PF=0),
    # phase stamps (tools/board_phases.py) of the kept schedule and of the previous one
    "stamps": dict(_ON, STAMPS=1),
    "stamps_pf0": dict(_ON, PF=0, STAMPS=1),
}


def main(names):
    B.build()
    out_dir = os.path.join(B.LIB_DIR, "variants")
    os.makedirs(out_dir, exist_ok=True)
    obj_dir = os.path.join(B.LIB_DIR, "obj")
    others = [os.path.join(obj_dir, s.replace(".cu", ".o")) for s in B.SOURCES if s != "cfr_board.cu"]
    for name in names:
        defs = ["-DPRL_BV_%s=%d" % kv for kv in VARIANTS[name].items()]
        o = os.path.join(out_dir, "cfr_board_%s.o" % name)
        subprocess.check_call([B.NVCC] + B.ARCH + B.COMMON + B.SOURCES["cfr_board.cu"] + defs +
                              ["-c", os.path.join(B.HERE, "cfr_board.cu"), "-o", o])
        lib = os.path.join(out_dir, "lib_%s.so" % name)
        subprocess.check_call([B.NVCC] + B.ARCH + ["-shared", "-o", lib, o] + others)
        print(lib)


if __name__ == "__main__":
    main(sys.argv[1:] or list(VARIANTS))
