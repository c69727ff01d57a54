"""Phase-stamp build of the board sweep kernel: python tools/build_variants.py stamps
Compiles csrc/cfr_board.cu with PRL_BV_STAMPS=1 into pokerrl_b200/lib/variants/lib_stamps.so (the other translation units
are taken from the regular build); run it with PRL_LIB_PATH=<that file> python tools/board_phases.py."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pokerrl_b200.csrc import build as B  # noqa: E402

VARIANTS = {
    "stamps": dict(STAMPS=1),  # phase stamps (tools/board_phases.py)
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
