#!/usr/bin/env python
"""Per-step timeline of the persistent LSTM recurrence for one shape: builds a -DAERO_TC_TRACE twin of the library
(clock64 stamps of CTA 0: MMA warpgroup / cell-update events per step) and prints per-step intervals.
    python tools/tc_trace.py lstm96"""
import ctypes as C
import glob
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
LIB = os.path.join(ROOT, "aero_b200", "libaero_b200_trace.so")


def build():
    from aero_b200 import build as b
    srcs = sorted(glob.glob(os.path.join(b.CSRC, "*.cu")))
    if os.path.exists(LIB) and all(os.path.getmtime(LIB) > os.path.getmtime(s) for s in srcs + glob.glob(os.path.join(b.CSRC, "*.cuh"))):
        return
    subprocess.check_call(["nvcc", *b.NVCC_FLAGS, "-DAERO_TC_TRACE", "-shared", "-o", LIB, *srcs, "-lcudart", "-lcuda"])


if __name__ == "__main__":
    if sys.argv[1] == "--build":
        build()
        sys.exit(0)
    from aero_b200 import cabi
    cabi.LIB_PATH = LIB
    import tools.kprof as kp
    sys.argv = [sys.argv[0], sys.argv[1], "--iters", "1"] + sys.argv[2:]
    kp.main()
    lib = cabi.load()
    assert sys.argv[1].startswith("lstm"), "only the LSTM recurrence carries trace stamps"
    buf = (C.c_longlong * (128 * 8))()
    lib.aero_debug_lstm_trace.argtypes = [C.c_void_p]
    assert lib.aero_debug_lstm_trace(buf) == 0
    rows = [[buf[i * 8 + j] for j in range(8)] for i in range(128)]
    names = ["mma:h_ready", "mma:commit", "upd:top", "upd:acc", "upd:act", "upd:h_stored", "upd:arrived"]
    t0 = rows[1][0]
    print("step " + " ".join(f"{n:>12s}" for n in names) + "   (cycles; update warp 0 lane 0)")
    for i in range(1, int(os.environ.get("ROWS", 24))):
        print(f"{i:4d} " + " ".join(f"{v - t0:12d}" if v else " " * 12 for v in rows[i][:7]))
    print(f"steady state: {(rows[100][0] - rows[20][0]) / 80:.0f} cycles per step")
    sys.exit(0)
