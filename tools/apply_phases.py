"""Where a window of the region replay (shuffle_algo 9) spends its time: the phase clocks of nhood_apply_part_kernel at
configs[1] (1M spots, 30 clusters, P permutations), in cycles per window as warp 0 of a CTA sees them.  They exist in the
clocks build only (tools/native/libsquidpy_b200_clocks.so, make -C squidpy_b200/csrc clocks), which this script loads unless
$SQB_LIB_PATH names another build with the clocks.  usage: python tools/apply_phases.py [P] [algo:threads:r[:key=value...]] ..."""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, ".")
os.environ.setdefault("SQB_LIB_PATH", os.path.abspath("tools/native/libsquidpy_b200_clocks.so"))
import squidpy_b200 as sq  # noqa: E402
from squidpy_b200 import _lib  # noqa: E402
from squidpy_b200._rng import spawn_states  # noqa: E402
from squidpy_b200.gr import NhoodPlan  # noqa: E402
from tools import synth  # noqa: E402

# the order of SqbPartClk in squidpy_b200/csrc/nhood.cu
PHASES = ["entry", "gather", "A", "barrier 1", "B", "barrier 2", "C", "barrier 3", "clear", "region"]
N = len(PHASES) + 2

lib = C.CDLL(_lib.LIB_PATH)
lib.sqb_test_part_clocks.restype = C.c_int
lib.sqb_test_part_clocks.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]

args = sys.argv[1:]
P = int(args[0]) if args else 1000
variants = args[1:] or ["9:512:2"]
ctx = sq.default_context(0)
g = synth.hex_graph(1000, 1000)
base = synth.categorical_labels(g.shape[0], 30, seed=0).cat.codes.to_numpy().astype(np.uint32)
for v in variants:
    parts = v.split(":")
    plan = NhoodPlan(g.indptr, g.indices, 30, ctx)
    plan.set_option("shuffle_algo", int(parts[0]))
    plan.set_option("shuffle_threads", int(parts[1]))
    plan.set_option("shuffle_r", int(parts[2]))
    for kv in parts[3:]:
        k, x = kv.split("=")
        plan.set_option(k, int(x))
    plan.set_base(base)
    plan.upload(spawn_states(0, P))
    plan.run_async()
    ctx.sync()
    clk = (C.c_ulonglong * N)()
    assert lib.sqb_test_part_clocks(None, 1) == 0
    ctx.profile(True)
    ctx.profile_reset()
    plan.run_async()
    ctx.sync()
    ms = ctx.profile_get("shuffle")[0]
    ctx.profile(False)
    assert lib.sqb_test_part_clocks(clk, 1) == 0
    plan.close()
    windows, regions = clk[N - 2], clk[N - 1]
    assert windows > 0, "no window ran: is this the region replay (algo 9) in a build with the phase clocks?"
    per_window = sum(clk[:N - 3]) / windows
    print(f"{v}  P={P}  apply {ms:.3f} ms  {windows} windows, {regions} region passes  {per_window:.0f} cycles/window")
    for i, name in enumerate(PHASES[:-1]):
        print(f"  {name:10s} {clk[i] / windows:8.0f} cycles/window  {100 * clk[i] / windows / per_window:5.1f} %")
    print(f"  {'region':10s} {clk[N - 3] / regions:8.0f} cycles/region pass ({clk[N - 3] / windows:.0f} per window)", flush=True)
