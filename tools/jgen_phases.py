"""Where the partitioned target generation (nhood_jgen_kernel<Q, true>, shuffle_algo 9) spends its time at configs[1] (1M
spots, 30 clusters, P permutations): the clock totals of its generator and partition warps, summed over the warps as lane 0
of each sees them.  Generator: the share of its run spent waiting for a free block buffer.  Partition warp: cycles per
2048-step block of its wait for a full buffer and of its count, scan, scatter and stream-out.  They exist in the clocks build
only (tools/native/libsquidpy_b200_clocks.so, make -C squidpy_b200/csrc clocks), which this script loads unless $SQB_LIB_PATH
names another build with the clocks.  usage: python tools/jgen_phases.py [P]"""
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

# the order of SqbJgenClk in squidpy_b200/csrc/nhood.cu
GEN_WAIT, GEN_RUN, PART_WAIT, COUNT, SCAN, SCATTER, STREAM, PART_RUN, BLOCKS = range(9)
N = 9

lib = C.CDLL(_lib.LIB_PATH)
lib.sqb_test_jgen_clocks.restype = C.c_int
lib.sqb_test_jgen_clocks.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]

P = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
ctx = sq.default_context(0)
g = synth.hex_graph(1000, 1000)
base = synth.categorical_labels(g.shape[0], 30, seed=0).cat.codes.to_numpy().astype(np.uint32)
plan = NhoodPlan(g.indptr, g.indices, 30, ctx)
plan.set_base(base)
plan.upload(spawn_states(0, P))
plan.run_async()
ctx.sync()
clk = (C.c_ulonglong * N)()
assert lib.sqb_test_jgen_clocks(None, 1) == 0
ctx.profile(True)
ctx.profile_reset()
plan.run_async()
ctx.sync()
ms = ctx.profile_get("misc")[0]
ctx.profile(False)
assert lib.sqb_test_jgen_clocks(clk, 1) == 0
plan.close()
blocks = clk[BLOCKS]
assert blocks > 0, "no block was partitioned: is this a build with the clocks?"
print(f"P={P}  target generation {ms:.3f} ms  {blocks} blocks of 2048 steps")
print(f"  generator: waits for a free buffer {clk[GEN_WAIT] / blocks:8.0f} cycles/block  "
      f"{100 * clk[GEN_WAIT] / clk[GEN_RUN]:5.1f} % of its run ({clk[GEN_RUN] / blocks:.0f} cycles/block)")
print(f"  partition warp, cycles/block ({clk[PART_RUN] / blocks:.0f} per block over its run):")
for name, k in (("wait full", PART_WAIT), ("count", COUNT), ("scan", SCAN), ("scatter", SCATTER), ("stream-out", STREAM)):
    print(f"    {name:10s} {clk[k] / blocks:8.0f}  {100 * clk[k] / clk[PART_RUN]:5.1f} %", flush=True)
