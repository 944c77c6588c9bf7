"""Exact-mode nhood at configs[1] (1M spots, 30 clusters, P permutations): what transposing the finished label groups under
the region replay's last round costs that round and saves the step.  usage: python tools/tail_time.py [P] [reps]

Three plans on one context, measured in turn `reps` times in one process:
  overlap       the product path (tail_overlap 1): the last round beside the transpose of the whole rounds' groups;
  no_overlap    tail_overlap 0: one replay launch, then the whole transpose;
  whole_rounds  the P_A = floor(P / grid) * grid permutations of the whole rounds alone (one launch).
For each: the step (CUDA events around run_async with the L2 flushed before it, median of 10) and one profiled run's
per-class times.  The last round's time (`last_round`) is the apply (`shuffle`) of a plan less that of whole_rounds; in the
overlap plan it runs beside the early transpose, and that plan's `transpose` adds the early transpose's own span (from the
end of the whole rounds to its last CTA, overlapping the last round) to the remaining groups' transpose.  The counts of
overlap and no_overlap are compared."""
import json
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
import squidpy_b200 as sq  # noqa: E402
from squidpy_b200._rng import spawn_states  # noqa: E402
from squidpy_b200.gr import NhoodPlan  # noqa: E402
from tools import synth  # noqa: E402

P = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
stream = torch.cuda.Stream()
torch.cuda.set_stream(stream)
ctx = sq.Context(0, stream.cuda_stream)
flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
g = synth.hex_graph(1000, 1000)
base = synth.categorical_labels(g.shape[0], 30, seed=0).cat.codes.to_numpy().astype(np.uint32)
grid = 2 * ctx.sm_count  # two 512-thread replay CTAs per SM at 1M u8 spots
PA = P // grid * grid
st = spawn_states(0, P)


def make(n_perms, overlap):
    plan = NhoodPlan(g.indptr, g.indices, 30, ctx)
    plan.set_option("tail_overlap", overlap)
    plan.set_base(base)
    plan.upload(st[:n_perms])
    plan.run_async()
    ctx.sync()
    return plan


def step_ms(plan, n=10):
    ts = []
    for _ in range(n):
        flush_buf.add_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        plan.run_async()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def profiled(plan):
    flush_buf.add_(1)
    ctx.sync()
    ctx.profile(True)
    ctx.profile_reset()
    plan.run_async()
    ctx.sync()
    k = {name: round(ctx.profile_get(name)[0], 3) for name in ("misc", "shuffle", "transpose", "count")}
    ctx.profile(False)
    k["jgen"] = k.pop("misc")
    return k


plans = {"overlap": make(P, 1), "no_overlap": make(P, 0), "whole_rounds": make(PA, 1)}
print(json.dumps({"P": P, "grid": grid, "P_A": PA, "groups_early": PA // 64, "groups": -(-P // 64), "device": torch.cuda.get_device_name(0)}),
      flush=True)
for r in range(reps):
    res = {name: dict(step=round(step_ms(plan), 3), **profiled(plan)) for name, plan in plans.items()}
    whole = res["whole_rounds"]["shuffle"]
    for name in ("overlap", "no_overlap"):
        res[name]["last_round"] = round(res[name]["shuffle"] - whole, 3)
    print(json.dumps({"rep": r, **res}), flush=True)
same = np.array_equal(plans["overlap"].download(), plans["no_overlap"].download())
print(json.dumps({"counts_equal": bool(same)}), flush=True)
for plan in plans.values():
    plan.close()
