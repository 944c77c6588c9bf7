"""spatial_autocorr(copy=True) end to end on configs[2] (199 809 spots x G genes, CSR float32 at 10 %) with adata.X on the host
and with the same X already resident on the device (a torch sparse CSR tensor with int32 indices, what cupyx.scipy.sparse
holds), plus the device load alone (the autocorr_prep kernel class).  Prints the GPU and its power limit next to the numbers.
    python tools/autocorr_device_input.py [G] [reps]"""
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, ".")
import torch  # noqa: E402

import squidpy_b200 as sq  # noqa: E402
from squidpy_b200 import AnnDataLite  # noqa: E402
from squidpy_b200.gr import AutocorrPlan  # noqa: E402
from tools import synth  # noqa: E402

G = int(sys.argv[1]) if len(sys.argv) > 1 else 20000
REPS = int(sys.argv[2]) if len(sys.argv) > 2 else 5
if not torch.cuda.is_available():
    sys.exit("no CUDA device: this script measures the GPU path and has nothing to fall back to")
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
print("gpu:", q.stdout.strip() or torch.cuda.get_device_name(0), flush=True)

g = synth.hex_graph(447, 447).astype(np.float32)
x = synth.expression_csr(g.shape[0], G, density=0.1, coords=synth.hex_coords(447, 447), seed=1)
print(f"configs[2]: {x.shape[0]} x {x.shape[1]}, nnz {x.nnz}, X {x.data.nbytes + x.indices.nbytes + x.indptr.nbytes >> 20} MB", flush=True)
import pandas as pd  # noqa: E402

var = pd.DataFrame(index=[f"g{i}" for i in range(G)])
xd = torch.sparse_csr_tensor(torch.from_numpy(x.indptr.astype(np.int32)), torch.from_numpy(x.indices.astype(np.int32)),
                             torch.from_numpy(x.data), size=x.shape).cuda()
torch.cuda.synchronize()
host = AnnDataLite(X=x, obsp={"spatial_connectivities": g}, var=var)
dev = AnnDataLite(X=xd, obsp={"spatial_connectivities": g}, var=var)


def timed(adata):
    t0 = time.perf_counter()
    df = sq.gr.spatial_autocorr(adata, copy=True)  # returns host numpy / pandas: ends in a device synchronise
    return time.perf_counter() - t0, df


res = {}
for name, a in (("host X", host), ("device X", dev)):
    timed(a)  # warm-up
for name, a in (("host X", host), ("device X", dev)):
    ts = []
    for _ in range(REPS):  # alternate-free but back to back: both runs in the same process and on the same card
        t, df = timed(a)
        ts.append(t)
    res[name] = df
    print(f"spatial_autocorr(copy=True), {name}: median {statistics.median(ts) * 1e3:.1f} ms over {REPS} calls "
          f"(min {min(ts) * 1e3:.1f}, max {max(ts) * 1e3:.1f})", flush=True)
same = np.array_equal(res["host X"].to_numpy(np.float64), res["device X"].to_numpy(np.float64), equal_nan=True) and list(
    res["host X"].index) == list(res["device X"].index)
print("device result == host result bit for bit:", same, flush=True)

ctx = sq.default_context(0)
from sklearn.preprocessing import normalize  # noqa: E402

w = g.copy()
normalize(w, norm="l1", axis=1, copy=False)
plan = AutocorrPlan(w, ctx)
plan.load(xd, obs_major=True)
ctx.sync()
loads, prep = [], []
for _ in range(REPS):
    ctx.profile(True)
    ctx.profile_reset()
    plan.load(xd, obs_major=True)
    ctx.sync()
    prep.append(ctx.profile_get("autocorr_prep")[0])
    ctx.profile(False)
    t0 = time.perf_counter()
    plan.load(xd, obs_major=True)
    loads.append(time.perf_counter() - t0)
ctx.profile_reset()
ctx.profile(True)
plan.score("moran")
ctx.sync()
main_ms = ctx.profile_get("autocorr_main")[0]
ctx.profile(False)
plan.close()
print(f"device load: median {statistics.median(loads) * 1e3:.1f} ms wall, autocorr_prep kernels {statistics.median(prep):.1f} ms "
      f"(CUDA events, profiled pass); Moran main kernel {main_ms:.1f} ms", flush=True)
