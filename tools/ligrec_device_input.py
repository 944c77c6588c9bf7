"""ligrec(copy=True) and sepal(copy=True) end to end with adata.X on the host and with the same X already resident on the
device (a torch sparse CSR tensor with int32 indices, what cupyx.scipy.sparse holds).  Calls alternate host / device; the
medians are printed next to the GPU and its power limit, and the two results are compared.
    python tools/ligrec_device_input.py [n_cells] [n_genes] [n_interactions] [n_perms] [reps] [sepal_genes]"""
import statistics
import subprocess
import sys
import time

import numpy as np
import pandas as pd

sys.path.insert(0, ".")
import torch  # noqa: E402

import squidpy_b200 as sq  # noqa: E402
from squidpy_b200 import AnnDataLite  # noqa: E402
from tools import synth  # noqa: E402

args = [int(a) for a in sys.argv[1:]]
N, G, NI, P, REPS, SG = (args + [100_000, 5000, 500, 1000, 3, 300][len(args):])[:6]
if not torch.cuda.is_available():
    sys.exit("no CUDA device: this script measures the GPU path and has nothing to fall back to")
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
print("gpu:", q.stdout.strip() or torch.cuda.get_device_name(0), flush=True)


def to_device(x):
    return torch.sparse_csr_tensor(torch.from_numpy(x.indptr.astype(np.int32)), torch.from_numpy(x.indices.astype(np.int32)),
                                   torch.from_numpy(x.data), size=x.shape).cuda()


def alternate(name, calls, reps):
    """calls: {label: fn}; one warm-up each, then reps rounds alternating the labels; returns the last result per label."""
    out, ts = {}, {k: [] for k in calls}
    for k, f in calls.items():
        out[k] = f()
    for _ in range(reps):
        for k, f in calls.items():
            t0 = time.perf_counter()
            out[k] = f()  # returns host pandas frames: ends in a device synchronise
            ts[k].append(time.perf_counter() - t0)
    for k, v in ts.items():
        print(f"{name}, {k}: median {statistics.median(v) * 1e3:.1f} ms over {reps} calls (min {min(v) * 1e3:.1f}, max {max(v) * 1e3:.1f})",
              flush=True)
    return out


# ---- ligrec: N cells x G genes CSR float32 at 10 %, NI interactions among the genes, 10 clusters, P permutations
rng = np.random.default_rng(0)
x = synth.expression_csr(N, G, density=0.1, seed=1).astype(np.float32)
names = [f"G{i}" for i in range(G)]
inter = pd.DataFrame({"source": rng.choice(names, NI), "target": rng.choice(names, NI)})
obs = pd.DataFrame({"cl": pd.Categorical(rng.integers(0, 10, N).astype(str))}, index=[f"c{i}" for i in range(N)])
var = pd.DataFrame(index=names)
xd = to_device(x)
torch.cuda.synchronize()
print(f"ligrec: {N} x {G}, nnz {x.nnz}, {NI} interactions, {P} permutations", flush=True)
kw = dict(interactions=inter, n_perms=P, seed=0, copy=True, use_raw=False)
res = alternate("ligrec(copy=True)", {"host X": lambda: sq.gr.ligrec(AnnDataLite(X=x, obs=obs, var=var), "cl", **kw),
                                      "device X": lambda: sq.gr.ligrec(AnnDataLite(X=xd, obs=obs, var=var, shape=x.shape), "cl", **kw)}, REPS)
same = all(np.array_equal(res["host X"][k].sparse.to_dense().to_numpy(np.float64), res["device X"][k].sparse.to_dense().to_numpy(np.float64),
                          equal_nan=True) for k in ("means", "pvalues"))
print("ligrec device result == host result bit for bit:", same, flush=True)
del xd

# ---- sepal: SG genes on a 300 x 300 hex lattice, CSR float32 at 30 %
g = synth.hex_graph(300, 300)
co = synth.hex_coords(300, 300)
xs = synth.expression_csr(g.shape[0], SG, density=0.3, coords=co, seed=2).astype(np.float32)
xsd = to_device(xs)
torch.cuda.synchronize()
svar = pd.DataFrame(index=[f"S{i}" for i in range(SG)])
print(f"sepal: {g.shape[0]} spots x {SG} genes, nnz {xs.nnz}", flush=True)
skw = dict(max_neighs=6, copy=True)
sres = alternate("sepal(copy=True)", {
    "host X": lambda: sq.gr.sepal(AnnDataLite(X=xs, obsp={"spatial_connectivities": g}, obsm={"spatial": co}, var=svar), **skw),
    "device X": lambda: sq.gr.sepal(AnnDataLite(X=xsd, obsp={"spatial_connectivities": g}, obsm={"spatial": co}, var=svar, shape=xs.shape),
                                    **skw)}, REPS)
print("sepal device result == host result bit for bit:", sres["host X"].equals(sres["device X"]), flush=True)
