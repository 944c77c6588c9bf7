"""nhood_enrichment(copy=True) end to end on configs[1] (1000 x 1000 hex lattice = 1M spots, 30 clusters, 1000 permutations)
with the neighbour graph on the host (scipy CSR) against the same graph already in GPU memory (a torch sparse_csr CUDA tensor
with int64 indices).  Median of REPS calls each, the two alternating; prints the GPU and its power limit next to the numbers
and checks that both results are equal.
    python tools/nhood_device_graph.py [reps]"""
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, ".")
import torch  # noqa: E402

import squidpy_b200 as sq  # noqa: E402
from tools import synth  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 5
if not torch.cuda.is_available():
    sys.exit("no CUDA device: this script measures the GPU path and has nothing to fall back to")
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
print("gpu:", q.stdout.strip() or torch.cuda.get_device_name(0), flush=True)

g = synth.hex_graph(1000, 1000)
labels = synth.categorical_labels(g.shape[0], 30, seed=0)
host = synth.make_adata(synth.hex_coords(1000, 1000), g, labels)
dev = synth.make_adata(synth.hex_coords(1000, 1000), None, labels)
dev.obsp["spatial_connectivities"] = torch.sparse_csr_tensor(torch.from_numpy(g.indptr.astype(np.int64)), torch.from_numpy(g.indices.astype(np.int64)),
                                                             torch.from_numpy(g.data), size=g.shape).cuda()
torch.cuda.synchronize()
print(f"configs[1]: {g.shape[0]} spots, nnz {g.nnz}, host graph (int32 CSR) {(g.indptr.nbytes + g.indices.nbytes) / 1e6:.1f} MB", flush=True)


def timed(adata):
    t0 = time.perf_counter()
    r = sq.gr.nhood_enrichment(adata, "cluster", n_perms=1000, seed=0, copy=True)  # host numpy results: ends synchronised
    return time.perf_counter() - t0, r


ts = {"host graph": [], "device graph": []}
res = {}
for a in (host, dev):
    timed(a)  # warm-up
for _ in range(REPS):
    for name, a in (("host graph", host), ("device graph", dev)):
        t, res[name] = timed(a)
        ts[name].append(t)
for name, v in ts.items():
    print(f"nhood_enrichment(copy=True, n_perms=1000), {name}: median {statistics.median(v) * 1e3:.1f} ms over {REPS} calls "
          f"(min {min(v) * 1e3:.1f}, max {max(v) * 1e3:.1f})", flush=True)
h, d = res["host graph"], res["device graph"]
same = np.array_equal(h.counts, d.counts) and np.array_equal(h.zscore, d.zscore, equal_nan=True)
print("device result == host result bit for bit:", same, flush=True)
