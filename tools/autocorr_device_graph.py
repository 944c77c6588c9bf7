"""spatial_autocorr(copy=True) with X in GPU memory and the weight matrix W in GPU memory (a torch sparse_csr CUDA tensor with
int64 indices, float32 or float64 ones, row-normalised on the device) against the same call through the host copy of W (sklearn's
normalize, the host upload and scipy's moments: the path every device W took before the device build existed).  Workloads:
a 447 x 447 hex lattice (configs[2]'s graph) with 20 000 genes at density 0.01 (configs[2] itself has 0.1), and a 1000 x 1000
hex lattice (1M spots) with 2 000 genes at density 0.01, the latter with a float32 and a float64 W (float64 row-normalised
weights take the ordered S0 chain on one thread).  Median of
REPS calls each, the two paths alternating; the time of sqb_autocorr_create_device alone (CUDA events on the library's stream)
is reported separately.  Prints the GPU and its power limit next to the numbers and checks that both results are equal.
    python tools/autocorr_device_graph.py [reps]"""
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, ".")
import torch  # noqa: E402

import squidpy_b200 as sq  # noqa: E402
import squidpy_b200.gr._ppatterns as pp  # noqa: E402
from squidpy_b200._device import device_matrix, graph_args  # noqa: E402
from tools import synth  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 5
if not torch.cuda.is_available():
    sys.exit("no CUDA device: this script measures the GPU path and has nothing to fall back to")
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
print("gpu:", q.stdout.strip() or torch.cuda.get_device_name(0), flush=True)
from_device = pp.AutocorrPlan.from_device


def torch_csr(m):
    return torch.sparse_csr_tensor(torch.from_numpy(m.indptr.astype(np.int64)), torch.from_numpy(m.indices.astype(np.int64)),
                                   torch.from_numpy(m.data), size=m.shape).cuda()


def timed(adata, host_copy):
    # host_copy: the device build declines W, so spatial_autocorr copies it to the host and proceeds as for a host graph
    pp.AutocorrPlan.from_device = (lambda *a, **k: None) if host_copy else from_device
    try:
        t0 = time.perf_counter()
        r = sq.gr.spatial_autocorr(adata, copy=True)  # a host DataFrame: ends synchronised
        return time.perf_counter() - t0, r
    finally:
        pp.AutocorrPlan.from_device = from_device


def create_ms(w):
    """sqb_autocorr_create_device alone: CUDA events on the context's stream around the call."""
    ctx = sq.default_context()
    s = torch.cuda.ExternalStream(ctx.stream) if ctx.stream else torch.cuda.default_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    graph = graph_args(device_matrix(w), w.shape[0])
    out = []
    for _ in range(REPS):
        e0.record(s)
        plan = from_device(graph, True, ctx)
        e1.record(s)
        e1.synchronize()
        out.append(e0.elapsed_time(e1))
        plan.close()
    return statistics.median(out)


WORKLOADS = {"447 x 447 hex, 20 000 genes @0.01, float32 W": (447, 447, 20000, 0.01, np.float32),
             "1M hex, 2 000 genes @0.01, float32 W": (1000, 1000, 2000, 0.01, np.float32),
             "1M hex, 2 000 genes @0.01, float64 W": (1000, 1000, 2000, 0.01, np.float64)}
for name, (rows, cols, genes, density, wdt) in WORKLOADS.items():
    g = synth.hex_graph(rows, cols).astype(wdt)
    x = synth.expression_csr(g.shape[0], genes, density=density, coords=synth.hex_coords(rows, cols), seed=0)
    ad = synth.make_adata(synth.hex_coords(rows, cols), None, None, X=torch_csr(x))
    ad.obsp["spatial_connectivities"] = w = torch_csr(g)
    torch.cuda.synchronize()
    print(f"{name}: {g.shape[0]} spots, W nnz {g.nnz}, X {genes} genes, nnz {x.nnz}", flush=True)
    ts = {"device W": [], "host copy of W": []}
    res = {}
    for hc in (False, True):
        timed(ad, hc)  # warm-up
    for _ in range(REPS):
        for label, hc in (("device W", False), ("host copy of W", True)):
            t, res[label] = timed(ad, hc)
            ts[label].append(t)
    for label, v in ts.items():
        print(f"  spatial_autocorr(copy=True), device X, {label}: median {statistics.median(v) * 1e3:.1f} ms over {REPS} calls "
              f"(min {min(v) * 1e3:.1f}, max {max(v) * 1e3:.1f})", flush=True)
    print(f"  sqb_autocorr_create_device (transformation=True): median {create_ms(w):.2f} ms", flush=True)
    a, b = res["device W"], res["host copy of W"]
    same = list(a.index) == list(b.index) and np.array_equal(a.to_numpy(np.float64), b.to_numpy(np.float64), equal_nan=True)
    print("  device result == host-copy result bit for bit:", same, flush=True)
